/*
 * oracle/remove_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The removal faiss 1.6.x IndexIVF::remove_ids performs without a direct map (DirectMap::NoMap) [3P], written literally, on list-major
 * arrays (DESIGN.md 3.2).  Per list:
 *     j = 0, l = len;  while (j < l) { if (selected(id[j])) { l--; row[j] = row[l]; id[j] = id[l]; } else j++; }
 * then the lists are packed again.  selected(): the label is in sel[0 .. n_sel) (sorted ascending, as a binary search sees it), or,
 * with sel NULL, in [lo, hi).
 * What pins it: tests/test_remove_cpu.py (the numpy closed form np_remove on random selections and ragged lists, hand examples).
 *
 * Only tests/, __graft_entry__.smoke() and tools/bench_remove.py's host baseline may load this library.
 */
#include <stdint.h>
#include <string.h>

#define REF_API __attribute__((visibility("default")))

static int selected(int64_t id, const int64_t* sel, int64_t n_sel, int64_t lo, int64_t hi) {
    if (!sel) return lo <= id && id < hi;
    int64_t a = 0, b = n_sel;
    while (a < b) { int64_t mid = (a + b) / 2; if (sel[mid] < id) a = mid + 1; else b = mid; }
    return a < n_sel && sel[a] == id;
}

/* list_len [nlist] (in: lengths, out: new lengths), codes [ntotal, code_size] and ids [ntotal] list-major, modified in place (the
 * survivors packed at the front).  removed_per_list [nlist] out.  Returns the number of rows removed. */
REF_API int64_t ref_remove(int64_t nlist, int64_t* list_len, uint8_t* codes, int64_t* ids, int code_size, const int64_t* sel, int64_t n_sel,
                           int64_t lo, int64_t hi, int64_t* removed_per_list) {
    int64_t src = 0, dst = 0, total = 0;
    for (int64_t li = 0; li < nlist; li++) {
        const int64_t len = list_len[li];
        uint8_t* c = codes + (size_t)src * code_size;
        int64_t* id = ids + src;
        int64_t j = 0, l = len;
        while (j < l) {
            if (selected(id[j], sel, n_sel, lo, hi)) {
                l--;
                memmove(c + (size_t)j * code_size, c + (size_t)l * code_size, code_size);     /* j == l: itself */
                id[j] = id[l];
            } else j++;
        }
        memmove(codes + (size_t)dst * code_size, c, (size_t)l * code_size);
        memmove(ids + dst, id, (size_t)l * sizeof(int64_t));
        removed_per_list[li] = len - l;
        total += len - l;
        list_len[li] = l;
        src += len; dst += l;
    }
    return total;
}
