/*
 * oracle/filter_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the filtered search (DESIGN.md 3.6): faiss IndexIVF::search_preassigned with SearchParametersIVF(sel=...)
 * (faiss >= 1.7.3) [3P] at the index's nprobe -- the same probes and dis0 as the unfiltered search, and in the scan of every probed
 * list a row whose label is not selected is skipped before the heap.  ivfpq_ref.c is compiled into this library, so the rotation, the
 * coarse quantizer, the tables, the heap and the inverted lists are literally the search oracle's own code.
 * What pins it: tests/test_filter_cpu.py (equal to tests/filter_ref.py's numpy restatement bit for bit; selecting every row gives the
 * unfiltered oracle's result).
 *
 * Only tests/ and tools/bench_filter.py may load this library.
 */
#include "ivfpq_ref.c"

/* == ref_search_preassigned with selected [ntotal] (one byte per list-major row list_off[l] + j, non-zero: selected).  Rows are scored
 * one at a time in storage order: dis = dis0; for m ascending: dis += LUT[m][c[m]] (the same values as the unfiltered loop). */
REF_API void ref_search_preassigned_filtered(const ref_index* ix, const float* xr, int64_t n, const int64_t* key, int nprobe, int k,
                                             const uint8_t* selected, float* D, int64_t* I) {
#pragma omp parallel
    {
        float* lut = (float*)malloc(sizeof(float) * ix->M * ix->ksub);
        float* cen = (float*)malloc(sizeof(float) * ix->d);
        uint8_t* scratch = NULL; size_t cap = 0;
#pragma omp for schedule(dynamic, 1)
        for (int64_t i = 0; i < n; i++) {
            const float* q = xr + i * ix->d;
            float* simi = D + i * k; int64_t* idxi = I + i * k;
            ref_lut(q, ix->pq, ix->M, ix->ksub, ix->dsub, lut);
            heap_heapify(k, simi, idxi);
            for (int r = 0; r < nprobe; r++) {
                const int64_t l = key[i * nprobe + r];
                if (l < 0) continue;
                const int64_t len = ix->list_len[l];
                if (len == 0) continue;
                centroid_row(ix, l, cen);
                const float dis0 = dot_seq(q, cen, ix->d);
                const uint8_t* codes = list_codes(ix, l, &scratch, &cap);
                for (int64_t j = 0; j < len; j++) {
                    if (!selected[ix->list_off[l] + j]) continue;
                    const uint8_t* c = codes + j * ix->code_size;
                    const float* tab = lut;
                    float dis = dis0;
                    for (int m = 0; m < ix->M; m++) { dis += tab[c[m]]; tab += ix->ksub; }
                    if (simi[0] < dis) { heap_pop(k, simi, idxi); heap_push(k, simi, idxi, dis, list_id(ix, l, j)); }
                }
            }
            heap_reorder(k, simi, idxi);
        }
        free(lut); free(cen); free(scratch);
    }
}
