// query_filter.cu -- per-query filters for the filtered search (DESIGN.md 3.7, "Per-query filters"): F label selectors and the selector of
// every query of one batch.  Each selector is held sparse, as a CSR over the shard's lists: per list, the ascending block numbers that
// hold a selected row, and each such block's mask word (bit l = lane l's row is selected, as the row mask of filter.cu).  The one-query
// scan (scan.cu, DPH_FILT_QUERY) then walks only those blocks.  Building one reads the index and changes nothing; its cost follows the
// selected rows, not the shard.
#include "index_internal.cuh"
#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/functional.h>
#include <thrust/iterator/transform_iterator.h>
#include <thrust/reduce.h>
#include <thrust/scan.h>
#include <thrust/sort.h>

// A hit key: selector << 40 | the row's padded row in the shard (shard block * 32 + lane).  Sorted, the keys run by (selector, list,
// block, lane); key >> 5 is the (selector, shard block) pair that one mask word covers.
#define QF_ROW_BITS 40
#define QF_BLK_BITS (QF_ROW_BITS - 5)

__device__ __forceinline__ long long upper_bound_qf(const long long* a, long long n, long long key) {      // first i with a[i] > key
    long long lo = 0, hi = n;
    while (lo < hi) { const long long mid = (lo + hi) >> 1; if (a[mid] <= key) lo = mid + 1; else hi = mid; }
    return lo;
}

struct QfRunArgs {
    const long long* labels; long long nlab; const long long* lab_off; const long long* ranges; int nsel;
    const long long* dm_ids; long long dm_n;             // explicit labels: the direct map, sorted by label
    const long long* list_start; long long lo, hi;       // sequential labels: label = list_start[l] + j
    int* run_sel; long long* run_first; long long* run_cnt;
};
// Runs of hits: one per label (r < nlab) and one per range selector (r = nlab + s).  Explicit labels: a run of direct-map pairs
// [first, first + cnt) (a label on two rows is a run of two); sequential labels: a run of labels, every one of them a row of the shard.
__global__ void qf_runs_kernel(QfRunArgs a) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.nlab + a.nsel) return;
    long long first = 0, cnt = 0;
    int s;
    if (r < a.nlab) {
        s = (int)(upper_bound_qf(a.lab_off, a.nsel + 1, r) - 1);
        const long long label = a.labels[r];
        if (a.dm_ids) {
            first = lower_bound_ll(a.dm_ids, a.dm_n, label);
            cnt = upper_bound_qf(a.dm_ids, a.dm_n, label) - first;
        } else if (label >= a.list_start[a.lo] && label < a.list_start[a.hi]) {
            first = label; cnt = 1;
        }
    } else {
        s = (int)(r - a.nlab);
        const long long rlo = a.ranges ? a.ranges[2 * s] : 0, rhi = a.ranges ? a.ranges[2 * s + 1] : 0;
        if (rlo < rhi) {
            if (a.dm_ids) {
                first = lower_bound_ll(a.dm_ids, a.dm_n, rlo);
                cnt = lower_bound_ll(a.dm_ids, a.dm_n, rhi) - first;
            } else {
                const long long s0 = max(rlo, a.list_start[a.lo]), s1 = min(rhi, a.list_start[a.hi]);
                if (s0 < s1) { first = s0; cnt = s1 - s0; }
            }
        }
    }
    a.run_sel[r] = s; a.run_first[r] = first; a.run_cnt[r] = cnt;
}

// One thread per hit h: its run (the last run starting at or before h), its row, its key.
__global__ void qf_keys_kernel(const int* run_sel, const long long* run_first, const long long* run_off, long long R, long long H,
                               const long long* dm_rows, const long long* list_start, const long long* blk_off, long long lo, long long hi,
                               unsigned long long* keys) {
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= H) return;
    const long long r = upper_bound_qf(run_off, R, h) - 1;
    const long long t = run_first[r] + h - run_off[r];
    long long prow;
    if (dm_rows) prow = dm_rows[t];
    else {
        const long long l = lo + upper_bound_qf(list_start + lo, hi - lo, t) - 1;       // the list holding label t
        prow = blk_off[l] * 32 + (t - list_start[l]);
    }
    keys[h] = ((unsigned long long)run_sel[r] << QF_ROW_BITS) | (unsigned long long)prow;
}

struct QfBlockOf { __host__ __device__ unsigned long long operator()(unsigned long long k) const { return k >> 5; } };
struct QfBitOf { __host__ __device__ unsigned operator()(unsigned long long k) const { return 1u << (unsigned)(k & 31u); } };

// One thread per (selector, shard block) entry: the list's block number, the word, the selector's row count.
__global__ void qf_entries_kernel(const unsigned long long* ukeys, const unsigned* uwords, long long U, const long long* blk_off, long long lo,
                                  long long hi, uint32_t* blk, uint32_t* word, unsigned long long* rows) {
    const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= U) return;
    const long long sb = (long long)(ukeys[u] & ((1ull << QF_BLK_BITS) - 1));
    const long long l = list_of_block(blk_off, lo, hi, sb);
    blk[u] = (uint32_t)(sb - blk_off[l]);
    word[u] = uwords[u];
    atomicAdd(rows + (ukeys[u] >> QF_BLK_BITS), (unsigned long long)__popc(uwords[u]));
}
// One thread per (selector s, shard list lo + i), i <= nl: the selector's first entry at or after the list's first block, relative to
// the selector's first entry base[s] (i = nl: the selector's end).
__global__ void qf_offsets_kernel(const unsigned long long* ukeys, long long U, const long long* blk_off, long long lo, long long nl,
                                  long long nblocks, long long nsel, uint32_t* off, long long* base) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nsel * (nl + 1)) return;
    const long long s = t / (nl + 1), i = t % (nl + 1);
    const long long* k = (const long long*)ukeys;
    const long long b0 = lower_bound_ll(k, U, s << QF_BLK_BITS);
    const long long key = (s << QF_BLK_BITS) | (i < nl ? blk_off[lo + i] : nblocks);
    off[t] = (uint32_t)(lower_bound_ll(k, U, key) - b0);
    if (i == 0) base[s] = b0;
    if (t == 0) base[nsel] = U;
}

DPH_API int dph_query_filter_create(dph_query_filter** out, dph_index* ix, const int64_t* labels, const int64_t* label_off,
                                    const int64_t* ranges, int64_t nsel, const int32_t* assign, int64_t n, int mem) {
    DPH_CHECK(out != nullptr, "make_query_filters: null out");
    *out = nullptr;
    DPH_CHECK(ix && ix->list_len, "make_query_filters: lists are not set");
    DPH_CHECK(nsel >= 0 && nsel < (1ll << (63 - QF_ROW_BITS)), "make_query_filters: bad selector count");
    DPH_CHECK(n >= 0 && (assign != nullptr || n == 0), "make_query_filters: bad assignment array");
    DPH_CHECK(nsel == 0 || label_off != nullptr || ranges != nullptr, "make_query_filters: give label offsets or ranges");
    DPH_CHECK(ix->nblocks_local < (1ll << QF_BLK_BITS), "make_query_filters: the shard has too many code blocks");
    for (int64_t q = 0; q < n; q++)
        if (assign[q] < -1 || assign[q] >= nsel) {
            dph_set_error("make_query_filters: query " + std::to_string(q) + " is assigned selector " + std::to_string(assign[q]) +
                          "; selectors are 0.." + std::to_string(nsel - 1) + ", or -1 for none");
            return 1;
        }
    int64_t nlab = 0;
    if (label_off) {
        DPH_CHECK(nsel == 0 || label_off[0] == 0, "make_query_filters: label offsets must start at 0");
        for (int64_t s = 0; s < nsel; s++) {
            DPH_CHECK(label_off[s + 1] >= label_off[s], "make_query_filters: label offsets must not decrease");
            const bool has_labels = label_off[s + 1] > label_off[s];
            const bool has_range = ranges && (ranges[2 * s] != 0 || ranges[2 * s + 1] != 0);
            if (has_labels && has_range) {
                dph_set_error("make_query_filters: selector " + std::to_string(s) + ": give a label set or a label range, not both");
                return 1;
            }
        }
        nlab = nsel > 0 ? label_off[nsel] : 0;
        DPH_CHECK(labels != nullptr || nlab == 0, "make_query_filters: label offsets without labels");
    }
    DPH_CUDA(cudaSetDevice(ix->device));
    cudaStream_t st = ix->stream;
    const char* oom = "make_query_filters: not enough device memory for the filter";
    const int64_t lo = ix->list_lo, hi = ix->list_hi, nl = hi - lo, R = nlab + nsel;
    const bool explicit_ids = ix->ids != nullptr;
    DevTmp tmp;

    // 1. runs of hits, their offsets and the hit count H
    long long *d_labels = nullptr, *d_lab_off = nullptr, *d_ranges = nullptr, *run_first, *run_cnt, *run_off;
    int* run_sel;
    DPH_TRY(tmp.alloc(&run_sel, R, oom)); DPH_TRY(tmp.alloc(&run_first, R, oom)); DPH_TRY(tmp.alloc(&run_cnt, R, oom));
    DPH_TRY(tmp.alloc(&run_off, R + 1, oom));
    if (nlab > 0) {
        DPH_TRY(tmp.alloc(&d_labels, nlab, oom)); DPH_TRY(tmp.alloc(&d_lab_off, nsel + 1, oom));
        DPH_CUDA(cudaMemcpyAsync(d_labels, labels, (size_t)nlab * 8, mem == DPH_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, st));
        DPH_CUDA(cudaMemcpyAsync(d_lab_off, label_off, (size_t)(nsel + 1) * 8, cudaMemcpyHostToDevice, st));
    }
    if (ranges && nsel > 0) {
        DPH_TRY(tmp.alloc(&d_ranges, 2 * nsel, oom));
        DPH_CUDA(cudaMemcpyAsync(d_ranges, ranges, (size_t)nsel * 16, cudaMemcpyHostToDevice, st));
    }
    int64_t H = 0;
    if (R > 0) {
        QfRunArgs a;
        a.labels = d_labels; a.nlab = nlab; a.lab_off = d_lab_off; a.ranges = d_ranges; a.nsel = (int)nsel;
        a.dm_ids = explicit_ids ? (const long long*)ix->dm_ids : nullptr; a.dm_n = ix->dm_n;
        a.list_start = (const long long*)ix->list_start; a.lo = lo; a.hi = hi;
        a.run_sel = run_sel; a.run_first = run_first; a.run_cnt = run_cnt;
        qf_runs_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(a);
        DPH_CUDA(cudaGetLastError());
        try {
            thrust::device_ptr<long long> cp(run_cnt), op(run_off);
            thrust::inclusive_scan(thrust::cuda::par.on(st), cp, cp + R, op + 1);
        } catch (const std::exception& e) {
            cudaGetLastError();
            dph_set_error(std::string("make_query_filters: device scan failed: ") + e.what());
            return 1;
        }
        DPH_CUDA(cudaMemsetAsync(run_off, 0, 8, st));
        DPH_CUDA(cudaMemcpyAsync(&H, run_off + R, 8, cudaMemcpyDeviceToHost, st));
        DPH_CUDA(cudaStreamSynchronize(st));
    }

    // 2. one key per hit, sorted; OR-reduced per (selector, shard block) into U entries
    unsigned long long *keys = nullptr, *ukeys = nullptr;
    unsigned* uwords = nullptr;
    int64_t U = 0;
    if (H > 0) {
        DPH_TRY(tmp.alloc(&keys, H, oom)); DPH_TRY(tmp.alloc(&ukeys, H, oom)); DPH_TRY(tmp.alloc(&uwords, H, oom));
        qf_keys_kernel<<<(unsigned)((H + 255) / 256), 256, 0, st>>>(run_sel, run_first, run_off, R, H,
                                                                    explicit_ids ? (const long long*)ix->dm_rows : nullptr,
                                                                    (const long long*)ix->list_start, (const long long*)ix->blk_off, lo, hi, keys);
        DPH_CUDA(cudaGetLastError());
        try {
            thrust::device_ptr<unsigned long long> kp(keys), ukp(ukeys);
            thrust::device_ptr<unsigned> uwp(uwords);
            thrust::sort(thrust::cuda::par.on(st), kp, kp + H);
            auto kb = thrust::make_transform_iterator(kp, QfBlockOf());
            auto vb = thrust::make_transform_iterator(kp, QfBitOf());
            U = thrust::reduce_by_key(thrust::cuda::par.on(st), kb, kb + H, vb, ukp, uwp, thrust::equal_to<unsigned long long>(),
                                      thrust::bit_or<unsigned>()).first - ukp;
        } catch (const std::exception& e) {
            cudaGetLastError();
            dph_set_error(std::string("make_query_filters: device sort failed: ") + e.what());
            return 1;
        }
    }

    // 3. the filter's arrays (every allocation before any of them is written), the entries and the per-list offsets
    int32_t* d_assign; uint32_t *d_off, *d_blk, *d_word; int64_t* d_base; unsigned long long* d_rows;
    DPH_TRY(tmp.alloc(&d_assign, n, oom)); DPH_TRY(tmp.alloc(&d_off, nsel * (nl + 1), oom)); DPH_TRY(tmp.alloc(&d_base, nsel + 1, oom));
    DPH_TRY(tmp.alloc(&d_blk, U, oom)); DPH_TRY(tmp.alloc(&d_word, U, oom)); DPH_TRY(tmp.alloc(&d_rows, nsel, oom));
    if (n > 0) DPH_CUDA(cudaMemcpyAsync(d_assign, assign, (size_t)n * 4, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemsetAsync(d_rows, 0, (size_t)std::max<int64_t>(nsel, 1) * 8, st));
    DPH_CUDA(cudaMemsetAsync(d_base, 0, (size_t)(nsel + 1) * 8, st));
    if (U > 0)
        qf_entries_kernel<<<(unsigned)((U + 255) / 256), 256, 0, st>>>(ukeys, uwords, U, (const long long*)ix->blk_off, lo, hi, d_blk, d_word, d_rows);
    if (nsel > 0)
        qf_offsets_kernel<<<(unsigned)((nsel * (nl + 1) + 255) / 256), 256, 0, st>>>(ukeys, U, (const long long*)ix->blk_off, lo, nl,
                                                                                      ix->nblocks_local, nsel, d_off, (long long*)d_base);
    DPH_CUDA(cudaGetLastError());
    dph_query_filter* f = new dph_query_filter();
    f->h_base.assign(nsel + 1, 0);
    f->rows.assign(nsel, 0);
    DPH_CUDA(cudaMemcpyAsync(f->h_base.data(), d_base, (size_t)(nsel + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (nsel > 0) DPH_CUDA(cudaMemcpyAsync(f->rows.data(), d_rows, (size_t)nsel * 8, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        delete f;
        dph_set_error(std::string("make_query_filters: ") + cudaGetErrorString(e));
        return 1;
    }
    f->ix = ix; f->version = ix->layout_version; f->nsel = nsel; f->n = n; f->lo = lo; f->nl = nl;
    f->assign = d_assign; f->off = d_off; f->base = d_base; f->blk = d_blk; f->word = d_word; f->nblk = U;
    for (void* p : {(void*)d_assign, (void*)d_off, (void*)d_base, (void*)d_blk, (void*)d_word}) tmp.release(p);
    *out = f;
    return 0;
}

DPH_API void dph_query_filter_free(dph_query_filter* f) {
    if (!f) return;
    if (f->ix->qfilter == f) f->ix->qfilter = nullptr;
    cudaSetDevice(f->ix->device);
    for (void* p : {(void*)f->assign, (void*)f->off, (void*)f->base, (void*)f->blk, (void*)f->word}) cudaFree(p);
    delete f;
}
DPH_API int64_t dph_query_filter_bytes(const dph_query_filter* f) {
    return f->nblk * 8 + f->nsel * (f->nl + 1) * 4 + (f->nsel + 1) * 8 + f->n * 4;
}
DPH_API int64_t dph_query_filter_rows(const dph_query_filter* f, int64_t s) { return s >= 0 && s < f->nsel ? f->rows[s] : -1; }
DPH_API int64_t dph_query_filter_blocks(const dph_query_filter* f, int64_t s) {
    return s >= 0 && s < f->nsel ? f->h_base[s + 1] - f->h_base[s] : -1;
}
DPH_API int dph_query_filter_copy_selector(const dph_query_filter* f, int64_t s, uint32_t* off_out, uint32_t* blk_out, uint32_t* word_out) {
    DPH_CHECK(s >= 0 && s < f->nsel, "query filter: no such selector");
    DPH_CUDA(cudaSetDevice(f->ix->device));
    const int64_t b0 = f->h_base[s], nb = f->h_base[s + 1] - b0;
    DPH_CUDA(cudaMemcpy(off_out, f->off + s * (f->nl + 1), (size_t)(f->nl + 1) * 4, cudaMemcpyDeviceToHost));
    if (nb > 0) {
        DPH_CUDA(cudaMemcpy(blk_out, f->blk + b0, (size_t)nb * 4, cudaMemcpyDeviceToHost));
        DPH_CUDA(cudaMemcpy(word_out, f->word + b0, (size_t)nb * 4, cudaMemcpyDeviceToHost));
    }
    return 0;
}
DPH_API int dph_index_set_query_filter(dph_index* ix, const dph_query_filter* f) {
    DPH_CHECK(ix != nullptr, "null index");
    DPH_CHECK(f == nullptr || f->ix == ix,
              "set_query_filter: the query filter was built for another index; build it with this index's make_query_filters");
    ix->qfilter = f;
    if (f) ix->filter = nullptr;
    return 0;
}
