// filter.cu -- row masks for the filtered search (DESIGN.md 3.6, "Filtered search"): faiss' SearchParametersIVF(sel=IDSelector...)
// [3P].  A filter is one uint32 per 32-row code block of the shard, bit l = lane l's row is selected; the scan kernels (scan.cu, FILT
// variants) read it in the shard's own block numbering.  Building one reads the index and changes nothing.
#include "index_internal.cuh"

// One warp per code block, one lane per row: the row's label (explicit, or the sequential list_start[l] + j) against the selector --
// the sorted, de-duplicated label set sel [nsel] when `set`, else the range [rlo, rhi) -- inverted by `exclude`; padding rows are 0.
// Each CTA adds its selected rows to *rows.
__global__ void __launch_bounds__(256) filter_mask_kernel(uint32_t* __restrict__ mask, long long nblocks, const long long* blk_off,
                                                          const int* list_len, const long long* list_start, long long lo, long long hi,
                                                          const long long* ids, bool set, const long long* sel, long long nsel,
                                                          long long rlo, long long rhi, bool exclude, unsigned long long* rows) {
    __shared__ unsigned cta_rows;
    if (threadIdx.x == 0) cta_rows = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const long long blk = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (blk < nblocks) {                                   // warp-uniform
        const long long l = list_of_block(blk_off, lo, hi, blk);
        const long long j = (blk - blk_off[l]) * 32 + lane;
        const bool real = j < (long long)list_len[l];
        bool hit = false;
        if (real) {
            const long long label = ids ? ids[blk * 32 + lane] : list_start[l] + j;
            if (set) { const long long i = lower_bound_ll(sel, nsel, label); hit = i < nsel && sel[i] == label; }
            else hit = label >= rlo && label < rhi;
        }
        const unsigned w = __ballot_sync(0xffffffffu, real && hit != exclude);
        if (lane == 0) { mask[blk] = w; atomicAdd(&cta_rows, (unsigned)__popc(w)); }
    }
    __syncthreads();
    if (threadIdx.x == 0 && cta_rows) atomicAdd(rows, (unsigned long long)cta_rows);
}

DPH_API int dph_filter_create(dph_filter** out, dph_index* ix, const int64_t* ids, int64_t n_ids, int64_t range_lo, int64_t range_hi,
                              int exclude, int mem) {
    DPH_CHECK(out != nullptr, "make_filter: null out");
    *out = nullptr;
    DPH_CHECK(ix && ix->list_len, "make_filter: lists are not set");
    DPH_CHECK(n_ids >= 0, "make_filter: n_ids must be >= 0");
    DPH_CHECK(!(ids && (range_lo != 0 || range_hi != 0)), "make_filter: give a label set or a label range, not both");
    DPH_CHECK(ids || n_ids == 0, "make_filter: n_ids > 0 without labels");
    DPH_CUDA(cudaSetDevice(ix->device));
    cudaStream_t st = ix->stream;
    const char* oom = "make_filter: not enough device memory for the mask";
    DevTmp tmp;
    const int64_t nb = ix->nblocks_local;
    uint32_t* mask;
    unsigned long long* rows;
    DPH_TRY(tmp.alloc(&mask, nb, oom));
    DPH_TRY(tmp.alloc(&rows, 1, oom));
    long long* sel = nullptr;
    int64_t nsel = 0;
    if (ids && n_ids > 0) DPH_TRY(dph_label_set(tmp, ids, n_ids, mem, st, &sel, &nsel, "make_filter"));
    DPH_CUDA(cudaMemsetAsync(rows, 0, 8, st));
    if (nb > 0)
        filter_mask_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, st>>>(mask, nb, (const long long*)ix->blk_off, ix->list_len,
                                                                    (const long long*)ix->list_start, ix->list_lo, ix->list_hi,
                                                                    (const long long*)ix->ids, ids != nullptr, sel, nsel, range_lo, range_hi,
                                                                    exclude != 0, rows);
    DPH_CUDA(cudaGetLastError());
    unsigned long long h_rows = 0;
    DPH_CUDA(cudaMemcpyAsync(&h_rows, rows, 8, cudaMemcpyDeviceToHost, st));
    DPH_CUDA(cudaStreamSynchronize(st));
    dph_filter* f = new dph_filter();
    f->ix = ix; f->version = ix->layout_version; f->mask = mask; f->nwords = nb; f->rows = (int64_t)h_rows;
    tmp.release(mask);
    *out = f;
    return 0;
}

DPH_API void dph_filter_free(dph_filter* f) {
    if (!f) return;
    if (f->ix->filter == f) f->ix->filter = nullptr;
    cudaSetDevice(f->ix->device);
    cudaFree(f->mask);
    delete f;
}
DPH_API int64_t dph_filter_rows(const dph_filter* f) { return f->rows; }
DPH_API int64_t dph_filter_bytes(const dph_filter* f) { return f->nwords * 4; }
DPH_API int dph_filter_copy_mask(const dph_filter* f, uint32_t* out_host) {
    DPH_CUDA(cudaSetDevice(f->ix->device));
    if (f->nwords > 0) DPH_CUDA(cudaMemcpy(out_host, f->mask, (size_t)f->nwords * 4, cudaMemcpyDeviceToHost));
    return 0;
}
DPH_API int dph_index_set_filter(dph_index* ix, const dph_filter* f) {
    DPH_CHECK(ix != nullptr, "null index");
    DPH_CHECK(f == nullptr || f->ix == ix, "set_filter: the filter was built for another index; build it with this index's make_filter");
    ix->filter = f;
    if (f) ix->qfilter = nullptr;         // one active filter per handle
    return 0;
}
