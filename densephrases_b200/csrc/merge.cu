// merge.cu -- dph_index_merge_from (DESIGN.md 3.4, "Merging indexes"): faiss InvertedLists::merge_from as the merge stage of
// build_phrase_index.py:282-338 uses it.  For every list l the result holds this index's rows, then source 1's rows of l, then
// source 2's, ..., each in its stored order; a source row's label is its stored label + add_id.  The sources are not modified.
// One pass over the shard: every old block moves once, whole (relayout_codes/ids_kernel, as in the add); one warp per source block
// copies that source's rows into place, re-rotated for their new lane; the direct maps, each sorted by label, are merged, not
// re-sorted.  The result is byte-identical to set_lists of the concatenated list-major arrays.
#include "index_internal.cuh"
#include <limits.h>
#include <thrust/execution_policy.h>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <thrust/merge.h>

// flag = 1 if the two tables differ in any bit
__global__ void tables_differ_kernel(const uint32_t* a, const uint32_t* b, long long n, int* flag) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        if (a[i] != b[i]) { *flag = 1; return; }
}

// One warp per block of a source's shard, lane = the row's lane there.  Row j of list l lands at j + base[l - lo] of the same list in
// the new layout (base = this index's old length of l plus the earlier sources' lengths of l), re-rotated for its new lane; its label
// is the stored one (sequential: list_start_src[l] + j) plus add_id.  A source with sequential labels also writes each row's
// direct-map pair at the row's local position, which is label order; an explicit-label source's pairs come from its own map.  Codes
// go to the rows whose new block is in [w0, w1), block w0 at codes_new (the whole layout: 0, LLONG_MAX; a host index's staged chunk:
// its blocks); labels and direct-map pairs only when ids_new is set.
__global__ void __launch_bounds__(256) merge_rows_kernel(long long nb_src, const long long* boff_src, const int* len_src, const uint8_t* codes_src,
                                                         const long long* ids_src, const long long* list_start_src, const long long* lrs_src,
                                                         long long lo, long long hi, const long long* base, const long long* boff_new,
                                                         long long add_id, uint8_t* codes_new, long long w0, long long w1, long long* ids_new,
                                                         long long* dm_ids, long long* dm_rows) {
    const long long b = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (b >= nb_src) return;
    const long long l = list_of_block(boff_src, lo, hi, b);
    const long long j = (b - boff_src[l]) * 32 + lane;
    if (j >= (long long)len_src[l]) return;
    const long long prow = boff_new[l] * 32 + base[l - lo] + j;          // the new list's blocks are consecutive
    if ((prow >> 5) >= w0 && (prow >> 5) < w1) {
        unsigned char row[DPH_CODE];
        dph_load_row(codes_src, b, lane, row);
        dph_store_row(codes_new, (prow >> 5) - w0, (int)(prow & 31), row);
    }
    if (!ids_new) return;
    const long long id = (ids_src ? ids_src[b * 32 + lane] : list_start_src[l] + j) + add_id;
    ids_new[prow] = id;
    if (!ids_src) {
        dm_ids[lrs_src[l - lo] + j] = id;
        dm_rows[lrs_src[l - lo] + j] = prow;
    }
}
// An explicit-label source's direct map -> (label + add_id, padded row in the new layout), in its own (label) order.
__global__ void merge_dm_remap_kernel(const long long* dm_ids_src, const long long* dm_rows_src, long long n, const long long* boff_src,
                                      long long lo, long long hi, const long long* base, const long long* boff_new, long long add_id,
                                      long long* dm_ids, long long* dm_rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long prow = dm_rows_src[i], b = prow >> 5;
    const long long l = list_of_block(boff_src, lo, hi, b);
    dm_ids[i] = dm_ids_src[i] + add_id;
    dm_rows[i] = boff_new[l] * 32 + base[l - lo] + (b - boff_src[l]) * 32 + (prow & 31);
}

// This index's direct-map pairs, read in place through iterators (its old arrays stay untouched until the commit):
// explicit labels: the old padded row -> the same (list, j) in the new layout (remap_dm_kernel's rule)
struct RemapRow {
    const long long *boff_old, *boff_new;
    long long lo, hi;
    __device__ long long operator()(long long prow) const {
        const long long ob = prow >> 5, l = list_of_block(boff_old, lo, hi, ob);
        return ((boff_new[l] + ob - boff_old[l]) << 5) | (prow & 31);
    }
};
// sequential labels: local row i carries label list_start[lo] + i; its padded row in the new layout
struct LocalRow {
    const long long *lrs, *boff_new;     // lrs [hi - lo]: local row of each shard list's first vector
    long long lo, ns;
    __device__ long long operator()(long long i) const {
        const long long l = list_of_block(lrs, 0, ns, i) + lo;      // last list starting at or before i: the non-empty one holding it
        return boff_new[l] * 32 + (i - lrs[l - lo]);
    }
};

// Stable merge: on equal labels the pairs of (ka, va) come first.
template <class K, class V>
static void merge_pairs(cudaStream_t st, K ka, V va, int64_t na, const long long* kb, const long long* vb, int64_t nb, long long* ko, long long* vo) {
    thrust::merge_by_key(thrust::cuda::par.on(st), ka, ka + na, kb, kb + nb, va, vb, ko, vo);
}

static bool label_ok(int64_t v, int64_t add_id) {
    int64_t r;
    return !__builtin_add_overflow(v, add_id, &r) && r >= 0;
}

DPH_API int dph_index_merge_from(dph_index* ix, const dph_index* const* src, int n_src, int64_t add_id) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CHECK(n_src >= 0 && (src != nullptr || n_src == 0), "merge_from: bad source list; the index is unchanged");
    if (!ix->host_mutable)          // a host index without a reserved capacity (reserve_host_codes) stays read-only
        DPH_CHECK(!ix->on_host, "merge_from: the codes of this index are in host memory, which is read-only after set_lists; the index is unchanged");
    DPH_CUDA(cudaSetDevice(ix->device));
    for (float& a : ix->merge_ms) a = 0.f;
    cudaStream_t st = ix->stream;
    const bool prof = ix->profile && ix->aev[0];
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[0], st));
    const int64_t nlist = ix->nlist, lo = ix->list_lo, hi = ix->list_hi, ns = hi - lo;

    // 1. compatibility and labels, before anything changes
    int64_t src_total = 0, src_local = 0;
    for (int s = 0; s < n_src; s++) {
        const dph_index* o = src[s];
        DPH_CHECK(o != nullptr, "merge_from: a source is null; the index is unchanged");
        DPH_CHECK(o != ix, "merge_from: the index cannot be its own source; the index is unchanged");
        DPH_CHECK(!o->on_host, "merge_from: a source keeps its codes in host memory, which a merge does not read; the index is unchanged");
        DPH_CHECK(o->A && o->C && o->pq && o->list_len, "merge_from: a source is not fully constructed (opq/centroids/pq/lists); the index is unchanged");
        DPH_CHECK(o->d == ix->d && o->M == ix->M && o->nlist == nlist && o->device == ix->device,
                  "merge_from: a source has another d, nlist, M or device; the index is unchanged");
        DPH_CHECK(o->list_lo == lo && o->list_hi == hi, "merge_from: a source holds another shard range; the index is unchanged");
        src_total += o->ntotal; src_local += o->ntotal_local;
    }
    DevTmp tmp;
    const char* oom = "merge_from: not enough device memory for the old and the new code, label and direct-map buffers of the shard at once; "
                      "the index is unchanged";
    if (n_src > 0) {
        int* flag;
        DPH_TRY(tmp.alloc(&flag, 1, oom));
        DPH_CUDA(cudaMemsetAsync(flag, 0, 4, st));
        for (int s = 0; s < n_src; s++) {
            const dph_index* o = src[s];
            DPH_CUDA(cudaStreamSynchronize(o->stream));          // the source's own pending work
            const float* tabs[3][2] = {{ix->A, o->A}, {ix->C, o->C}, {ix->pq, o->pq}};
            const long long cnt[3] = {(long long)ix->d * ix->d, (long long)nlist * ix->d, (long long)DPH_M * 256 * DPH_DSUB};
            for (int t = 0; t < 3; t++)
                tables_differ_kernel<<<264, 256, 0, st>>>((const uint32_t*)tabs[t][0], (const uint32_t*)tabs[t][1], cnt[t], flag);
        }
        DPH_CUDA(cudaGetLastError());
        int h_flag = 0;
        DPH_CUDA(cudaMemcpyAsync(&h_flag, flag, 4, cudaMemcpyDeviceToHost, st));
        DPH_CUDA(cudaStreamSynchronize(st));
        DPH_CHECK(h_flag == 0, "merge_from: a source has another OPQ matrix, other centroids or other PQ codebooks; the index is unchanged");
    }
    for (int s = 0; s < n_src; s++) {
        const dph_index* o = src[s];
        if (o->ntotal_local == 0) continue;
        int64_t mn, mx;                                          // the smallest and largest label of the source's rows in this shard
        if (o->ids) {
            DPH_CHECK(o->dm_n > 0, "merge_from: a source's direct map is empty; the index is unchanged");
            DPH_CUDA(cudaMemcpy(&mn, o->dm_ids, 8, cudaMemcpyDeviceToHost));
            DPH_CUDA(cudaMemcpy(&mx, o->dm_ids + o->dm_n - 1, 8, cudaMemcpyDeviceToHost));
        } else {
            mn = o->lay.start[lo]; mx = mn + o->ntotal_local - 1;
        }
        DPH_CHECK(label_ok(mn, add_id) && label_ok(mx, add_id),
                  "merge_from: a label + add_id would be negative or overflow int64; the index is unchanged");
    }
    if (src_total == 0) return 0;                                // nothing to merge: not even the labels change

    // 2. the new layout: per list, this index's rows, then each source's
    const DphLayout& old = ix->lay;
    std::vector<int64_t> len_new(old.len.begin(), old.len.end()), base((size_t)n_src * std::max<int64_t>(ns, 1), 0);
    for (int s = 0; s < n_src; s++)
        for (int64_t l = 0; l < nlist; l++) {
            if (l >= lo && l < hi) base[(size_t)s * std::max<int64_t>(ns, 1) + (l - lo)] = len_new[l];
            len_new[l] += src[s]->lay.len[l];
        }
    DphLayout L;
    DPH_TRY(L.build(ix, len_new.data(), "merge_from: a list would exceed 2^31 - 1 rows; the index is unchanged"));
    DPH_TRY(dph_host_capacity_check(ix, L, "merge_from"));
    const int64_t nb = L.nblocks, nsb = std::max<int64_t>(ns, 1);
    const bool was_explicit = ix->ids != nullptr;
    const int64_t dm_dest = was_explicit ? ix->dm_n : ix->ntotal_local, dm_n = dm_dest + src_local;

    // 3. every buffer before anything changes: a failed allocation leaves the index as it was.  A host index re-lays its code array in
    //    place (host_move.cu) through two staging buffers instead of a new code buffer.
    uint8_t* codes_new = nullptr;
    int64_t *ids_new, *dm_ids_new, *dm_rows_new, *d_boff_new, *d_base, *d_lrs, *xk, *xv, *yk = nullptr, *yv = nullptr, *zk = nullptr, *zv = nullptr;
    DphHostMover mover;
    const int64_t d_first = ix->on_host ? dph_first_changed_block(old, L) : 0;
    if (ix->on_host) DPH_TRY(mover.prepare(ix, tmp, nb - d_first, oom));
    else DPH_TRY(tmp.alloc(&codes_new, (size_t)nb * DPH_BLK_BYTES, oom));
    DPH_TRY(tmp.alloc(&ids_new, (size_t)nb * 32, oom));
    DPH_TRY(tmp.alloc(&dm_ids_new, dm_n, oom)); DPH_TRY(tmp.alloc(&dm_rows_new, dm_n, oom));
    DPH_TRY(tmp.alloc(&d_boff_new, nlist, oom)); DPH_TRY(tmp.alloc(&d_base, base.size(), oom));
    DPH_TRY(tmp.alloc(&d_lrs, (size_t)(n_src + 1) * nsb, oom));        // [0]: this index's local row starts, [1 + s]: source s's
    DPH_TRY(tmp.alloc(&xk, src_local, oom)); DPH_TRY(tmp.alloc(&xv, src_local, oom));       // the sources' pairs, one run per source
    if (n_src > 1) { DPH_TRY(tmp.alloc(&yk, src_local, oom)); DPH_TRY(tmp.alloc(&yv, src_local, oom)); }    // ping-pong of their merge
    if (n_src > 2) { DPH_TRY(tmp.alloc(&zk, src_local, oom)); DPH_TRY(tmp.alloc(&zv, src_local, oom)); }
    DPH_CUDA(cudaMemcpyAsync(d_boff_new, L.blk_off.data(), nlist * 8, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemcpyAsync(d_base, base.data(), base.size() * 8, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemcpyAsync(d_lrs, old.row_start.data(), old.row_start.size() * 8, cudaMemcpyHostToDevice, st));
    for (int s = 0; s < n_src; s++)
        DPH_CUDA(cudaMemcpyAsync(d_lrs + (size_t)(s + 1) * nsb, src[s]->lay.row_start.data(), src[s]->lay.row_start.size() * 8,
                                 cudaMemcpyHostToDevice, st));
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[1], st));

    // 4. this index's blocks move whole (zeros and label -1 past each list's old end)
    const long long *bo_new = (const long long*)d_boff_new, *bo_old = (const long long*)ix->blk_off;
    if (nb > 0) {
        if (!ix->on_host) relayout_codes_kernel<<<(unsigned)nb, 192, 0, st>>>(codes_new, 0, bo_new, bo_old, ix->list_len, lo, hi, ix->codes);
        relayout_ids_kernel<<<(unsigned)nb, 32, 0, st>>>((long long*)ids_new, 0, bo_new, bo_old, ix->list_len, lo, hi, (const long long*)ix->ids,
                                                       (const long long*)ix->list_start, nullptr, nullptr, nullptr);
    }
    DPH_CUDA(cudaGetLastError());
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[2], st));

    // 5. each source's rows into place, behind this index's and the earlier sources' rows of the same list
    std::vector<int64_t> xoff(n_src + 1, 0);
    for (int s = 0; s < n_src; s++) {
        const dph_index* o = src[s];
        xoff[s + 1] = xoff[s] + o->ntotal_local;
        if (o->nblocks_local == 0) continue;
        merge_rows_kernel<<<(unsigned)((o->nblocks_local * 32 + 255) / 256), 256, 0, st>>>(
            o->nblocks_local, (const long long*)o->blk_off, o->list_len, o->codes, (const long long*)o->ids, (const long long*)o->list_start,
            (const long long*)(d_lrs + (size_t)(s + 1) * nsb), lo, hi, (const long long*)(d_base + (size_t)s * nsb), bo_new, add_id, codes_new,
            0, ix->on_host ? 0 : LLONG_MAX, (long long*)ids_new, (long long*)(xk + xoff[s]), (long long*)(xv + xoff[s]));
    }
    DPH_CUDA(cudaGetLastError());
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[3], st));

    // 6. direct map: the sources' sorted runs merged in argument order, then merged behind this index's pairs (stable: on a label
    //    present twice the later input comes later, and locate_label takes the last entry)
    for (int s = 0; s < n_src; s++) {
        const dph_index* o = src[s];
        if (o->ids && o->dm_n > 0)
            merge_dm_remap_kernel<<<(unsigned)((o->dm_n + 255) / 256), 256, 0, st>>>(
                (const long long*)o->dm_ids, (const long long*)o->dm_rows, o->dm_n, (const long long*)o->blk_off, lo, hi,
                (const long long*)(d_base + (size_t)s * nsb), bo_new, add_id, (long long*)(xk + xoff[s]), (long long*)(xv + xoff[s]));
    }
    DPH_CUDA(cudaGetLastError());
    try {
        const long long *bk = (const long long*)xk, *bv = (const long long*)xv;
        for (int s = 1; s < n_src; s++) {
            long long* ok = (long long*)(s & 1 ? yk : zk);
            long long* ov = (long long*)(s & 1 ? yv : zv);
            merge_pairs(st, bk, bv, xoff[s], (const long long*)(xk + xoff[s]), (const long long*)(xv + xoff[s]), xoff[s + 1] - xoff[s], ok, ov);
            bk = ok; bv = ov;
        }
        if (was_explicit)
            merge_pairs(st, (const long long*)ix->dm_ids,
                        thrust::make_transform_iterator((const long long*)ix->dm_rows, RemapRow{bo_old, bo_new, lo, hi}), dm_dest, bk, bv,
                        src_local, (long long*)dm_ids_new, (long long*)dm_rows_new);
        else
            merge_pairs(st, thrust::make_counting_iterator<long long>(old.start[lo]),
                        thrust::make_transform_iterator(thrust::make_counting_iterator<long long>(0),
                                                        LocalRow{(const long long*)d_lrs, bo_new, lo, ns}),
                        dm_dest, bk, bv, src_local, (long long*)dm_ids_new, (long long*)dm_rows_new);
    } catch (const std::exception& e) {
        cudaGetLastError();
        dph_set_error(std::string("merge_from: device merge failed; the index is unchanged: ") + e.what());
        return 1;
    }
    DPH_CUDA(cudaGetLastError());
    // 7. a host index: the old blocks move up in place, each staged chunk receiving every source's rows that land in it.  Last, after
    //    the device merge that may still fail with the index unchanged (its time is in the direct-map stage and in last_host_move).
    if (ix->on_host)
        DPH_TRY(mover.run(ix, L, d_first, bo_new, true, [&](uint8_t* buf, int64_t c0, int64_t c1, cudaStream_t rs) {
            for (int s = 0; s < n_src; s++) {
                const dph_index* o = src[s];
                if (o->nblocks_local == 0) continue;
                merge_rows_kernel<<<(unsigned)((o->nblocks_local * 32 + 255) / 256), 256, 0, rs>>>(
                    o->nblocks_local, (const long long*)o->blk_off, o->list_len, o->codes, (const long long*)o->ids, (const long long*)o->list_start,
                    (const long long*)(d_lrs + (size_t)(s + 1) * nsb), lo, hi, (const long long*)(d_base + (size_t)s * nsb), bo_new, add_id, buf,
                    c0, c1, nullptr, nullptr, nullptr);
            }
            DPH_CUDA(cudaGetLastError());
            return 0;
        }));
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[4], st));
    DPH_CUDA(cudaStreamSynchronize(st));

    // 8. commit: the layout, then the buffers (a host index keeps its code array)
    const bool shard_changed = dph_shard_changed(ix, L);
    DPH_TRY(dph_commit_layout(ix, std::move(L)));
    void* olds[] = {ix->on_host ? nullptr : ix->codes, ix->ids, ix->dm_ids, ix->dm_rows};
    for (void* p : olds) if (p) cudaFree(p);
    if (!ix->on_host) ix->codes = codes_new;
    ix->ids = ids_new; ix->dm_ids = dm_ids_new; ix->dm_rows = dm_rows_new;
    for (void* p : {(void*)codes_new, (void*)ids_new, (void*)dm_ids_new, (void*)dm_rows_new}) tmp.release(p);
    ix->dm_n = ix->dm_cap = dm_n; ix->blk_cap = nb;
    if (ix->on_host) DPH_TRY(dph_host_after_mutation(ix, shard_changed));
    if (prof)
        for (int s = 0; s < 4; s++) DPH_CUDA(cudaEventElapsedTime(&ix->merge_ms[s], ix->aev[s], ix->aev[s + 1]));
    return 0;
}

DPH_API int dph_index_last_merge_ms(const dph_index* ix, float* ms_out) {
    DPH_CHECK(ix->aev[0] != nullptr, "profiling was never enabled");
    std::copy(ix->merge_ms, ix->merge_ms + 4, ms_out);
    return 0;
}
