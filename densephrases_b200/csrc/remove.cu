// remove.cu -- dph_index_remove_ids and dph_index_sync_list_len (DESIGN.md 3.2, "Removing vectors").
// The survivors of every list, and their order, are those of faiss 1.6.x IndexIVF::remove_ids (DirectMap::NoMap branch) [3P]:
//     j = 0, l = len;  while (j < l) { if (selected(j)) { l--; row[j] = row[l]; } else j++; }
// In closed form, with S the selected positions and L' = len - |S|: kept rows below L' stay where they are, and the h-th hole below
// L' (ascending) receives the h-th kept row at or above L', counted from the end of the list.  Sources are >= L' and destinations
// < L', so the moves are disjoint and run all at once.  The shard then compacts in place: blocks move down (dst <= src) through a
// bounded staging buffer, and the direct map is compacted the same way; the code allocation is not shrunk.
#include "index_internal.cuh"
#include <limits.h>
#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/scan.h>
#include <thrust/sequence.h>
#include <thrust/sort.h>
#include <thrust/unique.h>

__device__ __forceinline__ long long lower_bound_ll(const long long* a, long long n, long long key) {      // first i with a[i] >= key
    long long lo = 0, hi = n;
    while (lo < hi) { const long long mid = (lo + hi) >> 1; if (a[mid] < key) lo = mid + 1; else hi = mid; }
    return lo;
}
__device__ __forceinline__ long long upper_bound_ll(const long long* a, long long n, long long key) {      // first i with a[i] > key
    long long lo = 0, hi = n;
    while (lo < hi) { const long long mid = (lo + hi) >> 1; if (a[mid] <= key) lo = mid + 1; else hi = mid; }
    return lo;
}

// ---- 1. mark: the direct map is sorted by label, so a label's rows are one run of it ----
// label set (sorted, unique): run [first, first + cnt) of every selected label; a label that is absent (or negative) has cnt 0
__global__ void rm_find_kernel(const long long* sel, long long n, const long long* dm_ids, long long dm_n, long long* first, long long* cnt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long a = lower_bound_ll(dm_ids, dm_n, sel[i]);
    first[i] = a;
    cnt[i] = upper_bound_ll(dm_ids, dm_n, sel[i]) - a;
}
// label range [lo, hi): one run of the direct map
__global__ void rm_range_kernel(const long long* dm_ids, long long dm_n, long long lo, long long hi, long long* out) {
    out[0] = lower_bound_ll(dm_ids, dm_n, lo);
    out[1] = lower_bound_ll(dm_ids, dm_n, hi);
}
__global__ void rm_expand_kernel(const long long* first, const long long* cnt, const long long* off, long long n, long long* rm_dm) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (long long t = 0; t < cnt[i]; t++) rm_dm[off[i] + t] = first[i] + t;
}
// removed direct-map pair k -> its padded row, and the per-list count (rm_dm null: the pairs are the run [p0, p0 + R))
__global__ void rm_rows_kernel(const long long* rm_dm, long long p0, long long R, const long long* dm_rows, const long long* boff, long long lo,
                               long long hi, long long* rm_prow, int* cnt) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= R) return;
    const long long prow = dm_rows[rm_dm ? rm_dm[k] : p0 + k];
    rm_prow[k] = prow;
    atomicAdd(&cnt[list_of_block(boff, lo, hi, prow >> 5)], 1);
}

// ---- 2. plan the hole fills (writes nothing of the index).  rm_prow is sorted, so list l's removed rows are rm_prow[rm_off[l] ..)
// ascending and its holes (j < L') come first: hole q takes the q-th kept row at or above L' from the end, i.e. the largest p in
// [L', len) with kept(p) = (len - p) - #{removed >= p} >= q + 1.  (mv_src, mv_dst) = (source, destination) padded rows; LLONG_MAX: none.
__global__ void rm_plan_moves_kernel(const long long* rm_prow, long long R, const long long* boff, const int* len_old, const int* cnt,
                                     const long long* rm_off, long long lo, long long hi, long long* mv_src, long long* mv_dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R) return;
    const long long prow = rm_prow[i];
    const long long l = list_of_block(boff, lo, hi, prow >> 5);
    const long long base = boff[l] * 32, r = cnt[l], len = len_old[l], Lp = len - r;
    mv_src[i] = LLONG_MAX; mv_dst[i] = -1;
    if (prow - base >= Lp) return;
    const long long q = i - rm_off[l];
    const long long* s = rm_prow + rm_off[l];
    long long a = Lp, b = len;                                  // kept(a) >= q + 1 > kept(b)
    while (b - a > 1) {
        const long long mid = (a + b) >> 1;
        const long long kept = (len - mid) - (r - lower_bound_ll(s, r, base + mid));
        if (kept >= q + 1) a = mid; else b = mid;
    }
    mv_src[i] = base + a; mv_dst[i] = prow;
}
// ---- 3. fill the holes (old layout): sources are >= L' and destinations < L', so the moves are disjoint and run all at once
__global__ void rm_fill_holes_kernel(const long long* mv_src, const long long* mv_dst, long long R, uint8_t* codes, long long* ids) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R || mv_src[i] == LLONG_MAX) return;
    const long long src = mv_src[i], dst = mv_dst[i];
    unsigned char row[DPH_CODE];
    dph_load_row(codes, src >> 5, (int)(src & 31), row);
    dph_store_row(codes, dst >> 5, (int)(dst & 31), row);       // re-rotated for the destination lane
    ids[dst] = ids[src];
}
// rows [L', end of L''s block) of every touched list become padding: zero codes, label -1 (what fill_ids_kernel writes)
__global__ void rm_clear_tail_kernel(const long long* boff, const int* len_old, const int* cnt, long long lo, uint8_t* codes, long long* ids) {
    const long long l = lo + blockIdx.x;
    const long long r = cnt[l];
    if (r == 0) return;
    const long long len = len_old[l], Lp = len - r, j = Lp + threadIdx.x;
    if (j >= ((Lp + 31) & ~31ll) || j >= len) return;
    const long long prow = boff[l] * 32 + j;
#pragma unroll
    for (int c = 0; c < 6; c++) *reinterpret_cast<uint4*>(codes + (prow >> 5) * DPH_BLK_BYTES + c * 512 + (prow & 31) * 16) = make_uint4(0, 0, 0, 0);
    ids[prow] = -1;
}

// ---- 5. direct map: destination entries [d0, d0 + n) gathered from the surviving pair that lands there (src >= dst), its row remapped
// through the hole fills (mv_src sorted, LLONG_MAX padding) and the block shift.  Stays sorted by label, repeated labels in order.
__global__ void rm_dm_gather_kernel(long long d0, long long n, const long long* rm_dm, long long p0, long long R, const long long* dm_ids,
                                    const long long* dm_rows, const long long* mv_src, const long long* mv_dst, const long long* boff_old,
                                    const long long* boff_new, long long lo, long long hi, long long* out_ids, long long* out_rows) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const long long d = d0 + k;
    long long src;
    if (rm_dm) {            // src = d + #{removed pairs before it} = d + #{j : rm_dm[j] - j <= d}
        long long a = 0, b = R;
        while (a < b) { const long long mid = (a + b) >> 1; if (rm_dm[mid] - mid <= d) a = mid + 1; else b = mid; }
        src = d + a;
    } else src = d < p0 ? d : d + R;
    long long row = dm_rows[src];
    const long long t = lower_bound_ll(mv_src, R, row);
    if (t < R && mv_src[t] == row) row = mv_dst[t];
    const long long ob = row >> 5, l = list_of_block(boff_old, lo, hi, ob);
    out_ids[k] = dm_ids[src];
    out_rows[k] = ((boff_new[l] + ob - boff_old[l]) << 5) | (row & 31);
}

DPH_API int dph_index_remove_ids(dph_index* ix, const int64_t* ids, int64_t n_ids, int64_t range_lo, int64_t range_hi, int mem,
                                 int64_t* n_removed_out, int64_t* removed_per_list_out) {
    DPH_CHECK(ix && ix->list_len, "remove_ids: lists are not set");
    DPH_CHECK(n_ids >= 0, "remove_ids: n_ids must be >= 0; the index is unchanged");
    DPH_CHECK(!(ids && (range_lo != 0 || range_hi != 0)), "remove_ids: give a label set or a label range, not both; the index is unchanged");
    DPH_CHECK(ids || n_ids == 0, "remove_ids: n_ids > 0 without labels; the index is unchanged");
    DPH_CUDA(cudaSetDevice(ix->device));
    const int64_t nlist = ix->nlist, lo = ix->list_lo, hi = ix->list_hi;
    if (n_removed_out) *n_removed_out = 0;
    if (removed_per_list_out) std::fill(removed_per_list_out, removed_per_list_out + nlist, (int64_t)0);
    for (float& a : ix->remove_ms) a = 0.f;
    ix->remove_tmp_peak = 0;
    if (ids ? n_ids == 0 : range_lo >= range_hi) return 0;          // empty selector: nothing changes, not even the labels
    cudaStream_t st = ix->stream;
    const char* oom = "remove_ids: not enough device memory for the temporary buffers; the index is unchanged";
    const bool prof = ix->profile && ix->aev[0];
    DevTmp tmp, conv;          // conv: the label and direct-map arrays an implicit-label index gains (part of the index once committed)
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[0], st));

    // 0. implicit labels become explicit (list_start[l] + j), exactly as the first add does, into new arrays
    const DphLayout& old = ix->lay;
    const int64_t nb = ix->nblocks_local;
    const long long* bo = (const long long*)ix->blk_off;
    long long *w_ids = (long long*)ix->ids, *w_dm_ids = (long long*)ix->dm_ids, *w_dm_rows = (long long*)ix->dm_rows;
    int64_t dm_n = ix->dm_n;
    const bool was_implicit = ix->ids == nullptr;
    if (was_implicit) {
        const char* oom0 = "remove_ids: not enough device memory for the labels and direct map of an index with sequential labels; the index is unchanged";
        int64_t* d_lrs;
        DPH_TRY(conv.alloc(&w_ids, (size_t)nb * 32, oom0)); DPH_TRY(conv.alloc(&w_dm_ids, ix->ntotal_local, oom0));
        DPH_TRY(conv.alloc(&w_dm_rows, ix->ntotal_local, oom0)); DPH_TRY(tmp.alloc(&d_lrs, old.row_start.size(), oom));
        DPH_CUDA(cudaMemcpyAsync(d_lrs, old.row_start.data(), old.row_start.size() * 8, cudaMemcpyHostToDevice, st));
        if (nb > 0)
            relayout_ids_kernel<<<(unsigned)nb, 32, 0, st>>>(w_ids, 0, bo, bo, ix->list_len, lo, hi, nullptr, (const long long*)ix->list_start,
                                                           (const long long*)d_lrs, w_dm_ids, w_dm_rows);
        DPH_CUDA(cudaGetLastError());
        dm_n = ix->ntotal_local;
    }

    // 1. mark: the removed direct-map pairs (a sorted list of positions, or one run) and their padded rows
    long long* rm_dm = nullptr;
    int64_t p0 = 0, R = 0;
    try {
        if (ids) {
            long long *sel, *first, *cnt, *off;
            DPH_TRY(tmp.alloc(&sel, n_ids, oom));
            DPH_CUDA(cudaMemcpyAsync(sel, ids, (size_t)n_ids * 8, mem == DPH_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, st));
            thrust::device_ptr<long long> sp(sel);
            thrust::sort(thrust::cuda::par.on(st), sp, sp + n_ids);
            const int64_t nu = thrust::unique(thrust::cuda::par.on(st), sp, sp + n_ids) - sp;
            DPH_TRY(tmp.alloc(&first, nu, oom)); DPH_TRY(tmp.alloc(&cnt, nu, oom)); DPH_TRY(tmp.alloc(&off, nu, oom));
            rm_find_kernel<<<(unsigned)((nu + 255) / 256), 256, 0, st>>>(sel, nu, w_dm_ids, dm_n, first, cnt);
            DPH_CUDA(cudaGetLastError());
            thrust::device_ptr<long long> cp(cnt), op(off);
            thrust::exclusive_scan(thrust::cuda::par.on(st), cp, cp + nu, op);
            int64_t last[2];
            DPH_CUDA(cudaMemcpyAsync(&last[0], off + nu - 1, 8, cudaMemcpyDeviceToHost, st));
            DPH_CUDA(cudaMemcpyAsync(&last[1], cnt + nu - 1, 8, cudaMemcpyDeviceToHost, st));
            DPH_CUDA(cudaStreamSynchronize(st));
            R = last[0] + last[1];
            if (R > 0) {
                DPH_TRY(tmp.alloc(&rm_dm, R, oom));
                rm_expand_kernel<<<(unsigned)((nu + 255) / 256), 256, 0, st>>>(first, cnt, off, nu, rm_dm);
            }
        } else {
            long long* run;
            DPH_TRY(tmp.alloc(&run, 2, oom));
            rm_range_kernel<<<1, 1, 0, st>>>(w_dm_ids, dm_n, range_lo, range_hi, run);
            int64_t h_run[2];
            DPH_CUDA(cudaMemcpyAsync(h_run, run, 16, cudaMemcpyDeviceToHost, st));
            DPH_CUDA(cudaStreamSynchronize(st));
            p0 = h_run[0]; R = h_run[1] - h_run[0];
        }
    } catch (const std::exception& e) {
        cudaGetLastError();
        dph_set_error(std::string("remove_ids: device sort failed; the index is unchanged: ") + e.what());
        return 1;
    }
    DPH_CUDA(cudaGetLastError());

    std::vector<int32_t> h_cnt(nlist, 0);
    long long *rm_prow = nullptr, *mv_src = nullptr, *mv_dst = nullptr, *d_boff_new = nullptr, *d_rm_off = nullptr;
    int* d_cnt = nullptr;
    if (R > 0) {
        DPH_TRY(tmp.alloc(&rm_prow, R, oom)); DPH_TRY(tmp.alloc(&mv_src, R, oom)); DPH_TRY(tmp.alloc(&mv_dst, R, oom));
        DPH_TRY(tmp.alloc(&d_cnt, nlist, oom)); DPH_TRY(tmp.alloc(&d_boff_new, nlist, oom)); DPH_TRY(tmp.alloc(&d_rm_off, nlist, oom));
        DPH_CUDA(cudaMemsetAsync(d_cnt, 0, nlist * 4, st));
        rm_rows_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(rm_dm, p0, R, w_dm_rows, bo, lo, hi, rm_prow, d_cnt);
        DPH_CUDA(cudaGetLastError());
        try {
            thrust::device_ptr<long long> rp(rm_prow);
            thrust::sort(thrust::cuda::par.on(st), rp, rp + R);
        } catch (const std::exception& e) {
            cudaGetLastError();
            dph_set_error(std::string("remove_ids: device sort failed; the index is unchanged: ") + e.what());
            return 1;
        }
        DPH_CUDA(cudaMemcpyAsync(h_cnt.data(), d_cnt, nlist * 4, cudaMemcpyDeviceToHost, st));
        DPH_CUDA(cudaStreamSynchronize(st));
    }

    // 2. plan: the new layout; the first block that moves
    std::vector<int64_t> len_new(old.len.begin(), old.len.end()), rm_off(nlist, 0);
    for (int64_t l = lo, acc = 0; l < hi; l++) { len_new[l] -= h_cnt[l]; rm_off[l] = acc; acc += h_cnt[l]; }
    DphLayout L;
    DPH_TRY(L.build(ix, len_new.data(), "remove_ids: bad list length; the index is unchanged"));
    const int64_t nb_new = L.nblocks;
    int64_t d_first = nb_new;
    for (int64_t l = lo; l < hi; l++)
        if (L.blk_off[l] != old.blk_off[l]) { d_first = L.blk_off[l]; break; }
    const int64_t dm_new = dm_n - R;
    // one staging buffer (<= ~256 MB) serves the block shift (codes + labels of chunk_blocks blocks) and the direct map (pairs)
    const int64_t max_blocks = std::max<int64_t>(1, dph_chunk_rows() * DPH_CODE / (DPH_BLK_BYTES + 256));
    const int64_t chunk_blocks = std::max<int64_t>(1, std::min(max_blocks, nb_new - d_first));
    const int64_t chunk_pairs = std::max<int64_t>(1, std::min(max_blocks * (DPH_BLK_BYTES + 256) / 16, dm_new));
    const int64_t stage_bytes = std::max(chunk_blocks * (DPH_BLK_BYTES + 256), chunk_pairs * 16);
    uint8_t* stage = nullptr;
    if (R > 0) {
        DPH_TRY(tmp.alloc(&stage, (size_t)stage_bytes, oom));
        DPH_CUDA(cudaMemcpyAsync(d_boff_new, L.blk_off.data(), nlist * 8, cudaMemcpyHostToDevice, st));
        DPH_CUDA(cudaMemcpyAsync(d_rm_off, rm_off.data(), nlist * 8, cudaMemcpyHostToDevice, st));
        rm_plan_moves_kernel<<<(unsigned)((R + 127) / 128), 128, 0, st>>>(rm_prow, R, bo, ix->list_len, d_cnt, d_rm_off, lo, hi, mv_src, mv_dst);
        DPH_CUDA(cudaGetLastError());
        try {                       // sorted by source for the direct-map remap; the sort's scratch is allocated before the index changes
            thrust::device_ptr<long long> ms(mv_src), md(mv_dst);
            thrust::sort_by_key(thrust::cuda::par.on(st), ms, ms + R, md);
        } catch (const std::exception& e) {
            cudaGetLastError();
            dph_set_error(std::string("remove_ids: device sort failed; the index is unchanged: ") + e.what());
            return 1;
        }
    }
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[1], st));
    // Every allocation is done: from here on the index changes.

    if (R > 0) {
        // 3. fill the holes, clear the tails (old layout)
        rm_fill_holes_kernel<<<(unsigned)((R + 127) / 128), 128, 0, st>>>(mv_src, mv_dst, R, ix->codes, w_ids);
        rm_clear_tail_kernel<<<(unsigned)(hi - lo), 32, 0, st>>>(bo, ix->list_len, d_cnt, lo, ix->codes, w_ids);
        DPH_CUDA(cudaGetLastError());
        // 4. shift blocks [d_first, nb_new) down, ascending, one staged chunk at a time: every source is at or above its destination,
        //    so a chunk's writes land below the sources of every later chunk
        uint8_t* st_codes = stage;
        long long* st_ids = (long long*)(stage + chunk_blocks * DPH_BLK_BYTES);
        for (int64_t d0 = d_first; d0 < nb_new; d0 += chunk_blocks) {
            const int64_t m = std::min(chunk_blocks, nb_new - d0);
            relayout_codes_kernel<<<(unsigned)m, 192, 0, st>>>(st_codes, d0, d_boff_new, bo, ix->list_len, lo, hi, ix->codes);
            relayout_ids_kernel<<<(unsigned)m, 32, 0, st>>>(st_ids, d0, d_boff_new, bo, ix->list_len, lo, hi, w_ids, nullptr, nullptr, nullptr, nullptr);
            DPH_CUDA(cudaGetLastError());
            DPH_CUDA(cudaMemcpyAsync(ix->codes + d0 * DPH_BLK_BYTES, st_codes, (size_t)m * DPH_BLK_BYTES, cudaMemcpyDeviceToDevice, st));
            DPH_CUDA(cudaMemcpyAsync(w_ids + d0 * 32, st_ids, (size_t)m * 256, cudaMemcpyDeviceToDevice, st));
        }
        if (prof) DPH_CUDA(cudaEventRecord(ix->aev[2], st));
        // 5. direct map: stable in-place compaction, rows remapped, through the same staging buffer
        long long *st_dm_ids = (long long*)stage, *st_dm_rows = (long long*)stage + chunk_pairs;
        for (int64_t d0 = 0; d0 < dm_new; d0 += chunk_pairs) {
            const int64_t m = std::min(chunk_pairs, dm_new - d0);
            rm_dm_gather_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(d0, m, rm_dm, p0, R, w_dm_ids, w_dm_rows, mv_src, mv_dst, bo,
                                                                            d_boff_new, lo, hi, st_dm_ids, st_dm_rows);
            DPH_CUDA(cudaGetLastError());
            DPH_CUDA(cudaMemcpyAsync(w_dm_ids + d0, st_dm_ids, (size_t)m * 8, cudaMemcpyDeviceToDevice, st));
            DPH_CUDA(cudaMemcpyAsync(w_dm_rows + d0, st_dm_rows, (size_t)m * 8, cudaMemcpyDeviceToDevice, st));
        }
    } else if (prof) DPH_CUDA(cudaEventRecord(ix->aev[2], st));
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[3], st));
    DPH_CUDA(cudaStreamSynchronize(st));

    // 6. commit: the label arrays an implicit-label index gained, then the layout
    if (was_implicit) {
        ix->ids = (int64_t*)w_ids; ix->dm_ids = (int64_t*)w_dm_ids; ix->dm_rows = (int64_t*)w_dm_rows;
        for (void* p : {(void*)w_ids, (void*)w_dm_ids, (void*)w_dm_rows}) conv.release(p);
        ix->dm_cap = ix->ntotal_local;
    }
    if (R > 0) DPH_TRY(dph_commit_layout(ix, std::move(L)));
    ix->dm_n = dm_new;
    ix->remove_tmp_peak = tmp.peak;
    if (prof)
        for (int s = 0; s < 3; s++) DPH_CUDA(cudaEventElapsedTime(&ix->remove_ms[s], ix->aev[s], ix->aev[s + 1]));
    if (n_removed_out) *n_removed_out = R;
    if (removed_per_list_out) for (int64_t l = lo; l < hi; l++) removed_per_list_out[l] = h_cnt[l];
    return 0;
}

DPH_API int dph_index_sync_list_len(dph_index* ix, const int64_t* list_len) {
    DPH_CHECK(ix && ix->list_len, "sync_list_len: lists are not set");
    DphLayout L;
    DPH_TRY(L.build(ix, list_len, "sync_list_len: bad list length; the index is unchanged"));
    bool changed = false;
    for (int64_t l = 0; l < ix->nlist; l++) {
        if (l >= ix->list_lo && l < ix->list_hi)
            DPH_CHECK(list_len[l] == ix->lay.len[l], "sync_list_len: a list of this shard has another length here; the index is unchanged");
        changed |= list_len[l] != ix->lay.len[l];
    }
    if (!changed) return 0;
    DPH_CHECK(ix->ids != nullptr, "sync_list_len: the labels of this shard are sequential and would move; the index is unchanged");
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    return dph_commit_layout(ix, std::move(L));
}

DPH_API int dph_index_last_remove_ms(const dph_index* ix, float* ms_out) {
    DPH_CHECK(ix->aev[0] != nullptr, "profiling was never enabled");
    std::copy(ix->remove_ms, ix->remove_ms + 3, ms_out);
    return 0;
}
DPH_API int64_t dph_index_last_remove_tmp_bytes(const dph_index* ix) { return ix->remove_tmp_peak; }
