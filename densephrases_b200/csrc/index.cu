// index.cu -- the dph_index handle: construction, the model tables, getters, reconstruct (lists: lists.cu, search: search.cu).
// C ABI declared in include/dph_b200.h (each entry point cites the reference call it replaces).
#include "index_internal.cuh"
#include <algorithm>
#include <string.h>

static thread_local std::string g_err;
void dph_set_error(const std::string& msg) { g_err = msg; }
DPH_API const char* dph_last_error(void) { return g_err.c_str(); }
DPH_API int dph_version(void) { return 103; }
int g_dph_tune[8] = {1, 0, 0, 0, 0, 0, 0, 0};      // [0] quad-scan IMAD level, [1] SGEMM tile (0 auto), [2] PQ-table kernel shape (0 auto)
DPH_API int dph_set_tuning(int knob, int value) {
    DPH_CHECK(knob >= 0 && knob < 8, "dph_set_tuning: unknown knob");
    g_dph_tune[knob] = value;
    return 0;
}

int DevBuf::ensure(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    DPH_CUDA(cudaMalloc(&p, want));
    cap = want;
    return 0;
}

// -------------------------------------------------------------------------------------------------
// generators (bit-identical to oracle/ivfpq_ref.c)
// -------------------------------------------------------------------------------------------------
__global__ void gen_normal_kernel(float* out, long long rows, int cols, uint64_t seed, uint64_t stream, float sc) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    long long r = i / cols; int t = (int)(i % cols);
    out[i] = dph_approx_normal(dph_rnd64(seed, stream, (uint64_t)r, (uint64_t)t), sc);
}

// -------------------------------------------------------------------------------------------------
// construction
// -------------------------------------------------------------------------------------------------
DPH_API int dph_index_create(dph_index** out, int d, int64_t nlist, int M, int nbits, int device) {
    DPH_CHECK(out != nullptr, "null out");
    DPH_CHECK(d == DPH_D && M == DPH_M && nbits == 8, "only d=768, M=96, nbits=8 (OPQ96/PQ96 of build_phrase_index.py:113-116) is built");
    DPH_CHECK(nlist >= 1 && nlist < (1ll << 31), "bad nlist");
    DPH_CUDA(cudaSetDevice(device));
    dph_index* ix = new dph_index();
    ix->device = device; ix->nlist = nlist; ix->list_lo = 0; ix->list_hi = nlist;
    cudaDeviceProp prop;
    DPH_CUDA(cudaGetDeviceProperties(&prop, device));
    ix->num_sms = prop.multiProcessorCount;
    if (prop.major != 9 || prop.minor != 0) { delete ix; dph_set_error("libdph_b200 is built for sm_90a (H100) only; found sm_" + std::to_string(prop.major) + std::to_string(prop.minor)); return 1; }
    *out = ix;
    return 0;
}
DPH_API void dph_index_free(dph_index* ix) {
    if (!ix) return;
    cudaSetDevice(ix->device);
    for (void* p : {ix->A, ix->C, ix->pq}) if (p) cudaFree(p);
    dph_free_lists(ix);
    for (int i = 0; i < DPH_PROF_RING; i++) { if (ix->ev0[i]) cudaEventDestroy(ix->ev0[i]); if (ix->ev1[i]) cudaEventDestroy(ix->ev1[i]); }
    for (cudaEvent_t e : ix->aev) if (e) cudaEventDestroy(e);
    delete ix;                                      // the workspace DevBufs free themselves, on the device set above
}
DPH_API int dph_index_set_stream(dph_index* ix, void* s) { ix->stream = (cudaStream_t)s; return 0; }

// A model table has one size per handle: the first call that sets it allocates it, later ones overwrite it in place.
static int model_table(float** p, size_t count) {
    if (!*p) DPH_CUDA(cudaMalloc((void**)p, count * sizeof(float)));
    return 0;
}
static int upload(float** dst, const float* src, size_t count, int mem, dph_index* ix) {
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_TRY(model_table(dst, count));
    DPH_CUDA(cudaMemcpyAsync(*dst, src, count * sizeof(float), mem == DPH_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, ix->stream));
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    return 0;
}
DPH_API int dph_index_set_opq(dph_index* ix, const float* A, int mem) { return upload(&ix->A, A, (size_t)ix->d * ix->d, mem, ix); }
DPH_API int dph_index_set_centroids(dph_index* ix, const float* C, int mem) { ix->csplit_lo = -1; return upload(&ix->C, C, (size_t)ix->nlist * ix->d, mem, ix); }
DPH_API int dph_index_set_pq(dph_index* ix, const float* pq, int mem) { return upload(&ix->pq, pq, (size_t)DPH_M * 256 * DPH_DSUB, mem, ix); }

DPH_API int dph_index_gen_centroids(dph_index* ix, uint64_t seed, float sigma) {
    DPH_CUDA(cudaSetDevice(ix->device));
    ix->csplit_lo = -1;
    DPH_TRY(model_table(&ix->C, (size_t)ix->nlist * ix->d));
    long long tot = (long long)ix->nlist * ix->d;
    gen_normal_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, ix->stream>>>(ix->C, ix->nlist, ix->d, seed, DPH_STREAM_CENTROIDS, sigma / DPH_IH4_STD);
    DPH_CUDA(cudaGetLastError());
    return 0;
}
DPH_API int dph_index_gen_pq(dph_index* ix, uint64_t seed, float sigma) {
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_TRY(model_table(&ix->pq, (size_t)DPH_M * 256 * DPH_DSUB));
    long long rows = DPH_M * 256;
    gen_normal_kernel<<<(unsigned)((rows * DPH_DSUB + 255) / 256), 256, 0, ix->stream>>>(ix->pq, rows, DPH_DSUB, seed, DPH_STREAM_PQ, sigma / DPH_IH4_STD);
    DPH_CUDA(cudaGetLastError());
    return 0;
}
DPH_API int dph_index_set_shard(dph_index* ix, int64_t lo, int64_t hi) {
    DPH_CHECK(0 <= lo && lo <= hi && hi <= ix->nlist, "bad shard range");
    DPH_CHECK(ix->codes == nullptr, "set_shard must precede set_lists");
    ix->list_lo = lo; ix->list_hi = hi;
    return 0;
}

// -------------------------------------------------------------------------------------------------
// getters
// -------------------------------------------------------------------------------------------------
DPH_API int64_t dph_index_ntotal(const dph_index* ix) { return ix->ntotal; }
DPH_API int64_t dph_index_ntotal_local(const dph_index* ix) { return ix->ntotal_local; }
DPH_API int dph_index_d(const dph_index* ix) { return ix->d; }
DPH_API int64_t dph_index_nlist(const dph_index* ix) { return ix->nlist; }
DPH_API int dph_index_nprobe(const dph_index* ix) { return ix->nprobe; }
DPH_API int dph_index_set_nprobe(dph_index* ix, int nprobe) {
    DPH_CHECK(nprobe >= 1 && nprobe <= DPH_MAX_NPROBE, "nprobe must be in [1,1024]");
    ix->nprobe = nprobe;
    return 0;
}
DPH_API int dph_index_set_coarse_tc(dph_index* ix, int on) { ix->coarse_tc = on ? 1 : 0; return 0; }
DPH_API int dph_index_set_scan_mode(dph_index* ix, int mode) {
    DPH_CHECK(mode >= 0 && mode <= 4, "bad scan mode");
    ix->scan_mode = mode;
    return 0;
}
DPH_API int dph_index_get_opq(const dph_index* ix, float* A_out, int mem) {
    DPH_CHECK(ix->A != nullptr, "OPQ matrix not set");
    DPH_CUDA(cudaMemcpy(A_out, ix->A, (size_t)ix->d * ix->d * 4, mem == DPH_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice));
    return 0;
}
DPH_API int dph_index_set_profile(dph_index* ix, int on) {
    DPH_CUDA(cudaSetDevice(ix->device));
    if (on && !ix->ev0[0])
        for (int i = 0; i < DPH_PROF_RING; i++) { DPH_CUDA(cudaEventCreate(&ix->ev0[i])); DPH_CUDA(cudaEventCreate(&ix->ev1[i])); }
    if (on && !ix->aev[0])
        for (cudaEvent_t& e : ix->aev) DPH_CUDA(cudaEventCreate(&e));
    ix->profile = on != 0;
    ix->prof_n = 0;
    return 0;
}
DPH_API int dph_index_last_scan_ms(dph_index* ix, float* ms) {
    DPH_CHECK(ix->ev0[0] && ix->prof_n > 0, "no profiled search");
    int i = (int)((ix->prof_n - 1) % DPH_PROF_RING);
    DPH_CUDA(cudaEventSynchronize(ix->ev1[i]));
    DPH_CUDA(cudaEventElapsedTime(ms, ix->ev0[i], ix->ev1[i]));
    return 0;
}
DPH_API int dph_index_profile_scan_ms(dph_index* ix, float* ms_out, int max_out) {
    DPH_CHECK(ix->ev0[0] != nullptr, "profiling was never enabled");
    int n = (int)std::min<int64_t>(std::min<int64_t>(ix->prof_n, DPH_PROF_RING), max_out);
    for (int j = 0; j < n; j++) {
        int i = (int)((ix->prof_n - n + j) % DPH_PROF_RING);
        DPH_CUDA(cudaEventSynchronize(ix->ev1[i]));
        DPH_CUDA(cudaEventElapsedTime(ms_out + j, ix->ev0[i], ix->ev1[i]));
    }
    return 0;
}
DPH_API int dph_index_profile_count(const dph_index* ix) { return (int)std::min<int64_t>(ix->prof_n, DPH_PROF_RING); }
DPH_API int64_t dph_index_device_bytes(const dph_index* ix) {
    auto sz = [](int64_t count, int64_t elem) { return std::max<int64_t>(count, 1) * elem; };      // what each array was allocated with
    const int64_t nlist = ix->nlist;
    int64_t b = 0;
    if (ix->A) b += sz((int64_t)ix->d * ix->d, 4);
    if (ix->C) b += sz(nlist * ix->d, 4);
    if (ix->pq) b += sz(DPH_M * 256 * DPH_DSUB, 4);
    if (ix->list_len) b += sz(nlist, 4) + sz(nlist + 1, 8) + sz(nlist, 8);
    if (ix->codes) b += sz(ix->blk_cap * DPH_BLK_BYTES, 1);
    if (ix->ids) b += sz(ix->blk_cap * 32, 8);
    if (ix->dm_ids) b += 2 * sz(ix->dm_cap, 8);
    return b;
}
DPH_API const int32_t* dph_index_last_flags(const dph_index* ix) { return ix->flags.as<int32_t>(); }
DPH_API const int32_t* dph_index_last_probes(const dph_index* ix) { return ix->key.as<int32_t>(); }
DPH_API const float* dph_index_last_coarse(const dph_index* ix) { return ix->cd.as<float>(); }
DPH_API const float* dph_index_last_xr(const dph_index* ix) { return ix->xr.as<float>(); }
DPH_API int dph_index_last_used_pair_mode(const dph_index* ix) { return ix->last_group > 1 ? 1 : 0; }
DPH_API int dph_index_last_group_size(const dph_index* ix) { return ix->last_group; }
DPH_API int dph_index_copy_last(dph_index* ix, int which, void* dst_host, int64_t bytes) {
    const void* src = which == 0 ? ix->flags.p : which == 1 ? ix->key.p : which == 2 ? ix->cd.p : which == 3 ? ix->xr.p : nullptr;
    DPH_CHECK(src != nullptr, "copy_last: nothing to copy");
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    DPH_CUDA(cudaMemcpy(dst_host, src, (size_t)bytes, cudaMemcpyDeviceToHost));
    return 0;
}

int check_ready(dph_index* ix, int k) {
    DPH_CHECK(ix && ix->A && ix->C && ix->pq && ix->list_len, "index is not fully constructed (opq/centroids/pq/lists)");
    DPH_CHECK(k >= 1 && k <= DPH_MAX_K, "k must be in [1,1024]");
    return 0;
}

// -------------------------------------------------------------------------------------------------
// reconstruct: label -> (list, offset) -> centroid + PQ decode (rotated space)
// -------------------------------------------------------------------------------------------------
struct LocateArgs {
    const long long* list_start; long long nlist; long long list_lo, list_hi; const long long* blk_off; const int* list_len;
    const long long* dm_ids; const long long* dm_rows; long long dm_n; bool explicit_ids;
};
__device__ __forceinline__ bool locate_label(const LocateArgs& a, long long id, long long& l, long long& prow) {
    if (!a.explicit_ids) {
        if (id < 0 || id >= a.list_start[a.nlist]) return false;
        long long lo = 0, hi = a.nlist;      // last l with list_start[l] <= id
        while (hi - lo > 1) { long long mid = (lo + hi) >> 1; if (a.list_start[mid] <= id) lo = mid; else hi = mid; }
        l = lo;
        if (l < a.list_lo || l >= a.list_hi) return false;
        long long j = id - a.list_start[l];
        prow = (a.blk_off[l] + (j >> 5)) * 32 + (j & 31);
        return true;
    }
    long long lo = 0, hi = a.dm_n;
    if (hi == 0) return false;
    while (hi - lo > 1) { long long mid = (lo + hi) >> 1; if (a.dm_ids[mid] <= id) lo = mid; else hi = mid; }
    if (a.dm_ids[lo] != id) return false;
    prow = a.dm_rows[lo];
    l = list_of_block(a.blk_off, a.list_lo, a.list_hi, prow >> 5);
    return true;
}

__global__ void __launch_bounds__(96) reconstruct_kernel(LocateArgs la, const long long* ids, long long m, const uint8_t* codes, const float* C,
                                                          const float* pq, float* out, unsigned char* found) {
    const long long i = blockIdx.x;
    const int t = threadIdx.x;      // sub-quantizer
    __shared__ long long s_l, s_prow; __shared__ int s_ok;
    if (t == 0) { long long l = 0, pr = 0; s_ok = locate_label(la, ids[i], l, pr) ? 1 : 0; s_l = l; s_prow = pr; }
    __syncthreads();
    float4* o = reinterpret_cast<float4*>(out + i * DPH_D + t * 8);
    if (!s_ok) { o[0] = make_float4(0, 0, 0, 0); o[1] = make_float4(0, 0, 0, 0); if (t == 0 && found) found[i] = 0; return; }
    const long long blk = s_prow >> 5; const int lane = (int)(s_prow & 31);
    const unsigned char code = codes[blk * DPH_BLK_BYTES + dph_blk_addr(lane, t)];
    const float4* cb = reinterpret_cast<const float4*>(pq + ((size_t)t * 256 + code) * 8);
    const float4* ce = reinterpret_cast<const float4*>(C + s_l * DPH_D + t * 8);
    float4 a0 = cb[0], a1 = cb[1], c0 = ce[0], c1 = ce[1];
    o[0] = make_float4(a0.x + c0.x, a0.y + c0.y, a0.z + c0.z, a0.w + c0.w);
    o[1] = make_float4(a1.x + c1.x, a1.y + c1.y, a1.z + c1.z, a1.w + c1.w);
    if (t == 0 && found) found[i] = 1;
}

static LocateArgs make_locate(const dph_index* ix) {
    LocateArgs la;
    la.list_start = (const long long*)ix->list_start; la.nlist = ix->nlist; la.list_lo = ix->list_lo; la.list_hi = ix->list_hi;
    la.blk_off = (const long long*)ix->blk_off; la.list_len = ix->list_len; la.dm_ids = (const long long*)ix->dm_ids;
    la.dm_rows = (const long long*)ix->dm_rows; la.dm_n = ix->dm_n; la.explicit_ids = ix->ids != nullptr;
    return la;
}

DPH_API int dph_index_reconstruct_batch(dph_index* ix, const int64_t* ids, int64_t m, float* out, uint8_t* found, int mem) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CUDA(cudaSetDevice(ix->device));
    if (m == 0) return 0;
    const int64_t* d_ids = ids; float* d_out = out; uint8_t* d_found = found;
    DevBuf &tmp_ids = ix->rb_ids, &tmp_out = ix->rb_out, &tmp_found = ix->rb_found;       // grow-only pools: no cudaMalloc / cudaFree per call
    if (mem == DPH_MEM_HOST) {
        DPH_TRY(tmp_ids.ensure((size_t)m * 8)); DPH_TRY(tmp_out.ensure((size_t)m * ix->d * 4)); DPH_TRY(tmp_found.ensure((size_t)m));
        DPH_CUDA(cudaMemcpyAsync(tmp_ids.p, ids, (size_t)m * 8, cudaMemcpyHostToDevice, ix->stream));
        d_ids = tmp_ids.as<int64_t>(); d_out = tmp_out.as<float>(); d_found = tmp_found.as<uint8_t>();
    }
    reconstruct_kernel<<<(unsigned)m, 96, 0, ix->stream>>>(make_locate(ix), (const long long*)d_ids, m, ix->codes, ix->C, ix->pq, d_out, d_found);
    DPH_CUDA(cudaGetLastError());
    if (mem == DPH_MEM_HOST) {
        DPH_CUDA(cudaMemcpyAsync(out, d_out, (size_t)m * ix->d * 4, cudaMemcpyDeviceToHost, ix->stream));
        if (found) DPH_CUDA(cudaMemcpyAsync(found, d_found, (size_t)m, cudaMemcpyDeviceToHost, ix->stream));
        DPH_CUDA(cudaStreamSynchronize(ix->stream));
    }
    return 0;
}

// ---- fused phrase-window scoring (SURVEY.md 8f #1): score[i,l] = <q[i], R^T-unrotated reconstruct(first_id[i] + l)> --------------
// The reference reconstructs every window vector, multiplies by R and dots with the query (index.py:282-300,338-343,363-368).
// Here the query is rotated once (xq = A q, sequential-k SGEMM) and dotted with centroid + PQ decode on the fly:
// <q, A^T v> == <A q, v>.  A label that is not in this shard/index contributes 0 (the reference's zero vector).
__global__ void __launch_bounds__(96) window_scores_kernel(LocateArgs la, const float* __restrict__ xq, const long long* __restrict__ first_id,
                                                            int L, const uint8_t* __restrict__ codes, const float* __restrict__ C,
                                                            const float* __restrict__ pq, float* __restrict__ out) {
    const long long i = blockIdx.x;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    __shared__ long long s_l, s_prow; __shared__ int s_ok; __shared__ float red[3];
    const float4* xp = reinterpret_cast<const float4*>(xq + i * DPH_D + t * 8);
    const float4 x0 = xp[0], x1 = xp[1];
    for (int w = 0; w < L; w++) {
        if (t == 0) { long long l = 0, pr = 0; s_ok = locate_label(la, first_id[i] + w, l, pr) ? 1 : 0; s_l = l; s_prow = pr; }
        __syncthreads();
        float part = 0.f;
        if (s_ok) {
            const long long blk = s_prow >> 5; const int ln = (int)(s_prow & 31);
            const unsigned char code = codes[blk * DPH_BLK_BYTES + dph_blk_addr(ln, t)];
            const float4* cb = reinterpret_cast<const float4*>(pq + ((size_t)t * 256 + code) * 8);
            const float4* ce = reinterpret_cast<const float4*>(C + s_l * DPH_D + t * 8);
            const float4 a0 = cb[0], a1 = cb[1], c0 = ce[0], c1 = ce[1];
            part = fmaf(x0.x, a0.x + c0.x, part); part = fmaf(x0.y, a0.y + c0.y, part); part = fmaf(x0.z, a0.z + c0.z, part); part = fmaf(x0.w, a0.w + c0.w, part);
            part = fmaf(x1.x, a1.x + c1.x, part); part = fmaf(x1.y, a1.y + c1.y, part); part = fmaf(x1.z, a1.z + c1.z, part); part = fmaf(x1.w, a1.w + c1.w, part);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
        if (lane == 0) red[warp] = part;
        __syncthreads();
        if (t == 0) out[i * L + w] = (red[0] + red[1]) + red[2];
        __syncthreads();
    }
}

DPH_API int dph_index_window_scores(dph_index* ix, const float* q, const int64_t* first_id, int64_t m, int L, float* out_scores, int mem) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CHECK(L >= 1 && L <= 64, "window length out of range");
    DPH_CUDA(cudaSetDevice(ix->device));
    if (m == 0) return 0;
    DevBuf &tq = ix->ws_q, &tid = ix->ws_id, &tout = ix->ws_out, &txq = ix->ws_xq;           // grow-only pools
    const float* dq = q; const int64_t* did = first_id; float* dout = out_scores;
    if (mem == DPH_MEM_HOST) {
        DPH_TRY(tq.ensure((size_t)m * ix->d * 4)); DPH_TRY(tid.ensure((size_t)m * 8)); DPH_TRY(tout.ensure((size_t)m * L * 4));
        DPH_CUDA(cudaMemcpyAsync(tq.p, q, (size_t)m * ix->d * 4, cudaMemcpyHostToDevice, ix->stream));
        DPH_CUDA(cudaMemcpyAsync(tid.p, first_id, (size_t)m * 8, cudaMemcpyHostToDevice, ix->stream));
        dq = tq.as<float>(); did = tid.as<int64_t>(); dout = tout.as<float>();
    }
    DPH_TRY(txq.ensure((size_t)m * ix->d * 4));
    DPH_TRY(dph_launch_sgemm_nt_seq(dq, m, ix->A, ix->d, ix->d, txq.as<float>(), ix->stream));          // xq = A q
    window_scores_kernel<<<(unsigned)m, 96, 0, ix->stream>>>(make_locate(ix), txq.as<float>(), (const long long*)did, L, ix->codes, ix->C, ix->pq, dout);
    DPH_CUDA(cudaGetLastError());
    if (mem == DPH_MEM_HOST) DPH_CUDA(cudaMemcpyAsync(out_scores, dout, (size_t)m * L * 4, cudaMemcpyDeviceToHost, ix->stream));
    if (mem == DPH_MEM_HOST) DPH_CUDA(cudaStreamSynchronize(ix->stream));
    return 0;
}
