// index.cu -- the dph_index handle: construction, synthetic generation, search orchestration, reconstruct.
// C ABI declared in include/dph_b200.h (each entry point cites the reference call it replaces).
#include "index_internal.cuh"
#include <algorithm>
#include <numeric>
#include <stdlib.h>
#include <string.h>
#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/sequence.h>
#include <thrust/sort.h>

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
void DevBuf::release() { if (p) cudaFree(p); p = nullptr; cap = 0; }

template <class T> static int dev_alloc(T** out, size_t count, dph_index* ix) {
    if (*out) { cudaFree(*out); *out = nullptr; }
    size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
    DPH_CUDA(cudaMalloc((void**)out, bytes));
    ix->bytes += (int64_t)bytes;
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

int64_t dph_chunk_rows() {
    int64_t chunk_rows = (256ll << 20) / DPH_CODE;
    if (const char* ev = getenv("DPH_UPLOAD_CHUNK_ROWS")) chunk_rows = std::max<int64_t>(1, atoll(ev));      // tests: force many chunks
    return chunk_rows;
}

// One thread per (block, lane, 16-byte chunk): writes the interleaved/rotated layout (common.cuh).
// raw != nullptr: gather from list-major rows [*,96] (row index = local_row_start[l] + j); else synthesise from seed.
__global__ void __launch_bounds__(192) fill_blocks_kernel(uint8_t* codes, long long nblocks, const long long* blk_off, const int* list_len,
                                                          long long list_lo, long long list_hi, const uint8_t* raw,
                                                          const long long* local_row_start, uint64_t seed, long long blk0, long long raw_row0) {
    const long long blk = blk0 + blockIdx.x;                  // this launch covers blocks [blk0, nblocks)
    if (blk >= nblocks) return;
    const int lane = threadIdx.x & 31, c = threadIdx.x >> 5;   // c in 0..5
    __shared__ long long s_l;
    if (threadIdx.x == 0) s_l = list_of_block(blk_off, list_lo, list_hi, blk);
    __syncthreads();
    const long long l = s_l;
    const long long j = (blk - blk_off[l]) * 32 + lane;
    const bool valid = j < (long long)list_len[l];
    const int seg = c >> 1;
    unsigned char bytes[16];
    if (!valid) {
#pragma unroll
        for (int b = 0; b < 16; b++) bytes[b] = 0;
    } else if (raw) {
        const uint8_t* row = raw + (local_row_start[l - list_lo] + j - raw_row0) * DPH_CODE;      // raw holds rows [raw_row0, ...) of the shard
#pragma unroll
        for (int b = 0; b < 16; b++) { int t = c * 16 + b; int m = seg * 32 + ((lane + (t & 31)) & 31); bytes[b] = row[m]; }
    } else {
        uint64_t w[4];
#pragma unroll
        for (int i = 0; i < 4; i++) w[i] = dph_rnd64(seed, DPH_STREAM_CODES, (uint64_t)l, (uint64_t)(j * 12 + seg * 4 + i));
#pragma unroll
        for (int b = 0; b < 16; b++) {
            int t = c * 16 + b; int ml = (lane + (t & 31)) & 31;     // byte within the 32-byte segment
            bytes[b] = (unsigned char)(w[ml >> 3] >> (8 * (ml & 7)));
        }
    }
    uint4 v;
    memcpy(&v, bytes, 16);
    *reinterpret_cast<uint4*>(codes + blk * DPH_BLK_BYTES + c * 512 + lane * 16) = v;
}

// labels of the padded rows of blocks [blk0, nblocks) + the direct-map pairs (label, padded row) of the real rows
__global__ void fill_ids_kernel(long long* ids, long long nblocks, const long long* blk_off, const int* list_len, long long list_lo,
                                long long list_hi, const long long* raw_ids, const long long* local_row_start, long long blk0, long long raw_row0,
                                long long* dm_ids, long long* dm_rows) {
    const long long blk = blk0 + blockIdx.x;
    if (blk >= nblocks) return;
    const long long l = list_of_block(blk_off, list_lo, list_hi, blk);
    const long long j = (blk - blk_off[l]) * 32 + threadIdx.x;
    const bool real = j < (long long)list_len[l];
    const long long row = local_row_start[l - list_lo] + j;
    const long long id = real ? raw_ids[row - raw_row0] : -1;
    ids[blk * 32 + threadIdx.x] = id;
    if (real) { dm_ids[row] = id; dm_rows[row] = blk * 32 + threadIdx.x; }
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
    void* ptrs[] = {ix->A, ix->C, ix->pq, ix->list_len, ix->list_start, ix->blk_off, ix->codes, ix->ids, ix->dm_ids, ix->dm_rows};
    for (void* p : ptrs) if (p) cudaFree(p);
    DevBuf* bufs[] = {&ix->xdev, &ix->xr, &ix->S, &ix->key, &ix->cd, &ix->lut_canon, &ix->lutmax, &ix->segs, &ix->wpre, &ix->qinfo,
                      &ix->cand, &ix->cand_off, &ix->cand_cnt, &ix->gthr, &ix->flags, &ix->work, &ix->Dp, &ix->Ip, &ix->Gp, &ix->Dh, &ix->Ih, &ix->eps, &ix->nseg, &ix->lutmin, &ix->lutmaxv, &ix->lutq, &ix->qparams, &ix->gdense,
                      &ix->pl_cnt, &ix->pl_fill, &ix->pl_off, &ix->pl_blockpre, &ix->pl_entries, &ix->pl_unitpre, &ix->pl_units, &ix->pl_udesc, &ix->pairwork, &ix->csplit, &ix->xsplit, &ix->candkeys, &ix->cflags, &ix->selkeys, &ix->recbuf,
                      &ix->rb_ids, &ix->rb_out, &ix->rb_found, &ix->ws_q, &ix->ws_id, &ix->ws_out, &ix->ws_xq, &ix->enc_key, &ix->enc_cd,
                      &ix->enc_list, &ix->enc_codes};
    for (DevBuf* b : bufs) b->release();
    for (int i = 0; i < DPH_PROF_RING; i++) { if (ix->ev0[i]) cudaEventDestroy(ix->ev0[i]); if (ix->ev1[i]) cudaEventDestroy(ix->ev1[i]); }
    for (cudaEvent_t e : ix->aev) if (e) cudaEventDestroy(e);
    delete ix;
}
DPH_API int dph_index_set_stream(dph_index* ix, void* s) { ix->stream = (cudaStream_t)s; return 0; }

static int upload(float** dst, const float* src, size_t count, int mem, dph_index* ix) {
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_TRY(dev_alloc(dst, count, ix));
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
    DPH_TRY(dev_alloc(&ix->C, (size_t)ix->nlist * ix->d, ix));
    long long tot = (long long)ix->nlist * ix->d;
    gen_normal_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, ix->stream>>>(ix->C, ix->nlist, ix->d, seed, DPH_STREAM_CENTROIDS, sigma / DPH_IH4_STD);
    DPH_CUDA(cudaGetLastError());
    return 0;
}
DPH_API int dph_index_gen_pq(dph_index* ix, uint64_t seed, float sigma) {
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_TRY(dev_alloc(&ix->pq, (size_t)DPH_M * 256 * DPH_DSUB, ix));
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

static int set_lists_common(dph_index* ix, const int64_t* list_len, const uint8_t* codes, const int64_t* ids, bool synthetic, uint64_t seed) {
    DPH_CUDA(cudaSetDevice(ix->device));
    const int64_t nlist = ix->nlist, lo = ix->list_lo, hi = ix->list_hi;
    ix->h_list_len.assign(list_len, list_len + nlist);
    ix->h_list_start.assign(nlist + 1, 0);
    for (int64_t l = 0; l < nlist; l++) {
        DPH_CHECK(list_len[l] >= 0 && list_len[l] < (1ll << 31), "bad list length");
        ix->h_list_start[l + 1] = ix->h_list_start[l] + list_len[l];
    }
    ix->ntotal = ix->h_list_start[nlist];
    std::vector<int32_t> len32(nlist);
    std::vector<int64_t> blk_off(nlist, -1), local_row_start(std::max<int64_t>(hi - lo, 1), 0);
    int64_t nb = 0, rows = 0;
    for (int64_t l = 0; l < nlist; l++) len32[l] = (int32_t)list_len[l];
    for (int64_t l = lo; l < hi; l++) {
        blk_off[l] = nb; local_row_start[l - lo] = rows;
        nb += (list_len[l] + 31) / 32; rows += list_len[l];
    }
    ix->nblocks_local = nb; ix->ntotal_local = rows; ix->blk_cap = -1;
    DPH_TRY(dev_alloc(&ix->list_len, (size_t)nlist, ix));
    DPH_TRY(dev_alloc(&ix->list_start, (size_t)nlist + 1, ix));
    DPH_TRY(dev_alloc(&ix->blk_off, (size_t)nlist, ix));
    DPH_CUDA(cudaMemcpy(ix->list_len, len32.data(), nlist * 4, cudaMemcpyHostToDevice));
    DPH_CUDA(cudaMemcpy(ix->list_start, ix->h_list_start.data(), (nlist + 1) * 8, cudaMemcpyHostToDevice));
    DPH_CUDA(cudaMemcpy(ix->blk_off, blk_off.data(), nlist * 8, cudaMemcpyHostToDevice));
    DPH_TRY(dev_alloc(&ix->codes, (size_t)nb * DPH_BLK_BYTES, ix));
    if (nb == 0) return 0;
    int64_t* d_lrs = nullptr;
    DPH_CUDA(cudaMalloc((void**)&d_lrs, local_row_start.size() * 8));
    DPH_CUDA(cudaMemcpy(d_lrs, local_row_start.data(), local_row_start.size() * 8, cudaMemcpyHostToDevice));
    if (synthetic) {
        for (int64_t b0 = 0; b0 < nb; b0 += (1ll << 30)) {          // grid.x limit
            const unsigned g = (unsigned)std::min<int64_t>(nb - b0, 1ll << 30);
            fill_blocks_kernel<<<g, 192, 0, ix->stream>>>(ix->codes, std::min<int64_t>(nb, b0 + g), (const long long*)ix->blk_off, ix->list_len, lo, hi, nullptr,
                                                         (const long long*)d_lrs, seed, b0, 0);
        }
        DPH_CUDA(cudaGetLastError());
    } else {
        DPH_CHECK(codes != nullptr, "codes is null");
        // Upload in chunks of whole lists through a bounded staging buffer (<= ~256 MB of rows): the raw list-major copy never
        // sits on the device next to the blocked one.  Labels go the same way; the direct map (faiss DirectMap::Hashtable,
        // build_phrase_index.py:139-141) is filled by the same kernel and sorted ON THE DEVICE.
        const int64_t chunk_rows = dph_chunk_rows();
        auto chunk_end = [&](int64_t l0, int64_t& acc) {       // lists [l0, l1) of one upload: whole lists, <= chunk_rows rows (one list may exceed it)
            int64_t l1 = l0;
            acc = 0;
            while (l1 < hi && (acc == 0 || acc + list_len[l1] <= chunk_rows)) { acc += list_len[l1]; l1++; }
            return l1;
        };
        int64_t max_rows = 0;
        for (int64_t l0 = lo, acc = 0; l0 < hi;) { const int64_t l1 = chunk_end(l0, acc); max_rows = std::max(max_rows, acc); l0 = l1; }
        uint8_t* d_raw = nullptr; int64_t* d_rawids = nullptr;
        DPH_CUDA(cudaMalloc((void**)&d_raw, std::max<size_t>((size_t)max_rows * DPH_CODE, 1)));
        if (ids) {
            DPH_CUDA(cudaMalloc((void**)&d_rawids, std::max<size_t>((size_t)max_rows * 8, 8)));
            DPH_TRY(dev_alloc(&ix->ids, (size_t)nb * 32, ix));
            DPH_TRY(dev_alloc(&ix->dm_ids, (size_t)rows, ix));
            DPH_TRY(dev_alloc(&ix->dm_rows, (size_t)rows, ix));
        }
        int64_t l0 = lo;
        while (l0 < hi) {
            int64_t acc = 0;
            const int64_t l1 = chunk_end(l0, acc);
            const int64_t r0 = local_row_start[l0 - lo];
            const int64_t b0 = blk_off[l0], b1 = (l1 < hi) ? blk_off[l1] : nb;
            if (acc > 0 && b1 > b0) {
                DPH_CUDA(cudaMemcpyAsync(d_raw, codes + (size_t)r0 * DPH_CODE, (size_t)acc * DPH_CODE, cudaMemcpyHostToDevice, ix->stream));
                fill_blocks_kernel<<<(unsigned)(b1 - b0), 192, 0, ix->stream>>>(ix->codes, b1, (const long long*)ix->blk_off, ix->list_len, lo, hi, d_raw,
                                                                                 (const long long*)d_lrs, 0, b0, r0);
                if (ids) {
                    DPH_CUDA(cudaMemcpyAsync(d_rawids, ids + r0, (size_t)acc * 8, cudaMemcpyHostToDevice, ix->stream));
                    fill_ids_kernel<<<(unsigned)(b1 - b0), 32, 0, ix->stream>>>((long long*)ix->ids, b1, (const long long*)ix->blk_off, ix->list_len, lo, hi,
                                                                                 (const long long*)d_rawids, (const long long*)d_lrs, b0, r0,
                                                                                 (long long*)ix->dm_ids, (long long*)ix->dm_rows);
                }
                DPH_CUDA(cudaGetLastError());
                DPH_CUDA(cudaStreamSynchronize(ix->stream));       // the staging buffers are reused by the next chunk
            }
            l0 = l1;
        }
        cudaFree(d_raw);
        if (d_rawids) cudaFree(d_rawids);
        if (ids) {
            thrust::device_ptr<long long> kp((long long*)ix->dm_ids), vp((long long*)ix->dm_rows);
            thrust::sort_by_key(thrust::cuda::par.on(ix->stream), kp, kp + rows, vp);
            ix->dm_n = rows;
        }
    }
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    cudaFree(d_lrs);
    return 0;
}
DPH_API int dph_index_set_lists(dph_index* ix, const int64_t* list_len, const uint8_t* codes, const int64_t* ids) {
    return set_lists_common(ix, list_len, codes, ids, false, 0);
}
DPH_API int dph_index_set_lists_synthetic(dph_index* ix, const int64_t* list_len, uint64_t seed) {
    return set_lists_common(ix, list_len, nullptr, nullptr, true, seed);
}

// -------------------------------------------------------------------------------------------------
// add_with_ids (DESIGN.md 3, "Growing the index").  The batch is encoded (encode.cu), then the shard's lists are laid out again into
// buffers of the exact new size.  Old rows keep their offsets j inside their list, so every old 3 KB block moves whole; the new rows
// follow in input order.  The result is byte-identical to set_lists of the concatenated list-major arrays.
// -------------------------------------------------------------------------------------------------
static int check_ready(dph_index* ix, int k);

__global__ void iota_kernel(long long* out, long long n, long long base) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = base + i;
}
// flag bits: 2 = negative label, 4 = unassigned vector; cnt[l] += new rows of list l
__global__ void add_validate_kernel(const long long* list_no, const long long* ids, long long n, int* flag, int* cnt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long l = list_no[i];
    if (l < 0) atomicOr(flag, 4);
    else atomicAdd(&cnt[l], 1);
    if (ids[i] < 0) atomicOr(flag, 2);
}

// one CTA per block of the new layout: old blocks move whole (same rows, same lanes), blocks past a list's old end start as zeros
__global__ void __launch_bounds__(192) relayout_codes_kernel(uint8_t* dst, long long blk0, const long long* boff_new, const long long* boff_old,
                                                             const int* len_old, long long lo, long long hi, const uint8_t* codes_old) {
    const long long blk = blk0 + blockIdx.x;
    __shared__ long long s_l;
    if (threadIdx.x == 0) s_l = list_of_block(boff_new, lo, hi, blk);
    __syncthreads();
    const long long l = s_l, b = blk - boff_new[l];
    uint4 v = make_uint4(0, 0, 0, 0);
    if (b < ((long long)len_old[l] + 31) / 32) v = reinterpret_cast<const uint4*>(codes_old + (boff_old[l] + b) * DPH_BLK_BYTES)[threadIdx.x];
    reinterpret_cast<uint4*>(dst + (long long)blockIdx.x * DPH_BLK_BYTES)[threadIdx.x] = v;
}
// labels of the new layout's old rows (-1 elsewhere; the new rows are written by add_scatter_kernel).  Implicit labels (ids_old null)
// become explicit: list_start_old[l] + j, with their direct-map pairs at the row's old local position (already in label order).
__global__ void relayout_ids_kernel(long long* dst, long long blk0, const long long* boff_new, const long long* boff_old, const int* len_old,
                                    long long lo, long long hi, const long long* ids_old, const long long* list_start_old,
                                    const long long* lrs_old, long long* dm_ids, long long* dm_rows) {
    const long long blk = blk0 + blockIdx.x;
    const long long l = list_of_block(boff_new, lo, hi, blk), b = blk - boff_new[l];
    const long long j = b * 32 + threadIdx.x;
    long long id = -1;
    if (j < (long long)len_old[l]) {
        if (ids_old) id = ids_old[(boff_old[l] + b) * 32 + threadIdx.x];
        else {
            id = list_start_old[l] + j;
            dm_ids[lrs_old[l - lo] + j] = id;
            dm_rows[lrs_old[l - lo] + j] = blk * 32 + threadIdx.x;
        }
    }
    dst[(long long)blockIdx.x * 32 + threadIdx.x] = id;
}
// existing direct-map pairs (explicit labels): old padded row -> the same (list, j) in the new layout
__global__ void remap_dm_kernel(const long long* dm_ids_old, const long long* dm_rows_old, long long cnt, const long long* boff_old,
                                const long long* boff_new, long long lo, long long hi, long long* dm_ids_new, long long* dm_rows_new) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    const long long prow = dm_rows_old[i], ob = prow >> 5;
    const long long l = list_of_block(boff_old, lo, hi, ob);
    dm_ids_new[i] = dm_ids_old[i];
    dm_rows_new[i] = ((boff_new[l] + ob - boff_old[l]) << 5) | (prow & 31);
}
// new row of sorted position s (rows sorted stably by list: input order inside a list) -> j = old length + rank inside the batch.
// Its direct-map pair goes to slot dm0 + (input row), so that equal labels keep insertion order through the stable sort; rows of
// lists outside the shard get a sentinel label that sorts past the live entries.
__global__ void add_scatter_kernel(long long n, const long long* sorted_list, const long long* perm, const long long* bstart, const int* len_old,
                                   const long long* boff_new, long long lo, long long hi, const uint8_t* codes_all, const long long* ids_all,
                                   uint8_t* codes_new, long long* ids_new, long long* dm_ids, long long* dm_rows, long long dm0) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const long long l = sorted_list[s], r = perm[s];
    if (l < lo || l >= hi) { dm_ids[dm0 + r] = 0x7FFFFFFFFFFFFFFFll; dm_rows[dm0 + r] = -1; return; }
    const long long j = (long long)len_old[l] + (s - bstart[l]);
    const long long blk = boff_new[l] + (j >> 5);
    const int lane = (int)(j & 31);
    uint4 row4[6];
#pragma unroll
    for (int c = 0; c < 6; c++) row4[c] = reinterpret_cast<const uint4*>(codes_all + r * DPH_CODE)[c];
    dph_store_row(codes_new, blk, lane, reinterpret_cast<const unsigned char*>(row4));
    const long long id = ids_all[r];
    ids_new[blk * 32 + lane] = id;
    dm_ids[dm0 + r] = id;
    dm_rows[dm0 + r] = blk * 32 + lane;
}

DPH_API int dph_index_add_with_ids(dph_index* ix, const float* x, int64_t n, const int64_t* ids, int mem) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CHECK(n >= 0, "add_with_ids: n must be >= 0");
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n == 0) return 0;
    cudaStream_t st = ix->stream;
    const int64_t nlist = ix->nlist, lo = ix->list_lo, hi = ix->list_hi;
    for (float& a : ix->add_ms) a = 0.f;
    DevTmp tmp;
    const char* oom = "add_with_ids: not enough device memory for the batch; the index is unchanged";
    int64_t *list_all, *ids_all; uint8_t* codes_all; int *flag, *cnt;
    DPH_TRY(tmp.alloc(&list_all, n, oom)); DPH_TRY(tmp.alloc(&ids_all, n, oom)); DPH_TRY(tmp.alloc(&codes_all, (size_t)n * DPH_M, oom));
    DPH_TRY(tmp.alloc(&flag, 1, oom)); DPH_TRY(tmp.alloc(&cnt, nlist, oom));
    DPH_CUDA(cudaMemsetAsync(flag, 0, 4, st));
    DPH_CUDA(cudaMemsetAsync(cnt, 0, nlist * 4, st));
    // 1. assign + encode (host input: bounded staging, one encode chunk at a time)
    if (mem == DPH_MEM_DEVICE) DPH_TRY(dph_encode_rows(ix, x, n, list_all, codes_all, flag));
    else {
        const int64_t cs = std::min(dph_encode_chunk(ix), n);
        DPH_TRY(ix->xdev.ensure((size_t)cs * ix->d * 4));
        for (int64_t o = 0; o < n; o += cs) {
            const int64_t m = std::min(cs, n - o);
            DPH_CUDA(cudaMemcpyAsync(ix->xdev.p, x + o * ix->d, (size_t)m * ix->d * 4, cudaMemcpyHostToDevice, st));
            DPH_TRY(dph_encode_rows(ix, ix->xdev.as<float>(), m, list_all + o, codes_all + o * DPH_M, flag));
        }
    }
    if (ids) DPH_CUDA(cudaMemcpyAsync(ids_all, ids, (size_t)n * 8, mem == DPH_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, st));
    else iota_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((long long*)ids_all, n, ix->ntotal);        // IndexIVF::add: ntotal + i
    add_validate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const long long*)list_all, (const long long*)ids_all, n, flag, cnt);
    DPH_CUDA(cudaGetLastError());
    int h_flag = 0;
    std::vector<int32_t> h_cnt(nlist);
    DPH_CUDA(cudaMemcpyAsync(&h_flag, flag, 4, cudaMemcpyDeviceToHost, st));
    DPH_CUDA(cudaMemcpyAsync(h_cnt.data(), cnt, nlist * 4, cudaMemcpyDeviceToHost, st));
    DPH_CUDA(cudaStreamSynchronize(st));
    DPH_CHECK(!(h_flag & 1), "add_with_ids: the input holds a non-finite value; the index is unchanged");
    DPH_CHECK(!(h_flag & 2), "add_with_ids: negative label (-1 marks padding rows); the index is unchanged");
    DPH_CHECK(!(h_flag & 4), "add_with_ids: a vector has no best list; the index is unchanged");

    // 2. the new layout: every list's length (all shards), this shard's tightly packed blocks
    std::vector<int64_t> len_new(nlist), start_new(nlist + 1, 0), boff_new(nlist, -1), bstart(nlist, 0), lrs_old(std::max<int64_t>(hi - lo, 1), 0);
    std::vector<int32_t> len32(nlist);
    int64_t nb = 0, rows = 0, rows_old = 0, in_shard = 0;
    for (int64_t l = 0; l < nlist; l++) {
        len_new[l] = ix->h_list_len[l] + h_cnt[l];
        DPH_CHECK(len_new[l] < (1ll << 31), "add_with_ids: a list would exceed 2^31 - 1 rows; the index is unchanged");
        len32[l] = (int32_t)len_new[l];
        start_new[l + 1] = start_new[l] + len_new[l];
        if (l + 1 < nlist) bstart[l + 1] = bstart[l] + h_cnt[l];
    }
    for (int64_t l = lo; l < hi; l++) {
        boff_new[l] = nb; lrs_old[l - lo] = rows_old;
        nb += (len_new[l] + 31) / 32; rows += len_new[l]; rows_old += ix->h_list_len[l]; in_shard += h_cnt[l];
    }
    const bool was_explicit = ix->ids != nullptr;
    const int64_t dm_old = was_explicit ? ix->dm_n : ix->ntotal_local;       // pairs carried over
    const int64_t dm_cap = dm_old + n;

    // 3. every new buffer before anything changes: a failed allocation leaves the index as it was
    const char* oom2 = "add_with_ids: not enough device memory for the re-layout (the old and the new code buffers of the shard are live "
                       "together); the index is unchanged";
    uint8_t* codes_new; int64_t *ids_new, *dm_ids_new, *dm_rows_new, *d_boff_new, *d_bstart, *d_lrs, *perm;
    DPH_TRY(tmp.alloc(&codes_new, (size_t)nb * DPH_BLK_BYTES, oom2)); DPH_TRY(tmp.alloc(&ids_new, (size_t)nb * 32, oom2));
    DPH_TRY(tmp.alloc(&dm_ids_new, dm_cap, oom2)); DPH_TRY(tmp.alloc(&dm_rows_new, dm_cap, oom2));
    DPH_TRY(tmp.alloc(&d_boff_new, nlist, oom2)); DPH_TRY(tmp.alloc(&d_bstart, nlist, oom2));
    DPH_TRY(tmp.alloc(&d_lrs, lrs_old.size(), oom2)); DPH_TRY(tmp.alloc(&perm, n, oom2));
    DPH_CUDA(cudaMemcpyAsync(d_boff_new, boff_new.data(), nlist * 8, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemcpyAsync(d_bstart, bstart.data(), nlist * 8, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemcpyAsync(d_lrs, lrs_old.data(), lrs_old.size() * 8, cudaMemcpyHostToDevice, st));

    // 4. move the old blocks, scatter the new rows, merge the direct map
    const bool prof = ix->profile && ix->aev[0];
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[4], st));
    const long long *bo_new = (const long long*)d_boff_new, *bo_old = (const long long*)ix->blk_off;
    if (nb > 0) {
        relayout_codes_kernel<<<(unsigned)nb, 192, 0, st>>>(codes_new, 0, bo_new, bo_old, ix->list_len, lo, hi, ix->codes);
        relayout_ids_kernel<<<(unsigned)nb, 32, 0, st>>>((long long*)ids_new, 0, bo_new, bo_old, ix->list_len, lo, hi, (const long long*)ix->ids,
                                                       (const long long*)ix->list_start, (const long long*)d_lrs, (long long*)dm_ids_new,
                                                       (long long*)dm_rows_new);
    }
    if (was_explicit && ix->dm_n > 0)
        remap_dm_kernel<<<(unsigned)((ix->dm_n + 255) / 256), 256, 0, st>>>((const long long*)ix->dm_ids, (const long long*)ix->dm_rows, ix->dm_n,
                                                                           bo_old, bo_new, lo, hi, (long long*)dm_ids_new, (long long*)dm_rows_new);
    DPH_CUDA(cudaGetLastError());
    try {
        thrust::device_ptr<long long> kp((long long*)list_all), pp((long long*)perm);
        thrust::sequence(thrust::cuda::par.on(st), pp, pp + n);
        thrust::stable_sort_by_key(thrust::cuda::par.on(st), kp, kp + n, pp);
        add_scatter_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n, (const long long*)list_all, (const long long*)perm, (const long long*)d_bstart,
                                                                       ix->list_len, bo_new, lo, hi, codes_all, (const long long*)ids_all, codes_new,
                                                                       (long long*)ids_new, (long long*)dm_ids_new, (long long*)dm_rows_new, dm_old);
        DPH_CUDA(cudaGetLastError());
        thrust::device_ptr<long long> dk((long long*)dm_ids_new), dv((long long*)dm_rows_new);
        thrust::stable_sort_by_key(thrust::cuda::par.on(st), dk, dk + dm_cap, dv);       // equal labels keep insertion order
    } catch (const std::exception& e) {
        cudaGetLastError();
        dph_set_error(std::string("add_with_ids: device sort failed; the index is unchanged: ") + e.what());
        return 1;
    }
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[5], st));
    DPH_CUDA(cudaStreamSynchronize(st));

    // 5. commit: tables, then the buffers
    DPH_CUDA(cudaMemcpy(ix->blk_off, d_boff_new, nlist * 8, cudaMemcpyDeviceToDevice));
    DPH_CUDA(cudaMemcpy(ix->list_len, len32.data(), nlist * 4, cudaMemcpyHostToDevice));
    DPH_CUDA(cudaMemcpy(ix->list_start, start_new.data(), (nlist + 1) * 8, cudaMemcpyHostToDevice));
    const int64_t nb_old = ix->blk_cap < 0 ? ix->nblocks_local : ix->blk_cap;       // a remove leaves the allocation as it was
    int64_t old_bytes = std::max<int64_t>(nb_old * DPH_BLK_BYTES, 1);
    if (ix->ids) old_bytes += std::max<int64_t>(nb_old * 32, 1) * 8;
    if (ix->dm_ids) old_bytes += 2 * std::max<int64_t>(ix->dm_cap < 0 ? ix->ntotal_local : ix->dm_cap, 1) * 8;
    const int64_t new_bytes = std::max<int64_t>(nb * DPH_BLK_BYTES, 1) + std::max<int64_t>(nb * 32, 1) * 8 + 2 * std::max<int64_t>(dm_cap, 1) * 8;
    void* olds[] = {ix->codes, ix->ids, ix->dm_ids, ix->dm_rows};
    for (void* p : olds) if (p) cudaFree(p);
    ix->codes = codes_new; ix->ids = ids_new; ix->dm_ids = dm_ids_new; ix->dm_rows = dm_rows_new;
    for (void* p : {(void*)codes_new, (void*)ids_new, (void*)dm_ids_new, (void*)dm_rows_new}) tmp.release(p);
    ix->bytes += new_bytes - old_bytes;
    ix->dm_n = dm_old + in_shard; ix->dm_cap = dm_cap;
    ix->h_list_len = len_new; ix->h_list_start = start_new;
    ix->ntotal = start_new[nlist]; ix->ntotal_local = rows; ix->nblocks_local = nb; ix->blk_cap = -1;
    if (prof) DPH_CUDA(cudaEventElapsedTime(&ix->add_ms[3], ix->aev[4], ix->aev[5]));
    return 0;
}

// The inverse of set_lists: this shard's rows as list-major host arrays, through the same bounded staging.
__global__ void __launch_bounds__(192) read_blocks_kernel(const uint8_t* codes, long long nblocks, const long long* blk_off, const int* list_len,
                                                          long long list_lo, long long list_hi, const long long* ids, const long long* list_start,
                                                          const long long* local_row_start, long long blk0, long long raw_row0, uint8_t* raw,
                                                          long long* raw_ids) {
    const long long blk = blk0 + blockIdx.x;
    if (blk >= nblocks) return;
    const int lane = threadIdx.x & 31, c = threadIdx.x >> 5;
    __shared__ long long s_l;
    if (threadIdx.x == 0) s_l = list_of_block(blk_off, list_lo, list_hi, blk);
    __syncthreads();
    const long long l = s_l;
    const long long j = (blk - blk_off[l]) * 32 + lane;
    if (j >= (long long)list_len[l]) return;
    const long long row = local_row_start[l - list_lo] + j - raw_row0;
    const uint4 v = *reinterpret_cast<const uint4*>(codes + blk * DPH_BLK_BYTES + c * 512 + lane * 16);
    unsigned char bytes[16];
    memcpy(bytes, &v, 16);
    const int seg = c >> 1;
#pragma unroll
    for (int b = 0; b < 16; b++) { const int t = c * 16 + b; raw[row * DPH_CODE + seg * 32 + ((lane + (t & 31)) & 31)] = bytes[b]; }
    if (c == 0 && raw_ids) raw_ids[row] = ids ? ids[blk * 32 + lane] : list_start[l] + j;
}

DPH_API int dph_index_copy_lists(dph_index* ix, uint8_t* codes_out, int64_t* ids_out) {
    DPH_CHECK(ix && ix->list_len, "copy_lists: lists are not set");
    DPH_CUDA(cudaSetDevice(ix->device));
    const int64_t lo = ix->list_lo, hi = ix->list_hi;
    const std::vector<int64_t>& len = ix->h_list_len;
    if (ix->ntotal_local == 0) return 0;
    std::vector<int64_t> boff(hi - lo), lrs(hi - lo);
    for (int64_t l = lo, nb = 0, rows = 0; l < hi; l++) { boff[l - lo] = nb; lrs[l - lo] = rows; nb += (len[l] + 31) / 32; rows += len[l]; }
    const int64_t chunk_rows = dph_chunk_rows();
    auto chunk_end = [&](int64_t l0, int64_t& acc) {           // lists [l0, l1): whole lists, <= chunk_rows rows (one list may exceed it)
        int64_t l1 = l0;
        acc = 0;
        while (l1 < hi && (acc == 0 || acc + len[l1] <= chunk_rows)) { acc += len[l1]; l1++; }
        return l1;
    };
    int64_t max_rows = 0;
    for (int64_t l0 = lo, acc = 0; l0 < hi;) { const int64_t l1 = chunk_end(l0, acc); max_rows = std::max(max_rows, acc); l0 = l1; }
    DevTmp tmp;
    uint8_t* d_raw; int64_t *d_ids, *d_lrs;
    DPH_TRY(tmp.alloc(&d_raw, (size_t)max_rows * DPH_CODE, "copy_lists: staging"));
    DPH_TRY(tmp.alloc(&d_ids, (size_t)max_rows, "copy_lists: staging"));
    DPH_TRY(tmp.alloc(&d_lrs, lrs.size(), "copy_lists: staging"));
    DPH_CUDA(cudaMemcpyAsync(d_lrs, lrs.data(), lrs.size() * 8, cudaMemcpyHostToDevice, ix->stream));
    for (int64_t l0 = lo; l0 < hi;) {
        int64_t acc = 0;
        const int64_t l1 = chunk_end(l0, acc);
        const int64_t r0 = lrs[l0 - lo], b0 = boff[l0 - lo], b1 = l1 < hi ? boff[l1 - lo] : ix->nblocks_local;
        if (acc > 0 && b1 > b0) {
            read_blocks_kernel<<<(unsigned)(b1 - b0), 192, 0, ix->stream>>>(ix->codes, b1, (const long long*)ix->blk_off, ix->list_len, lo, hi,
                                                                           (const long long*)ix->ids, (const long long*)ix->list_start,
                                                                           (const long long*)d_lrs, b0, r0, d_raw, ids_out ? (long long*)d_ids : nullptr);
            DPH_CUDA(cudaGetLastError());
            DPH_CUDA(cudaMemcpyAsync(codes_out + (size_t)r0 * DPH_CODE, d_raw, (size_t)acc * DPH_CODE, cudaMemcpyDeviceToHost, ix->stream));
            if (ids_out) DPH_CUDA(cudaMemcpyAsync(ids_out + r0, d_ids, (size_t)acc * 8, cudaMemcpyDeviceToHost, ix->stream));
            DPH_CUDA(cudaStreamSynchronize(ix->stream));          // the staging buffers are reused by the next chunk
        }
        l0 = l1;
    }
    return 0;
}

DPH_API int dph_index_get_list_len(const dph_index* ix, int64_t* list_len_out) {
    DPH_CHECK(ix && ix->list_len, "lists are not set");
    std::copy(ix->h_list_len.begin(), ix->h_list_len.end(), list_len_out);
    return 0;
}
DPH_API int dph_index_last_add_ms(const dph_index* ix, float* ms_out) {
    DPH_CHECK(ix->aev[0] != nullptr, "profiling was never enabled");
    std::copy(ix->add_ms, ix->add_ms + 4, ms_out);
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
    return n < 0 ? 0 : 0 * n;
}
DPH_API int dph_index_profile_count(const dph_index* ix) { return (int)std::min<int64_t>(ix->prof_n, DPH_PROF_RING); }
DPH_API int64_t dph_index_device_bytes(const dph_index* ix) { return ix->bytes; }
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

// -------------------------------------------------------------------------------------------------
// search
// -------------------------------------------------------------------------------------------------
// stage: 0 = whole search; 1 = only rotation + this shard's coarse candidates (keys64 out); 2 = everything after the coarse
// quantizer, probes (key, cd) already in ix->key / ix->cd and rotated queries in ix->xr (sharded coarse quantizer, see sharded.py);
// 3 = only rotation + the coarse quantizer over ALL lists (query-split sharded search: this rank's slice of the batch)
static int search_chunk(dph_index* ix, const float* x_dev, int64_t n, int k, float* D, int64_t* I, uint32_t* G, int stage = 0,
                        unsigned long long* keys64 = nullptr) {
    cudaStream_t st = ix->stream;
    const int nprobe = ix->nprobe;
    const int grid = ix->num_sms;
    // candidates kept per CTA: k + slack.  The proof needs T_k - (k+slack)-th score > 2 eps; the pair filter's eps is dominated by
    // the 10-bit quantisation, so its slack grows with k (order statistics: the gap between ranks k and 1.5k is ~0.1 sigma).
    const int keep_single = k + DPH_KEEP_SLACK;
    const int keep_pair = k + (k / 2 > DPH_KEEP_SLACK ? k / 2 : DPH_KEEP_SLACK);
    // quad filter: 8-bit entries, eps ~2.7x the pair filter's: 2 eps ~ 0.26 sigma of the scores.  The drop threshold is some unit's
    // keep-th best, i.e. at global rank >= keep; the proof needs score(rank k) - score(rank keep) > 2 eps.  Order statistics of the
    // top of ~6 M scores: rank 10 -> rank 110 is ~0.5 sigma, which leaves a 2x margin (7-bit entries would need keep ~ 400).
    const int keep_quad = k + (2 * k > 100 ? 2 * k : 100);
    const int keep_max = keep_quad > keep_pair ? keep_quad : keep_pair;
    DPH_TRY(ix->xr.ensure((size_t)n * ix->d * 4));
    DPH_TRY(ix->S.ensure((size_t)n * ix->nlist * 4));
    DPH_TRY(ix->key.ensure((size_t)n * nprobe * 4));
    DPH_TRY(ix->cd.ensure((size_t)n * nprobe * 4));
    DPH_TRY(ix->lut_canon.ensure((size_t)n * DPH_LUT_CANON_FLOATS * 4));
    DPH_TRY(ix->lutmax.ensure((size_t)n * DPH_M * 4));
    DPH_TRY(ix->segs.ensure((size_t)n * nprobe * sizeof(DphSeg)));
    DPH_TRY(ix->wpre.ensure((size_t)(n + 1) * 8));
    DPH_TRY(ix->qinfo.ensure((size_t)n * 4));
    DPH_TRY(ix->eps.ensure((size_t)n * 4));
    DPH_TRY(ix->nseg.ensure((size_t)n * 4));
    // sharing gathers between the queries that probe a list pays when lists are probed by >= ~1.5 queries of the batch on average
    const int64_t eff_probe = std::min<int64_t>(nprobe, ix->nlist);
    // ... and when lists are long enough to amortise rebuilding the packed 192 KB LUT at every (list, query group) item
    const int64_t nl_local = std::max<int64_t>(ix->list_hi - ix->list_lo, 1);
    const bool long_lists = ix->ntotal_local / nl_local >= 4096;
    const bool shared = long_lists && n * eff_probe * 2 >= ix->nlist * 3;
    int group = 1;                                  // queries per gather: 1, 2 (pair-packed) or 4 (quad-packed)
    if (ix->scan_mode == DPH_SCAN_PAIR) group = 2;
    else if (ix->scan_mode == DPH_SCAN_QUAD) group = 4;
    else if (ix->scan_mode == DPH_SCAN_FAST && shared) group = 4;
    if (group == 4 && keep_quad > DPH_QUAD_KEEP_MAX) group = 2;
    if (group == 2 && keep_pair > 1536 - DPH_SCAN_THREADS) group = 1;
    const bool pair = group > 1;
    const int keep_fast = group == 4 ? keep_quad : (group == 2 ? keep_pair : keep_single);
    // group modes: query q's region holds nseg_q + blocks_q / per + 1 units of keep (plan_scan_kernel); summed over the batch,
    // sum_q blocks_q <= (queries per item) * sum over items of blocks <= (queries per item) * per * UNITS_PER_CTA * grid
    const size_t item_q = group == 4 ? DPH_QUAD_ITEM_Q : 2;
    DPH_TRY(ix->cand.ensure(((size_t)(2 * grid + 2 * n + 2) + (pair ? (size_t)(n * nprobe + item_q * DPH_PAIR_UNITS_PER_CTA * grid + 2 * n + 16) : 0)) * keep_max * 8));
    DPH_TRY(ix->cand_off.ensure((size_t)(n + 1) * 8));
    DPH_TRY(ix->cand_cnt.ensure((size_t)n * 4));
    DPH_TRY(ix->gthr.ensure((size_t)n * 4));
    DPH_TRY(ix->flags.ensure((size_t)n * 4));
    DPH_TRY(ix->work.ensure(sizeof(DphWork)));
    DPH_TRY(ix->lutmin.ensure((size_t)n * DPH_M * 4));
    DPH_TRY(ix->lutmaxv.ensure((size_t)n * DPH_M * 4));
    if (pair) {
        DPH_TRY(ix->lutq.ensure((size_t)n * (group == 4 ? DPH_LUTQ8_BYTES : DPH_LUT_SCAN_FLOATS * 2)));
        DPH_TRY(ix->qparams.ensure((size_t)n * 8));
        DPH_TRY(ix->gdense.ensure((size_t)n * nprobe * 4));
        DPH_TRY(ix->pl_cnt.ensure((size_t)ix->nlist * 4));
        DPH_TRY(ix->pl_fill.ensure((size_t)ix->nlist * 4));
        DPH_TRY(ix->pl_off.ensure((size_t)(ix->nlist + 1) * 4));
        DPH_TRY(ix->pl_blockpre.ensure((size_t)(ix->nlist + 1) * 8));
        DPH_TRY(ix->pl_entries.ensure((size_t)n * nprobe * 4));
        DPH_TRY(ix->pl_unitpre.ensure((size_t)(ix->nlist + 1) * 4));
        // units <= sum_l items_l * (blocks_l / seg + 1) <= total_blocks / seg + items <= UNITS_PER_CTA * grid + n * nprobe
        DPH_TRY(ix->pl_units.ensure((size_t)(n * nprobe + DPH_PAIR_UNITS_PER_CTA * grid + 16) * 8));
        if (group == 4) DPH_TRY(ix->pl_udesc.ensure((size_t)(n * nprobe + DPH_PAIR_UNITS_PER_CTA * grid + 16) * sizeof(DphUnit)));
        DPH_TRY(ix->pairwork.ensure(sizeof(DphPairWork)));
    }
    ix->last_n = n;
    if (stage != 1 && stage != 3) ix->last_group = group;
    if (stage == 1) ix->last_coarse_n = n;

    if (stage == 1) {
        const int64_t nl = ix->list_hi - ix->list_lo;
        DPH_TRY(dph_launch_sgemm_nt_seq(x_dev, n, ix->A, ix->d, ix->d, ix->xr.as<float>(), st));                   // OPQ rotation
        if (ix->coarse_tc) {
            int rc = dph_coarse_tc(ix, n, ix->list_lo, nl, nprobe, keys64, nullptr, nullptr, st);
            if (rc == 0) return 0;
            if (rc != 1) return rc;
        }
        DPH_TRY(dph_launch_sgemm_nt_seq(ix->xr.as<float>(), n, ix->C + ix->list_lo * ix->d, nl, ix->d, ix->S.as<float>(), st));   // this shard's centroids only
        DPH_TRY(dph_launch_coarse_select(ix->S.as<float>(), n, nl, nprobe, nullptr, nullptr, st, keys64, (unsigned)ix->list_lo));
        return 0;
    }
    if (stage == 0 || stage == 3) {
        DPH_TRY(dph_launch_sgemm_nt_seq(x_dev, n, ix->A, ix->d, ix->d, ix->xr.as<float>(), st));                   // OPQ rotation
        int rc = ix->coarse_tc ? dph_coarse_tc(ix, n, 0, ix->nlist, nprobe, nullptr, ix->key.as<int32_t>(), ix->cd.as<float>(), st) : 1;
        if (rc > 1) return rc;
        if (rc == 1) {
            DPH_TRY(dph_launch_sgemm_nt_seq(ix->xr.as<float>(), n, ix->C, ix->nlist, ix->d, ix->S.as<float>(), st));   // coarse scores
            DPH_TRY(dph_launch_coarse_select(ix->S.as<float>(), n, ix->nlist, nprobe, ix->key.as<int32_t>(), ix->cd.as<float>(), st, nullptr, 0u, nullptr, 0,
                                             &ix->selkeys));
        }
        if (stage == 3) return 0;
    }
    DPH_TRY(dph_launch_lut(ix->xr.as<float>(), n, ix->pq, ix->lut_canon.as<float>(), ix->lutmax.as<float>(),
                           ix->lutmin.as<float>(), ix->lutmaxv.as<float>(), pair ? ix->lutq.p : nullptr,
                           pair ? ix->qparams.as<float2>() : nullptr, st, group));
    if (ix->scan_mode != DPH_SCAN_EXACT) {
        DPH_TRY(dph_launch_plan(ix, n, k, keep_fast, grid, nullptr, st, group));
        if (ix->profile) DPH_CUDA(cudaEventRecord(ix->ev0[ix->prof_n % DPH_PROF_RING], st));
        if (pair) DPH_TRY(dph_launch_scan_pair(ix, n, keep_fast, grid, st, group));
        else DPH_TRY(dph_launch_scan(ix, n, k, keep_fast, DPH_SCAN_FAST, grid, st));
        if (ix->profile) { DPH_CUDA(cudaEventRecord(ix->ev1[ix->prof_n % DPH_PROF_RING], st)); ix->prof_n++; }
        DPH_TRY(dph_launch_merge(ix, n, k, DPH_SCAN_FAST, nullptr, D, I, G, st));
        // fallback for queries whose filter could not be proven exact (no-op launches when no flag is set)
        DPH_TRY(dph_launch_plan(ix, n, k, k, grid, ix->flags.as<int32_t>(), st, 1));
        DPH_TRY(dph_launch_scan(ix, n, k, k, DPH_SCAN_EXACT, grid, st));
        DPH_TRY(dph_launch_merge(ix, n, k, DPH_SCAN_EXACT, ix->flags.as<int32_t>(), D, I, G, st));
    } else {
        DPH_CUDA(cudaMemsetAsync(ix->flags.p, 0, (size_t)n * 4, st));
        DPH_TRY(dph_launch_plan(ix, n, k, k, grid, nullptr, st, 1));
        if (ix->profile) DPH_CUDA(cudaEventRecord(ix->ev0[ix->prof_n % DPH_PROF_RING], st));
        DPH_TRY(dph_launch_scan(ix, n, k, k, DPH_SCAN_EXACT, grid, st));
        if (ix->profile) { DPH_CUDA(cudaEventRecord(ix->ev1[ix->prof_n % DPH_PROF_RING], st)); ix->prof_n++; }
        DPH_TRY(dph_launch_merge(ix, n, k, DPH_SCAN_EXACT, nullptr, D, I, G, st));
    }
    return 0;
}

static int check_ready(dph_index* ix, int k) {
    DPH_CHECK(ix && ix->A && ix->C && ix->pq && ix->list_len, "index is not fully constructed (opq/centroids/pq/lists)");
    DPH_CHECK(k >= 1 && k <= DPH_MAX_K, "k must be in [1,1024]");
    return 0;
}
static int64_t chunk_size(const dph_index* ix, int64_t n) {
    int64_t c = (1ll << 28) / std::max<int64_t>(ix->nlist, 1);   // S chunk <= 1 GiB
    c = std::max<int64_t>(1, std::min<int64_t>(c, 4096));
    return std::min(c, n);
}

DPH_API int dph_index_search_partial(dph_index* ix, const float* x_dev, int64_t n, int k, float* D, int64_t* I, uint32_t* G) {
    DPH_TRY(check_ready(ix, k));
    DPH_CUDA(cudaSetDevice(ix->device));
    const int64_t cs = chunk_size(ix, n);
    for (int64_t o = 0; o < n; o += cs) {
        int64_t m = std::min(cs, n - o);
        DPH_TRY(search_chunk(ix, x_dev + o * ix->d, m, k, D + o * k, I + o * k, G + o * k));
    }
    return 0;
}

// ---- sharded coarse quantizer (every rank scores only its own lists' centroids; SURVEY.md 8e "Partitioning") ----
DPH_API int dph_index_coarse_local(dph_index* ix, const float* x_dev, int64_t n, uint64_t* keys_dev) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_CHECK(n <= chunk_size(ix, n), "coarse_local: batch too large for one chunk");
    return search_chunk(ix, x_dev, n, 1, nullptr, nullptr, nullptr, 1, (unsigned long long*)keys_dev);
}
DPH_API int dph_index_search_preassigned(dph_index* ix, const uint64_t* keys_gathered_dev, int nshards, int64_t n, int k, float* D_dev,
                                         int64_t* I_dev, uint32_t* G_dev) {
    DPH_TRY(check_ready(ix, k));
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_CHECK(n == ix->last_coarse_n, "search_preassigned must follow coarse_local with the same batch");
    DPH_TRY(ix->key.ensure((size_t)n * ix->nprobe * 4));
    DPH_TRY(ix->cd.ensure((size_t)n * ix->nprobe * 4));
    DPH_TRY(dph_launch_coarse_merge((const unsigned long long*)keys_gathered_dev, nshards, n, ix->nprobe, ix->key.as<int32_t>(), ix->cd.as<float>(),
                                    ix->stream));
    return search_chunk(ix, nullptr, n, k, D_dev, I_dev, G_dev, 2, nullptr);
}

// ---- query-split sharded search (sharded.py): every rank rotates and assigns ITS SLICE of the batch over ALL lists, the ranks
// exchange one record per query -- [768 f32 rotated query | nprobe i32 lists | nprobe f32 coarse scores] -- and then scan their own
// lists.  Against the list-split coarse quantizer above it removes the replicated rotation and exact re-rank (each done for n / W
// queries instead of n) and the merge of per-shard candidates; it needs the full centroid table on every rank (it is replicated).
__global__ void pack_records_kernel(const float* __restrict__ xr, const int* __restrict__ key, const float* __restrict__ cd, int nprobe, float* __restrict__ rec) {
    const long long q = blockIdx.x;
    const int R = DPH_D + 2 * nprobe;
    float* o = rec + q * R;
    for (int t = threadIdx.x; t < R; t += blockDim.x)
        o[t] = t < DPH_D ? xr[q * DPH_D + t] : (t < DPH_D + nprobe ? __int_as_float(key[q * nprobe + t - DPH_D]) : cd[q * nprobe + t - DPH_D - nprobe]);
}
__global__ void unpack_records_kernel(const float* __restrict__ rec, int nprobe, float* __restrict__ xr, int* __restrict__ key, float* __restrict__ cd) {
    const long long q = blockIdx.x;
    const int R = DPH_D + 2 * nprobe;
    const float* r = rec + q * R;
    for (int t = threadIdx.x; t < R; t += blockDim.x) {
        const float v = r[t];
        if (t < DPH_D) xr[q * DPH_D + t] = v;
        else if (t < DPH_D + nprobe) key[q * nprobe + t - DPH_D] = __float_as_int(v);
        else cd[q * nprobe + t - DPH_D - nprobe] = v;
    }
}
DPH_API int dph_index_record_floats(const dph_index* ix) { return ix->d + 2 * ix->nprobe; }
DPH_API int dph_index_coarse_split(dph_index* ix, const float* x_dev, int64_t n_local, float* rec_dev) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n_local == 0) return 0;
    DPH_CHECK(n_local <= chunk_size(ix, n_local), "coarse_split: slice too large for one chunk");
    DPH_TRY(search_chunk(ix, x_dev, n_local, 1, nullptr, nullptr, nullptr, 3, nullptr));
    pack_records_kernel<<<(unsigned)n_local, 256, 0, ix->stream>>>(ix->xr.as<float>(), ix->key.as<int>(), ix->cd.as<float>(), ix->nprobe, rec_dev);
    DPH_CUDA(cudaGetLastError());
    return 0;
}
DPH_API int dph_index_search_assigned(dph_index* ix, const float* rec_dev, int64_t n, int k, float* D_dev, int64_t* I_dev, uint32_t* G_dev) {
    DPH_TRY(check_ready(ix, k));
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n == 0) return 0;
    DPH_TRY(ix->xr.ensure((size_t)n * ix->d * 4));
    DPH_TRY(ix->key.ensure((size_t)n * ix->nprobe * 4));
    DPH_TRY(ix->cd.ensure((size_t)n * ix->nprobe * 4));
    unpack_records_kernel<<<(unsigned)n, 256, 0, ix->stream>>>(rec_dev, ix->nprobe, ix->xr.as<float>(), ix->key.as<int>(), ix->cd.as<float>());
    DPH_CUDA(cudaGetLastError());
    return search_chunk(ix, nullptr, n, k, D_dev, I_dev, G_dev, 2, nullptr);
}

DPH_API int dph_index_search(dph_index* ix, const float* x, int64_t n, int k, float* D, int64_t* I, int mem) {
    DPH_TRY(check_ready(ix, k));
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n == 0) return 0;
    DPH_TRY(ix->Gp.ensure((size_t)n * k * 4));
    if (mem == DPH_MEM_DEVICE) return dph_index_search_partial(ix, x, n, k, D, I, ix->Gp.as<uint32_t>());
    DPH_TRY(ix->xdev.ensure((size_t)n * ix->d * 4));
    DPH_TRY(ix->Dp.ensure((size_t)n * k * 4));
    DPH_TRY(ix->Ip.ensure((size_t)n * k * 8));
    DPH_CUDA(cudaMemcpyAsync(ix->xdev.p, x, (size_t)n * ix->d * 4, cudaMemcpyHostToDevice, ix->stream));
    DPH_TRY(dph_index_search_partial(ix, ix->xdev.as<float>(), n, k, ix->Dp.as<float>(), ix->Ip.as<int64_t>(), ix->Gp.as<uint32_t>()));
    DPH_CUDA(cudaMemcpyAsync(D, ix->Dp.p, (size_t)n * k * 4, cudaMemcpyDeviceToHost, ix->stream));
    DPH_CUDA(cudaMemcpyAsync(I, ix->Ip.p, (size_t)n * k * 8, cudaMemcpyDeviceToHost, ix->stream));
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
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
