// encode.cu -- assignment + PQ encoding of new vectors: faiss IndexPreTransform(OPQ) -> IndexIVFPQ::add_with_ids (by_residual),
// reference build_phrase_index.py:145-150,156-279, bit-identical to oracle/encode_ref.c:ref_encode (DESIGN.md 3, "Growing the index"):
//   xr = x A^T (sequential-k SGEMM), list = top-1 of the coarse quantizer (the search's coarse path with nprobe = 1: same scores, same
//   tie rule), r = xr - C[list] (fp32), dist[m][j] = fmaf chain over the 8 squared differences, code[m] = argmin_j (lowest j on ties).
#include "index_internal.cuh"
#include <algorithm>
#include <stdlib.h>

#define ENC_TILE 128           // vectors per CTA, one per thread
#define ENC_CB_FLOATS (DPH_KSUB * DPH_DSUB)   // one sub-quantizer's codebook: 256 x 8 fp32 = 8 KB
#define ENC_ROW_LD 97          // shared code tile row pitch (odd: the byte writes of one warp spread over the banks)

__device__ __forceinline__ void enc_stage_codebook(float* dst, const float* src) {
    const unsigned base = (unsigned)__cvta_generic_to_shared(dst);
    for (int i = threadIdx.x; i < ENC_CB_FLOATS / 4; i += ENC_TILE)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(base + i * 16), "l"(src + i * 4));
    asm volatile("cp.async.commit_group;\n" ::);
}

// grid (ceil(n / ENC_TILE), msplit): CTA (tile, s) encodes sub-quantizers [s * 96 / msplit, (s + 1) * 96 / msplit) of ENC_TILE vectors.
// Per sub-quantizer the 8 KB codebook is staged in shared memory (cp.async, double-buffered: the next one loads during this one's
// scan) and read as warp-wide broadcasts; each thread keeps its vector's 8 residual values in registers and scans j = 0..255 with a
// running strict-< minimum, i.e. the argmin over (dist, j) of the oracle, with no cross-thread reduction.  The scan is bound by
// the fp32 pipe: 8 FSUB + 8 FFMA per (vector, m, j).
__global__ void __launch_bounds__(ENC_TILE) pq_encode_kernel(const float* __restrict__ xr, const float* __restrict__ C, const float* __restrict__ pq,
                                                             const int* __restrict__ key, long long n, int msplit, long long* __restrict__ list_out,
                                                             uint8_t* __restrict__ codes_out) {
    __shared__ __align__(16) float cb[2][ENC_CB_FLOATS];
    __shared__ uint8_t sc[ENC_TILE * ENC_ROW_LD];
    const int tid = threadIdx.x;
    const long long v0 = (long long)blockIdx.x * ENC_TILE, v = v0 + tid;
    const int mcount = DPH_M / msplit, m0 = blockIdx.y * mcount;
    const long long l = v < n ? (long long)key[v] : -1;
    if (blockIdx.y == 0 && v < n) list_out[v] = l;
    enc_stage_codebook(cb[0], pq + (size_t)m0 * ENC_CB_FLOATS);
    for (int mi = 0; mi < mcount; mi++) {
        if (mi + 1 < mcount) enc_stage_codebook(cb[(mi + 1) & 1], pq + (size_t)(m0 + mi + 1) * ENC_CB_FLOATS);
        else asm volatile("cp.async.commit_group;\n" ::);              // keep one group per iteration: wait_group 1 = "this m's codebook"
        asm volatile("cp.async.wait_group 1;\n" ::);
        __syncthreads();
        int bj = 0;
        if (l >= 0) {
            const int m = m0 + mi;
            const float4* xp = reinterpret_cast<const float4*>(xr + v * DPH_D + m * DPH_DSUB);
            const float4* cp = reinterpret_cast<const float4*>(C + l * DPH_D + m * DPH_DSUB);
            const float4 x0 = xp[0], x1 = xp[1], c0 = cp[0], c1 = cp[1];
            const float r0 = __fsub_rn(x0.x, c0.x), r1 = __fsub_rn(x0.y, c0.y), r2 = __fsub_rn(x0.z, c0.z), r3 = __fsub_rn(x0.w, c0.w);
            const float r4 = __fsub_rn(x1.x, c1.x), r5 = __fsub_rn(x1.y, c1.y), r6 = __fsub_rn(x1.z, c1.z), r7 = __fsub_rn(x1.w, c1.w);
            const float4* w = reinterpret_cast<const float4*>(cb[mi & 1]);
            float best = __int_as_float(0x7f800000);                     // +inf
#pragma unroll 4
            for (int j = 0; j < DPH_KSUB; j++) {
                const float4 a = w[2 * j], b = w[2 * j + 1];
                float acc = 0.0f, d;
                d = __fsub_rn(r0, a.x); acc = fmaf(d, d, acc);
                d = __fsub_rn(r1, a.y); acc = fmaf(d, d, acc);
                d = __fsub_rn(r2, a.z); acc = fmaf(d, d, acc);
                d = __fsub_rn(r3, a.w); acc = fmaf(d, d, acc);
                d = __fsub_rn(r4, b.x); acc = fmaf(d, d, acc);
                d = __fsub_rn(r5, b.y); acc = fmaf(d, d, acc);
                d = __fsub_rn(r6, b.z); acc = fmaf(d, d, acc);
                d = __fsub_rn(r7, b.w); acc = fmaf(d, d, acc);
                if (acc < best) { best = acc; bj = j; }
            }
        }
        sc[tid * ENC_ROW_LD + mi] = (uint8_t)bj;
        __syncthreads();                                                 // the buffer is refilled by the next iteration's stage
    }
    asm volatile("cp.async.wait_group 0;\n" ::);
    // coalesced write of the tile's code bytes [v0, v0 + ENC_TILE) x [m0, m0 + mcount)
    for (int i = tid; i < ENC_TILE * mcount; i += ENC_TILE) {
        const int row = i / mcount, col = i - row * mcount;
        if (v0 + row < n) codes_out[(v0 + row) * DPH_M + m0 + col] = sc[row * ENC_ROW_LD + col];
    }
}

__global__ void nonfinite_kernel(const float* __restrict__ x, long long count, int* __restrict__ bad) {
    int hit = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
        hit |= !isfinite(x[i]);
    if (__syncthreads_or(hit) && threadIdx.x == 0) atomicOr(bad, 1);
}

int64_t dph_encode_chunk(const dph_index* ix) {
    const int64_t nlp = (ix->nlist + 127) / 128 * 128;
    int64_t c = std::min<int64_t>((1ll << 28) / nlp, 65536);           // coarse scores S [c, nlist] <= 1 GiB, as for search
    if (const char* ev = getenv("DPH_UPLOAD_CHUNK_ROWS")) c = std::min<int64_t>(c, atoll(ev));      // tests: force several chunks
    return std::max<int64_t>(c, 1);
}

int dph_coarse_top1(dph_index* ix, const float* xr, const float* C, int64_t n, int32_t* key, float* cd, cudaStream_t st) {
    const int rc = ix->coarse_tc ? dph_coarse_tc(ix, n, 0, ix->nlist, 1, nullptr, key, cd, st, xr, C) : 1;
    if (rc > 1) return rc;
    if (rc == 1) {
        DPH_TRY(dph_launch_sgemm_nt_seq(xr, n, C, ix->nlist, ix->d, ix->S.as<float>(), st));
        DPH_TRY(dph_launch_coarse_select(ix->S.as<float>(), n, ix->nlist, 1, key, cd, st, nullptr, 0u, nullptr, 0, &ix->selkeys));
    }
    return 0;
}

int dph_pq_assign(dph_index* ix, const float* xr, const float* C, const int32_t* key, const float* pq, int64_t n, int64_t* list_out,
                  uint8_t* codes_out, cudaStream_t st) {
    const int64_t tiles = (n + ENC_TILE - 1) / ENC_TILE;
    int msplit = 1;                                                       // enough CTAs for two waves; msplit divides 96
    while (msplit < 32 && tiles * msplit < 2 * ix->num_sms) msplit *= 2;
    pq_encode_kernel<<<dim3((unsigned)tiles, (unsigned)msplit), ENC_TILE, 0, st>>>(xr, C, pq, key, n, msplit, (long long*)list_out, codes_out);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

static int encode_rows_chunk(dph_index* ix, const float* x, int64_t n, int64_t* list_out, uint8_t* codes_out, int* bad) {
    cudaStream_t st = ix->stream;
    const bool prof = ix->profile && ix->aev[0];
    if (bad) {
        nonfinite_kernel<<<(unsigned)std::min<int64_t>((n * DPH_D + 255) / 256, 4 * ix->num_sms), 256, 0, st>>>(x, n * DPH_D, bad);
        DPH_CUDA(cudaGetLastError());
    }
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[0], st));
    DPH_TRY(dph_launch_sgemm_nt_seq(x, n, ix->A, ix->d, ix->d, ix->xr.as<float>(), st));                      // OPQ rotation
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[1], st));
    int32_t* key = ix->enc_key.as<int32_t>(); float* cd = ix->enc_cd.as<float>();
    DPH_TRY(dph_coarse_top1(ix, ix->xr.as<float>(), ix->C, n, key, cd, st));
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[2], st));
    DPH_TRY(dph_pq_assign(ix, ix->xr.as<float>(), ix->C, key, ix->pq, n, list_out, codes_out, st));
    DPH_CUDA(cudaGetLastError());
    if (prof) {
        DPH_CUDA(cudaEventRecord(ix->aev[3], st));
        DPH_CUDA(cudaEventSynchronize(ix->aev[3]));
        for (int s = 0; s < 3; s++) { float ms = 0.f; DPH_CUDA(cudaEventElapsedTime(&ms, ix->aev[s], ix->aev[s + 1])); ix->add_ms[s] += ms; }
    }
    return 0;
}

// Assign + encode x [n, d] (device) -> list_out [n] int64, codes_out [n, 96] (device), asynchronously on the index stream, in chunks
// of dph_encode_chunk rows.  bad (device int, optional): OR-ed with 1 when an input element is not finite.  Uses the search workspace
// xr / S (dph_index_last_xr is not preserved); the probes of the last search are.
int dph_encode_rows(dph_index* ix, const float* x, int64_t n, int64_t* list_out, uint8_t* codes_out, int* bad) {
    DPH_CHECK(ix->A && ix->C && ix->pq, "encode: OPQ matrix, centroids and PQ codebooks must be set");
    const int64_t cs = std::min(dph_encode_chunk(ix), n);
    if (n == 0) return 0;
    const int64_t nlp = (ix->nlist + 127) / 128 * 128;
    DPH_TRY(ix->xr.ensure((size_t)cs * ix->d * 4));
    DPH_TRY(ix->S.ensure((size_t)cs * nlp * 4));
    DPH_TRY(ix->enc_key.ensure((size_t)cs * 4));
    DPH_TRY(ix->enc_cd.ensure((size_t)cs * 4));
    for (int64_t o = 0; o < n; o += cs) {
        const int64_t m = std::min(cs, n - o);
        DPH_TRY(encode_rows_chunk(ix, x + o * ix->d, m, list_out + o, codes_out + o * DPH_M, bad));
    }
    return 0;
}

DPH_API int dph_index_encode(dph_index* ix, const float* x, int64_t n, int64_t* list_no_out, uint8_t* codes_out, int mem) {
    DPH_CHECK(ix != nullptr && n >= 0, "encode: bad arguments");
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n == 0) return 0;
    if (mem == DPH_MEM_DEVICE) return dph_encode_rows(ix, x, n, list_no_out, codes_out, nullptr);
    // host buffers: bounded staging, one chunk at a time (stream order keeps the staging buffers' reuse safe)
    const int64_t cs = std::min(dph_encode_chunk(ix), n);
    DPH_TRY(ix->xdev.ensure((size_t)cs * ix->d * 4));
    DPH_TRY(ix->enc_list.ensure((size_t)cs * 8));
    DPH_TRY(ix->enc_codes.ensure((size_t)cs * DPH_M));
    for (int64_t o = 0; o < n; o += cs) {
        const int64_t m = std::min(cs, n - o);
        DPH_CUDA(cudaMemcpyAsync(ix->xdev.p, x + o * ix->d, (size_t)m * ix->d * 4, cudaMemcpyHostToDevice, ix->stream));
        DPH_TRY(dph_encode_rows(ix, ix->xdev.as<float>(), m, ix->enc_list.as<int64_t>(), ix->enc_codes.as<uint8_t>(), nullptr));
        DPH_CUDA(cudaMemcpyAsync(list_no_out + o, ix->enc_list.p, (size_t)m * 8, cudaMemcpyDeviceToHost, ix->stream));
        DPH_CUDA(cudaMemcpyAsync(codes_out + o * DPH_M, ix->enc_codes.p, (size_t)m * DPH_M, cudaMemcpyDeviceToHost, ix->stream));
    }
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    return 0;
}
