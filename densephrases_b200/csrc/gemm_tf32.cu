// gemm_tf32.cu -- out[g] = epilogue(A[g] . W[g]^T + bias[g] (+ residual[g])) on the Hopper tensor cores.
//
// The dense contractions of the SpanBERT query towers (HF BertModel behind Encoder.embed_query, reference
// densephrases/encoder.py:101-118; QKV / attention-output / FFN projections, SURVEY.md Appendix B).
// fp32 operands in shared memory, wgmma kind tf32 (the precision torch 1.9 -- the reference's pin -- used for fp32 matmuls on
// Ampere+ by default), fp32 accumulators in registers; the kernel itself is gemm_wgmma_kernel (gemm_wgmma.cuh).
//
// Three schedules of the same wgmma sequence (dph_gemm_tf32_set_mode; bit-identical outputs): one 128 x 128 tile per CTA (also
// the 3xTF32 split kernel), the same as 2-CTA clusters sharing the A tile by TMA multicast, and persistent 128 x 256 tiles (default).
#include "gemm_wgmma.cuh"
#include "../../include/dph_b200.h"

// ---- host side ---------------------------------------------------------------------------------------
static dph_PFN_encodeTiled g_encode = nullptr;
int dph_tensormap_encoder(dph_PFN_encodeTiled* out) {
    if (!g_encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        DPH_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        DPH_CHECK(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
        g_encode = (dph_PFN_encodeTiled)fn;
    }
    if (out) *out = g_encode;
    return 0;
}
int dph_make_map_f32(CUtensorMap* map, const float* ptr, long long rows, long long cols, long long ld, int box_rows) {
    DPH_TRY(dph_tensormap_encoder(nullptr));
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    DPH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed");
    return 0;
}
// x -> (hi, lo): hi = round-to-nearest TF32 of x, lo = round-to-nearest TF32 of (x - hi)  (both exact TF32 values)
__global__ void split_tf32_kernel(const float4* __restrict__ x, float4* __restrict__ hi, float4* __restrict__ lo, long long n4) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 v = x[i];
    float4 h, l;
    const float* pv = &v.x; float* ph = &h.x; float* pl = &l.x;
#pragma unroll
    for (int e = 0; e < 4; e++) {
        unsigned hb, lb;
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(pv[e]));
        const float hf = __uint_as_float(hb);
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(pv[e] - hf));
        ph[e] = hf; pl[e] = __uint_as_float(lb);
    }
    hi[i] = h; lo[i] = l;
}
int dph_launch_split_tf32(const float* x, float* hi, float* lo, long long n, cudaStream_t st) {
    DPH_CHECK(n % 4 == 0, "split_tf32: n must be a multiple of 4");
    if (n == 0) return 0;
    split_tf32_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, st>>>((const float4*)x, (float4*)hi, (float4*)lo, n / 4);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

int dph_launch_split_bf16(const float* x, void* hi, void* lo, long long n, cudaStream_t st);                                                  // gemm_bf16x3.cu
int dph_launch_gemm_bf16x3(int group, const void* const* A_hi, const void* const* A_lo, const void* const* W_hi, const void* const* W_lo,
                           const float* const* bias, const float* const* residual, float* const* out, void* const* out_hi, void* const* out_lo,
                           int M, int N, int K, int act, cudaStream_t st);

// how 1xTF32 GEMMs are scheduled: 0 one 128x128 tile per CTA; 1 the same as 2-CTA clusters sharing the A tile by TMA multicast
// (needs an even number of N tiles); 2 persistent 128x256 tiles, one CTA per SM (needs N % 256 == 0)
static int g_gemm_mode = 2;
DPH_API int dph_gemm_tf32_set_mode(int mode) { DPH_CHECK(mode >= 0 && mode <= 2, "gemm mode 0..2"); g_gemm_mode = mode; return 0; }

// Grouped launch used by the encoder: problems share M, N, K and the epilogue; pointers are device pointers.
// A_lo / W_lo non-null -> 3xTF32 mode (A, W are then the hi parts).
int dph_launch_gemm_tf32(int group, const float* const* A, const float* const* W, const float* const* bias, const float* const* residual,
                         float* const* out, int M, int N, int K, int act, cudaStream_t st, const float* const* A_lo, const float* const* W_lo) {
    DPH_CHECK(group >= 1 && group <= GW_MAX_GROUP, "gemm group size");
    DPH_CHECK(N % 128 == 0 && K % GW_BK == 0 && M >= 1, "gemm_tf32 needs N % 128 == 0 and K % 32 == 0");
    const bool split = A_lo != nullptr && W_lo != nullptr;
    const bool persist = !split && g_gemm_mode == 2 && N % 256 == 0;
    const bool cluster = !split && g_gemm_mode == 1 && ((N / 128) % 2 == 0);
    const int BN = persist ? 256 : 128;
    GwMaps maps;
    GwArgs args;
    for (int g = 0; g < GW_MAX_GROUP; g++) {
        const int s = g < group ? g : 0;
        DPH_TRY(dph_make_map_f32(&maps.a[g], A[s], M, K, K, GW_BM));
        DPH_TRY(dph_make_map_f32(&maps.b[g], W[s], N, K, K, BN));
        if (cluster) DPH_TRY(dph_make_map_f32(&maps.a2[g], A[s], M, K, K, GW_BM / 2));
        else DPH_TRY(dph_make_map_f32(&maps.a2[g], split ? A_lo[s] : A[s], M, K, K, GW_BM));
        DPH_TRY(dph_make_map_f32(&maps.b2[g], split ? W_lo[s] : W[s], N, K, K, BN));
        args.bias[g] = bias ? bias[s] : nullptr;
        args.residual[g] = residual ? residual[s] : nullptr;
        args.out[g] = out[s];
        args.out_hi[g] = nullptr; args.out_lo[g] = nullptr;
    }
    args.M = M; args.N = N; args.K = K; args.act = act;
    args.tiles_m = (M + GW_BM - 1) / GW_BM; args.tiles_n = N / BN; args.total_tiles = group * args.tiles_m * args.tiles_n;
    if (split) return gw_launch<GW_TF32X3, 128, 1, 1, 3>(maps, args, args.total_tiles, st);
    if (cluster) return gw_launch<GW_TF32, 128, 1, 2, 4>(maps, args, args.total_tiles, st);
    if (!persist) return gw_launch<GW_TF32, 128, 1, 1, 4>(maps, args, args.total_tiles, st);
    int dev = 0, num_sms = 0;
    DPH_CUDA(cudaGetDevice(&dev));
    DPH_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    return gw_launch<GW_TF32, 128, 2, 1, 4>(maps, args, args.total_tiles < num_sms ? args.total_tiles : num_sms, st);
}

// C ABI (test / standalone use): out [M,N] = act(A [M,K] . W[N,K]^T + bias) + residual, device pointers, fp32 in/out.
// precise = 0: one TF32 MMA per product (operands truncated to 10 mantissa bits); precise = 1: 3xTF32 split (fp32-accurate;
// allocates 2 x (M + N) x K floats of scratch for the split operands).
DPH_API int dph_gemm_tf32_nt(const float* A, const float* W, const float* bias, const float* residual, float* out, int64_t M, int64_t N, int64_t K,
                             int act, int precise, void* cuda_stream) {
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const float* b[1] = {bias}; const float* r[1] = {residual}; float* o[1] = {out};
    if (precise == 2) {                          // bf16x3 (gemm_bf16x3.cu): split both operands into (hi, lo) bf16 planes, N % 256 == 0
        unsigned short* scratch = nullptr;
        const size_t na = (size_t)M * K, nw = (size_t)N * K;
        DPH_CUDA(cudaMalloc((void**)&scratch, (2 * na + 2 * nw) * 2));
        unsigned short *ahi = scratch, *alo = scratch + na, *whi = scratch + 2 * na, *wlo = whi + nw;
        int rc = dph_launch_split_bf16(A, ahi, alo, (long long)na, st);
        if (!rc) rc = dph_launch_split_bf16(W, whi, wlo, (long long)nw, st);
        const void* a1[1] = {ahi}; const void* a2[1] = {alo}; const void* w1[1] = {whi}; const void* w2[1] = {wlo};
        if (!rc) rc = dph_launch_gemm_bf16x3(1, a1, a2, w1, w2, bias ? b : nullptr, residual ? r : nullptr, o, nullptr, nullptr, (int)M, (int)N, (int)K, act, st);
        cudaStreamSynchronize(st);
        cudaFree(scratch);
        return rc;
    }
    if (!precise) {
        const float* a[1] = {A}; const float* w[1] = {W};
        return dph_launch_gemm_tf32(1, a, w, bias ? b : nullptr, residual ? r : nullptr, o, (int)M, (int)N, (int)K, act, st, nullptr, nullptr);
    }
    float* scratch = nullptr;
    const size_t na = (size_t)M * K, nw = (size_t)N * K;
    DPH_CUDA(cudaMalloc((void**)&scratch, (2 * na + 2 * nw) * 4));
    float *ahi = scratch, *alo = scratch + na, *whi = scratch + 2 * na, *wlo = whi + nw;
    int rc = dph_launch_split_tf32(A, ahi, alo, (long long)na, st);
    if (!rc) rc = dph_launch_split_tf32(W, whi, wlo, (long long)nw, st);
    const float* a[1] = {ahi}; const float* w[1] = {whi}; const float* al[1] = {alo}; const float* wl[1] = {wlo};
    if (!rc) rc = dph_launch_gemm_tf32(1, a, w, bias ? b : nullptr, residual ? r : nullptr, o, (int)M, (int)N, (int)K, act, st, al, wl);
    cudaStreamSynchronize(st);
    cudaFree(scratch);
    return rc;
}
