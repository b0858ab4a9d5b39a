// gemm_bf16x3.cu -- fp32-in / fp32-out dense layer on the Hopper tensor cores at bf16 MMA rate with ~2^-17 relative accuracy:
// every fp32 operand x is carried as TWO bf16 planes (hi = bf16(x), lo = bf16(x - hi), x = hi + lo up to 2^-18 |x|) and the kernel
// accumulates  a_hi.b_lo + a_lo.b_hi + a_hi.b_hi  in one fp32 register accumulator (each bf16 x bf16 product is exact in fp32; the
// dropped lo.lo term is 2^-18 relative).  Three bf16 wgmmas cost 1.5 TF32 wgmmas and the operand stream is the same 4 bytes per
// element as fp32, while meeting the 1e-3 tolerance the north star sets for the query vectors (tests/test_encoder.py) -- the
// 3xTF32 kernel (2^-22) needs 3 TF32 wgmmas and twice the operand bytes for that.
//
// Persistent schedule of gemm_wgmma_kernel (gemm_wgmma.cuh): one CTA per SM walks 128 x BN output tiles; a stage is a 32-element
// k block (A_hi, A_lo 128 x 32 and B_hi, B_lo BN x 32 bf16, SWIZZLE_64B); the epilogue writes fp32 rows and/or the (hi, lo) bf16
// planes the NEXT layer consumes.  Reference op: torch.nn.functional.linear inside HF BertModel (densephrases/encoder.py:101-118).
#include "gemm_wgmma.cuh"
#include "../../include/dph_b200.h"

// Tile width BN: 256 by default; 192 when it fills the last wave of the SMs better (N = 768, the attention-output and FFN-output
// projections: at B = 64, S = 64, 2 towers x 32 x 3 = 192 tiles of 128 x 256 fill 132 SMs 1.45 times (73 % of two waves),
// 256 tiles of 128 x 192 fill them 1.94 times (97 %)).
__device__ __forceinline__ void bx_split(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// ---- host side ---------------------------------------------------------------------------------------
int dph_make_map_bf16(CUtensorMap* map, const void* ptr, long long rows, long long cols, long long ld, int box_rows) {
    dph_PFN_encodeTiled enc = nullptr;
    DPH_TRY(dph_tensormap_encoder(&enc));
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    DPH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (bf16) failed");
    return 0;
}

// x fp32 -> (hi, lo) bf16 planes, 8 elements per thread
__global__ void split_bf16_kernel(const float4* __restrict__ x, uint4* __restrict__ hi, uint4* __restrict__ lo, long long n8) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n8) return;
    const float4 a = x[2 * i], b = x[2 * i + 1];
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    __align__(16) __nv_bfloat16 h8[8], l8[8];
#pragma unroll
    for (int e = 0; e < 8; e++) bx_split(v[e], h8[e], l8[e]);
    hi[i] = *reinterpret_cast<const uint4*>(h8);
    lo[i] = *reinterpret_cast<const uint4*>(l8);
}
int dph_launch_split_bf16(const float* x, void* hi, void* lo, long long n, cudaStream_t st) {
    DPH_CHECK(n % 8 == 0, "split_bf16: n must be a multiple of 8");
    if (n == 0) return 0;
    split_bf16_kernel<<<(unsigned)((n / 8 + 255) / 256), 256, 0, st>>>((const float4*)x, (uint4*)hi, (uint4*)lo, n / 8);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

// Grouped launch (the two towers of the encoder): operands as bf16 (hi, lo) planes, device pointers; out (fp32) and/or out_hi/out_lo.
int dph_launch_gemm_bf16x3(int group, const void* const* A_hi, const void* const* A_lo, const void* const* W_hi, const void* const* W_lo,
                           const float* const* bias, const float* const* residual, float* const* out, void* const* out_hi, void* const* out_lo,
                           int M, int N, int K, int act, cudaStream_t st) {
    DPH_CHECK(group >= 1 && group <= GW_MAX_GROUP, "gemm group size");
    DPH_CHECK((N % 256 == 0 || N % 192 == 0) && K % GW_BK == 0 && M >= 1, "gemm_bf16x3 needs N % 256 == 0 (or N % 192 == 0) and K % 32 == 0");
    int dev = 0, num_sms = 0;
    DPH_CUDA(cudaGetDevice(&dev));
    DPH_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    // tile width: the one that wastes less of the last wave (ties -> 256, the higher arithmetic intensity)
    const int tm = (M + GW_BM - 1) / GW_BM;
    auto waste = [&](int bn) { const long long t = (long long)group * tm * (N / bn); const long long w = (t + num_sms - 1) / num_sms; return (double)(w * num_sms) * bn / ((double)t * bn) ; };
    int BN = 256;
    if (N % 256 != 0 || (N % 192 == 0 && waste(192) + 0.2 < waste(256))) BN = 192;
    GwMaps mp;
    GwArgs ap;
    for (int g = 0; g < GW_MAX_GROUP; g++) {
        const int s = g < group ? g : 0;
        DPH_TRY(dph_make_map_bf16(&mp.a[g], A_hi[s], M, K, K, GW_BM));
        DPH_TRY(dph_make_map_bf16(&mp.a2[g], A_lo[s], M, K, K, GW_BM));
        DPH_TRY(dph_make_map_bf16(&mp.b[g], W_hi[s], N, K, K, BN));
        DPH_TRY(dph_make_map_bf16(&mp.b2[g], W_lo[s], N, K, K, BN));
        ap.bias[g] = bias ? bias[s] : nullptr;
        ap.residual[g] = residual ? residual[s] : nullptr;
        ap.out[g] = out ? out[s] : nullptr;
        ap.out_hi[g] = out_hi ? (__nv_bfloat16*)out_hi[s] : nullptr;
        ap.out_lo[g] = out_lo ? (__nv_bfloat16*)out_lo[s] : nullptr;
    }
    ap.M = M; ap.N = N; ap.K = K; ap.act = act;
    ap.tiles_m = tm; ap.tiles_n = N / BN; ap.total_tiles = group * tm * ap.tiles_n;
    const int grid = ap.total_tiles < num_sms ? ap.total_tiles : num_sms;
    if (BN == 256) return gw_launch<GW_BF16X3, 128, 2, 4>(mp, ap, grid, st);
    return gw_launch<GW_BF16X3, 192, 1, 4>(mp, ap, grid, st);
}
