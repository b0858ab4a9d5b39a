// gemm_wgmma.cuh -- out[g] = epilogue(A[g] . W[g]^T + bias[g] (+ residual[g])) on the Hopper tensor cores (wgmma.mma_async),
// shared by the TF32 / 3xTF32 GEMMs (gemm_tf32.cu) and the bf16x3 GEMM (gemm_bf16x3.cu).
//
// A CTA of 384 threads computes 128 x BN output tiles (BN = WN * NSUB): warpgroup 0 is the TMA producer (one thread keeps a
// STAGES-deep ring of 32-element k blocks full, SWIZZLE_128B rows of 32 fp32 or SWIZZLE_64B rows of 32 bf16), warpgroups 1 and 2
// each own 64 rows of the tile and issue m64 x WN wgmmas from shared memory into fp32 register accumulators, then run the epilogue
// (bias / erf-GELU / residual -> fp32 rows and/or the (hi, lo) bf16 planes the next bf16x3 layer consumes) straight from the
// registers.  The producer runs ahead across tile boundaries, so the next tile's operands stream in during the epilogue.
// Every output element sees the same wgmma sequence whatever the schedule (tile per CTA, 2-CTA cluster, persistent), so the
// schedules are bit-identical.
//
// KIND: GW_TF32 one TF32 MMA per product; GW_TF32X3 / GW_BF16X3: each operand arrives as an exact (hi, lo) pair and the kernel
// accumulates hi.lo + lo.hi + hi.hi (small cross terms first) in one fp32 accumulator.
// CL == 2: the two CTAs of a cluster are neighbours along N (same m block): each loads half of the shared A tile and multicasts it
// to both, so a stage may be refilled only when the consumers of BOTH CTAs have released it (empty barriers count 2 x CL arrivals).
#pragma once
#include "wgmma.cuh"
#include <cuda_bf16.h>

#define GW_BM 128
#define GW_BK 32
#define GW_MAX_GROUP 2
#define GW_THREADS 384
enum { GW_TF32 = 0, GW_TF32X3 = 1, GW_BF16X3 = 2 };

// a2 / b2: the lo planes (split kinds); in the cluster variant a2 is A with a 64-row box
struct GwMaps { CUtensorMap a[GW_MAX_GROUP], b[GW_MAX_GROUP], a2[GW_MAX_GROUP], b2[GW_MAX_GROUP]; };
struct GwArgs {
    const float* bias[GW_MAX_GROUP]; const float* residual[GW_MAX_GROUP];
    float* out[GW_MAX_GROUP];                       // fp32 result (nullable)
    __nv_bfloat16* out_hi[GW_MAX_GROUP];            // (hi, lo) bf16 planes of the result (nullable)
    __nv_bfloat16* out_lo[GW_MAX_GROUP];
    int M, N, K, act;                               // act: 0 none, 1 erf-GELU
    int tiles_m, tiles_n, total_tiles;              // tile t: group t / (tiles_m tiles_n), then m block, n block (n fastest)
};

template <int KIND, int WN, int NSUB, int STAGES>
struct GwCfg {
    static constexpr int EB = KIND == GW_BF16X3 ? 2 : 4;        // operand element bytes
    static constexpr int BN = WN * NSUB;
    static constexpr int ROWB = GW_BK * EB;                     // bytes of one k-block row: 128 (fp32) or 64 (bf16)
    static constexpr int A_BYTES = GW_BM * ROWB;
    static constexpr int B_BYTES = BN * ROWB;
    static constexpr int PLANES = KIND == GW_TF32 ? 1 : 2;
    static constexpr int STAGE_BYTES = PLANES * (A_BYTES + B_BYTES);   // [A_hi | B_hi | A_lo | B_lo]
    static constexpr int SMEM = STAGES * STAGE_BYTES + 256 + 1024;     // + barriers + alignment slack
};

template <int KIND, int WN>
__device__ __forceinline__ void gw_mma(float (&d)[WN / 2], unsigned long long a, unsigned long long b, int acc) {
    if (KIND == GW_BF16X3) wgmma_bf16<WN>(d, a, b, acc);
    else wgmma_tf32<WN>(d, a, b, acc);
}

template <int KIND, int WN, int NSUB, int CL, int STAGES>
__global__ void __launch_bounds__(GW_THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ GwMaps maps, const GwArgs args) {
    using C = GwCfg<KIND, WN, NSUB, STAGES>;
    static_assert(CL == 1 || KIND == GW_TF32, "cluster variant: 1xTF32 only");
    constexpr int KSTEP_BYTES = 32;                                 // k = 8 tf32 or 16 bf16 per wgmma
    extern __shared__ unsigned char gw_raw[];
    unsigned char* gsm = (unsigned char*)((((unsigned long long)gw_raw) + 1023ull) & ~1023ull);   // swizzle atoms: 1024-byte aligned
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(gsm + STAGES * C::STAGE_BYTES);     // full[STAGES], empty[STAGES]
    const unsigned full0 = smem_u32(bars), empty0 = smem_u32(bars + STAGES), stage0 = smem_u32(gsm);
    const int tid = threadIdx.x, wg = tid >> 7;
    const int num_k = args.K / GW_BK;
    const int per_group = args.tiles_m * args.tiles_n;

    if (tid == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 2 * CL); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    unsigned crank = 0;
    if (CL == 2) { crank = cluster_ctarank(); cluster_sync_all(); }      // the peer's barriers are initialised before anything signals them

    if (wg == 0) {
        if (tid == 0) {
            unsigned it = 0;
            for (int t = blockIdx.x; t < args.total_tiles; t += gridDim.x) {
                const int g = t / per_group, r = t - g * per_group, m_blk = r / args.tiles_n, n_blk = r - m_blk * args.tiles_n;
                for (int kb = 0; kb < num_k; kb++, it++) {
                    const unsigned s = it % STAGES, ph = (it / STAGES) & 1u;
                    mbar_wait(empty0 + 8 * s, ph ^ 1u);
                    mbar_expect_tx(full0 + 8 * s, C::STAGE_BYTES);
                    const unsigned dst = stage0 + s * C::STAGE_BYTES, full = full0 + 8 * s;
                    if (CL == 2) tma_load_2d_mc(dst + crank * (C::A_BYTES / 2), &maps.a2[g], kb * GW_BK, m_blk * GW_BM + (int)crank * (GW_BM / 2), full, (unsigned short)3);
                    else tma_load_2d(dst, &maps.a[g], kb * GW_BK, m_blk * GW_BM, full);
                    tma_load_2d(dst + C::A_BYTES, &maps.b[g], kb * GW_BK, n_blk * C::BN, full);
                    if (C::PLANES == 2) {
                        tma_load_2d(dst + C::A_BYTES + C::B_BYTES, &maps.a2[g], kb * GW_BK, m_blk * GW_BM, full);
                        tma_load_2d(dst + 2 * C::A_BYTES + C::B_BYTES, &maps.b2[g], kb * GW_BK, n_blk * C::BN, full);
                    }
                }
            }
        }
    } else {
        const int cw = wg - 1;                                       // rows 64 cw .. 64 cw + 63 of the tile
        const int warp = (tid >> 5) & 3, lane = tid & 31;
        const bool leader = (tid & 127) == 0;
        auto release = [&](unsigned s) {
            if (!leader) return;
            if (CL == 2) { mbar_arrive_cluster(empty0 + 8 * s, 0); mbar_arrive_cluster(empty0 + 8 * s, 1); }
            else mbar_arrive(empty0 + 8 * s);
        };
        float acc[NSUB][WN / 2];
        unsigned it = 0;
        for (int t = blockIdx.x; t < args.total_tiles; t += gridDim.x) {
            const int g = t / per_group, r = t - g * per_group, m_blk = r / args.tiles_n, n_blk = r - m_blk * args.tiles_n;
#pragma unroll
            for (int u = 0; u < NSUB; u++) wgmma_fence_acc(acc[u]);
            for (int kb = 0; kb < num_k; kb++, it++) {
                const unsigned s = it % STAGES, ph = (it / STAGES) & 1u;
                mbar_wait(full0 + 8 * s, ph);
                const unsigned base = stage0 + s * C::STAGE_BYTES;
                const unsigned a_hi = base + cw * 64 * C::ROWB, b_hi = base + C::A_BYTES;
                const unsigned a_lo = a_hi + C::A_BYTES + C::B_BYTES, b_lo = b_hi + C::A_BYTES + C::B_BYTES;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < C::ROWB / KSTEP_BYTES; k++) {
#pragma unroll
                    for (int u = 0; u < NSUB; u++) {
                        const unsigned ko = k * KSTEP_BYTES, bo = u * WN * C::ROWB + ko;
                        const unsigned long long ah = C::ROWB == 128 ? make_sw128_desc(a_hi + ko) : make_sw64_desc(a_hi + ko);
                        const unsigned long long bh = C::ROWB == 128 ? make_sw128_desc(b_hi + bo) : make_sw64_desc(b_hi + bo);
                        const int first = (kb | k) ? 1 : 0;
                        if (C::PLANES == 2) {
                            const unsigned long long al = C::ROWB == 128 ? make_sw128_desc(a_lo + ko) : make_sw64_desc(a_lo + ko);
                            const unsigned long long bl = C::ROWB == 128 ? make_sw128_desc(b_lo + bo) : make_sw64_desc(b_lo + bo);
                            gw_mma<KIND, WN>(acc[u], ah, bl, first);      // small cross terms first, then hi.hi
                            gw_mma<KIND, WN>(acc[u], al, bh, 1);
                            gw_mma<KIND, WN>(acc[u], ah, bh, 1);
                        } else {
                            gw_mma<KIND, WN>(acc[u], ah, bh, first);
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();                                     // the previous k block's wgmmas are done: free its stage
                if (kb > 0) release((it - 1) % STAGES);
            }
            wgmma_wait<0>();
            release((it - 1) % STAGES);
#pragma unroll
            for (int u = 0; u < NSUB; u++) wgmma_fence_acc(acc[u]);

            const float* bias = args.bias[g];
            const float* resid = args.residual[g];
            float* out = args.out[g];
            __nv_bfloat16* ohi = args.out_hi[g];
            __nv_bfloat16* olo = args.out_lo[g];
            const long long row0 = (long long)m_blk * GW_BM + cw * 64 + warp * 16 + (lane >> 2);
#pragma unroll
            for (int u = 0; u < NSUB; u++) {
#pragma unroll
                for (int j = 0; j < WN / 8; j++) {
                    const int col = n_blk * C::BN + u * WN + j * 8 + 2 * (lane & 3);
                    const float2 b2 = bias ? *reinterpret_cast<const float2*>(bias + col) : make_float2(0.f, 0.f);
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const long long row = row0 + 8 * h;
                        if (row >= args.M) continue;
                        float x0 = acc[u][4 * j + 2 * h] + b2.x, x1 = acc[u][4 * j + 2 * h + 1] + b2.y;
                        if (args.act == 1) {
                            x0 = 0.5f * x0 * (1.0f + erff(x0 * 0.70710678118654752440f));
                            x1 = 0.5f * x1 * (1.0f + erff(x1 * 0.70710678118654752440f));
                        }
                        if (resid) { const float2 r2 = *reinterpret_cast<const float2*>(resid + row * args.N + col); x0 += r2.x; x1 += r2.y; }
                        if (out) *reinterpret_cast<float2*>(out + row * args.N + col) = make_float2(x0, x1);
                        if (ohi) {
                            const __nv_bfloat162 hv = __floats2bfloat162_rn(x0, x1);
                            const float2 hf = __bfloat1622float2(hv);
                            *reinterpret_cast<__nv_bfloat162*>(ohi + row * args.N + col) = hv;
                            *reinterpret_cast<__nv_bfloat162*>(olo + row * args.N + col) = __floats2bfloat162_rn(x0 - hf.x, x1 - hf.y);
                        }
                    }
                }
            }
        }
    }
    if (CL == 2) cluster_sync_all();       // the peer may still multicast into this CTA's shared memory / signal its barriers
}

// Launch with `grid` CTAs (grid < total_tiles: persistent); CL == 2 launches clusters of two CTAs along x.
template <int KIND, int WN, int NSUB, int CL, int STAGES>
static int gw_launch(const GwMaps& maps, const GwArgs& args, int grid, cudaStream_t st) {
    auto kern = gemm_wgmma_kernel<KIND, WN, NSUB, CL, STAGES>;
    constexpr int smem = GwCfg<KIND, WN, NSUB, STAGES>::SMEM;
    static DphPerDeviceOnce once;
    if (once.first()) DPH_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if (CL == 1) {
        kern<<<grid, GW_THREADS, smem, st>>>(maps, args);
    } else {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(GW_THREADS); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        DPH_CUDA(cudaLaunchKernelEx(&cfg, kern, maps, args));
    }
    DPH_CUDA(cudaGetLastError());
    return 0;
}
