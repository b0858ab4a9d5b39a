// tools/lds_bench.cu -- microbenchmark: what shared-memory gather rate can one SM sustain on H100?
// (design input for scan.cu:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o lds_bench tools/lds_bench.cu && ./lds_bench)
#define NSM 132            // SMs of an H100 SXM: one CTA per SM
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
extern __shared__ __align__(1024) unsigned char dsm[];
template <int IMM> __device__ __forceinline__ float lds_imm(unsigned addr) {
    float v; asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(IMM)); return v;
}
#ifndef VARIANT
#define VARIANT 0
#endif
__device__ __forceinline__ void accum(float& a, float v) {
#if VARIANT == 1 || VARIANT == 4
    asm volatile("fma.rn.f32 %0, %1, 0f3F800000, %0;" : "+f"(a) : "f"(v));
#else
    a += v;
#endif
}
template <int T0> __device__ __forceinline__ void word4(unsigned wv, unsigned y, float& a0, float& a1, float& a2, float& a3) {
    constexpr int TB = 0x400 + (T0 >> 5) * 65536 + (T0 & 31) * 4;
#if VARIANT == 2
    accum(a0, lds_imm<TB + 0>(y + (wv & 0xff00))); accum(a1, lds_imm<TB + 4>(y + (wv & 0xff00))); accum(a2, lds_imm<TB + 8>(y + (wv & 0xff00))); accum(a3, lds_imm<TB + 12>(y + (wv & 0xff00)));
#elif VARIANT == 3 || VARIANT == 4
    // IMAD-based (fma pipe) byte extraction for 2 of 4 bytes: (wv >> 16) & 0xff00 etc. -- mix pipes
    accum(a0, lds_imm<TB + 0>(__byte_perm(wv, y, 0x7504)));
    accum(a1, lds_imm<TB + 4>((wv & 0xff00u) | y));
    accum(a2, lds_imm<TB + 8>(__byte_perm(wv, y, 0x7524)));
    accum(a3, lds_imm<TB + 12>(((wv >> 16) & 0xff00u) | y));
#else
    accum(a0, lds_imm<TB + 0>(__byte_perm(wv, y, 0x7504)));
    accum(a1, lds_imm<TB + 4>(__byte_perm(wv, y, 0x7514)));
    accum(a2, lds_imm<TB + 8>(__byte_perm(wv, y, 0x7524)));
    accum(a3, lds_imm<TB + 12>(__byte_perm(wv, y, 0x7534)));
#endif
}
template <int C> __device__ __forceinline__ void chunk(const uint4& v, unsigned y, float& a0, float& a1, float& a2, float& a3) {
    word4<C * 16 + 0>(v.x, y, a0, a1, a2, a3); word4<C * 16 + 4>(v.y, y, a0, a1, a2, a3);
    word4<C * 16 + 8>(v.z, y, a0, a1, a2, a3); word4<C * 16 + 12>(v.w, y, a0, a1, a2, a3);
}
// MODE 0: PRMT+LDS+FADD on register-resident "codes" (no global traffic).  MODE 1: same, codes re-derived each iter by xor (keeps PRMT live)
template <int MODE>
__global__ void __launch_bounds__(1024, 1) k_gather(float* out, int iters, long long* cyc) {
    for (int i = threadIdx.x; i < 49152; i += blockDim.x) ((float*)dsm)[i] = (float)(i & 1023) * 1e-3f;
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    const unsigned y = (((unsigned)__cvta_generic_to_shared(dsm)) & 0xFF000000u) | (lane * 4u);
    uint4 c[6];
    unsigned s = threadIdx.x * 2654435761u + blockIdx.x;
    for (int i = 0; i < 6; i++) { s = s * 1664525u + 1013904223u; c[i].x = s; s = s * 1664525u + 1013904223u; c[i].y = s; s = s * 1664525u + 1013904223u; c[i].z = s; s = s * 1664525u + 1013904223u; c[i].w = s; }
    float a0 = 0, a1 = 0, a2 = 0, a3 = 0;
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        chunk<0>(c[0], y, a0, a1, a2, a3); chunk<1>(c[1], y, a0, a1, a2, a3); chunk<2>(c[2], y, a0, a1, a2, a3);
        chunk<3>(c[3], y, a0, a1, a2, a3); chunk<4>(c[4], y, a0, a1, a2, a3); chunk<5>(c[5], y, a0, a1, a2, a3);
        if (MODE == 1) { for (int i = 0; i < 6; i++) { c[i].x ^= __float_as_uint(a0) & 0x01010101u; c[i].y += 0x01010101u; c[i].z ^= 0x10101010u; c[i].w += 0x02020202u; } }
    }
    long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
template <int W, int U> __device__ __forceinline__ void pure_step(unsigned base, float& acc) {
    if constexpr (U < 32) {
        if constexpr (W == 4) { float v; asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(base), "n"(U * 512)); acc += v; }
        if constexpr (W == 8) { float v, w; asm volatile("ld.shared.v2.f32 {%0,%1}, [%2+%3];" : "=f"(v), "=f"(w) : "r"(base), "n"(U * 512)); acc += v + w; }
        if constexpr (W == 16) { float v, w, x, z; asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4+%5];" : "=f"(v), "=f"(w), "=f"(x), "=f"(z) : "r"(base), "n"(U * 512)); acc += (v + w) + (x + z); }
        pure_step<W, U + 1>(base, acc);
    }
}
// gather + streaming global loads (6 x LDG.128 per lane per 96 gathers, 1-ahead register prefetch), like scan.cu
template <int LDMODE, int PD>
__global__ void __launch_bounds__(512, 1) k_stream(float* out, int iters, long long* cyc, const uint4* gbuf, long long nblk) {
    for (int i = threadIdx.x; i < 49152; i += blockDim.x) ((float*)dsm)[i] = (float)(i & 1023) * 1e-3f;
    __syncthreads();
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const unsigned y = (((unsigned)__cvta_generic_to_shared(dsm)) & 0xFF000000u) | (lane * 4u);
    float a0 = 0, a1 = 0, a2 = 0, a3 = 0;
    long long blk = ((long long)blockIdx.x * iters) * nw + warp;   // contiguous region per CTA
    uint4 nxt[6], cur[6];
    auto ld = [&](const uint4* p) {
        uint4 r;
        if (LDMODE != 1) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
        else asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
        return r; };
    for (int c = 0; c < 6; c++) nxt[c] = ld(gbuf + (blk % nblk) * 192 + c * 32 + lane);
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        for (int c = 0; c < 6; c++) cur[c] = nxt[c];
        blk += nw;
        if (LDMODE != 2) { for (int c = 0; c < 6; c++) nxt[c] = ld(gbuf + (blk % nblk) * 192 + c * 32 + lane); }
        else { for (int c = 0; c < 6; c++) { nxt[c].x ^= cur[c].y; nxt[c].y += 0x01010101u; nxt[c].z ^= 0x10101010u; nxt[c].w += 0x02020202u; } }
        if (LDMODE == 3 && lane == 0) asm volatile("cp.async.bulk.prefetch.L2.global [%0], 3072;" :: "l"(gbuf + ((blk + PD * nw) % nblk) * 192) : "memory");
        if (LDMODE == 4 && lane < 24) asm volatile("prefetch.global.L2 [%0];" :: "l"(gbuf + ((blk + PD * nw) % nblk) * 192 + lane * 8) : "memory");
        if (LDMODE == 5 && lane < 12) asm volatile("prefetch.global.L2::evict_last [%0];" :: "l"(gbuf + ((blk + PD * nw) % nblk) * 192 + lane * 16) : "memory");
        if (LDMODE == 6 && warp == 0 && lane == 0) asm volatile("cp.async.bulk.prefetch.L2.global [%0], 49152;" :: "l"(gbuf + ((blk + PD * nw) % nblk) * 192) : "memory");
        chunk<0>(cur[0], y, a0, a1, a2, a3); chunk<1>(cur[1], y, a0, a1, a2, a3); chunk<2>(cur[2], y, a0, a1, a2, a3);
        chunk<3>(cur[3], y, a0, a1, a2, a3); chunk<4>(cur[4], y, a0, a1, a2, a3); chunk<5>(cur[5], y, a0, a1, a2, a3);
    }
    long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
template <class K> void run_stream(const char* name, K kern, int nthreads, int iters, const uint4* gbuf, long long nblk) {
    const int smem = 200 * 1024;
    float* out; long long* cyc; cudaMalloc(&out, NSM * 1024 * 4); cudaMalloc(&cyc, NSM * 8);
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    kern<<<NSM, nthreads, smem>>>(out, 10, cyc, gbuf, nblk);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0); kern<<<NSM, nthreads, smem>>>(out, iters, cyc, gbuf, nblk); cudaEventRecord(e1); cudaDeviceSynchronize();
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    long long h[NSM]; cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    double avg = 0; for (int i = 0; i < NSM; i++) avg += h[i]; avg /= NSM;
    double lookups = 96.0 * iters * nthreads;
    double gbs = (double)NSM * iters * (nthreads / 32) * 3072.0 / (ms * 1e-3) / 1e9;
    printf("%-34s threads=%4d  warp-gathers/clk/SM=%.3f  %.0f GB/s (cycles %.0f, %.3f ms, err=%s)\n", name, nthreads, lookups / 32.0 / avg, gbs, avg, ms, cudaGetErrorString(cudaGetLastError()));
    cudaFree(out); cudaFree(cyc);
}
// pure LDS with fixed per-lane address (+imm), W bytes per access
template <int W>
__global__ void __launch_bounds__(1024, 1) k_pure(float* out, int iters, long long* cyc) {
    for (int i = threadIdx.x; i < 49152; i += blockDim.x) ((float*)dsm)[i] = (float)(i & 1023) * 1e-3f;
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    unsigned base = (unsigned)__cvta_generic_to_shared(dsm) + lane * W + (threadIdx.x >> 5) * 1024;
    float acc = 0;
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        pure_step<W, 0>(base, acc);
        base ^= (it & 1) << 4;
    }
    long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
template <class K> void run(const char* name, K kern, int nthreads, int iters, double per_iter_lookups_per_thread, int smem) {
    float* out; long long* cyc; cudaMalloc(&out, NSM * 1024 * 4); cudaMalloc(&cyc, NSM * 8);
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    kern<<<NSM, nthreads, smem>>>(out, 10, cyc);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0); kern<<<NSM, nthreads, smem>>>(out, iters, cyc); cudaEventRecord(e1); cudaDeviceSynchronize();
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    long long h[NSM]; cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    double avg = 0; for (int i = 0; i < NSM; i++) avg += h[i]; avg /= NSM;
    double lookups = per_iter_lookups_per_thread * iters * nthreads;
    printf("%-28s threads=%4d  warp-gathers/clk/SM=%.3f  (cycles %.0f, %.3f ms, err=%s)\n", name, nthreads, lookups / 32.0 / avg, avg, ms, cudaGetErrorString(cudaGetLastError()));
    cudaFree(out); cudaFree(cyc);
}
int main() {
    const int SM = 200 * 1024;
    printf("VARIANT %d\n", VARIANT);
    for (int nt : {256, 512, 1024}) run("gather (live codes)", k_gather<1>, nt, 400, 96, SM);
#if VARIANT != 0
    return 0;
#endif
    {
        long long nblk = 3000000;   // 9.2 GB
        uint4* g; cudaMalloc(&g, nblk * 3072); cudaMemset(g, 0x5a, nblk * 3072);
        for (int nt : {512}) {
            run_stream("stream LDG.128 no_allocate", k_stream<0, 0>, nt, 1200, g, nblk);
            run_stream("no global loads (alu only)", k_stream<2, 0>, nt, 1200, g, nblk);
            run_stream("bulk L2 prefetch 3KB/warp, PD=2", k_stream<3, 2>, nt, 1200, g, nblk);
            run_stream("bulk L2 prefetch 3KB/warp, PD=4", k_stream<3, 4>, nt, 1200, g, nblk);
            run_stream("bulk L2 prefetch 3KB/warp, PD=8", k_stream<3, 8>, nt, 1200, g, nblk);
            run_stream("bulk L2 prefetch 3KB/warp, PD=16", k_stream<3, 16>, nt, 1200, g, nblk);
            run_stream("prefetch.global.L2 x24 lanes, PD=4", k_stream<4, 4>, nt, 1200, g, nblk);
            run_stream("prefetch.global.L2 x24 lanes, PD=8", k_stream<4, 8>, nt, 1200, g, nblk);
            run_stream("bulk L2 prefetch 48KB/CTA, PD=4", k_stream<6, 4>, nt, 1200, g, nblk);
            run_stream("bulk L2 prefetch 48KB/CTA, PD=8", k_stream<6, 8>, nt, 1200, g, nblk);
        }
        cudaFree(g);
    }
    for (int nt : {128, 256, 512, 1024}) run("pure lds.32", k_pure<4>, nt, 1000, 32, SM);
    for (int nt : {128, 256, 512, 1024}) run("pure lds.64", k_pure<8>, nt, 1000, 32, SM);
    for (int nt : {128, 256, 512, 1024}) run("pure lds.128", k_pure<16>, nt, 1000, 32, SM);
    return 0;
}
