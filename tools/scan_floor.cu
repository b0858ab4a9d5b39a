// tools/scan_floor.cu -- microbenchmark: the HBM floor of the quad scan at C2 (100 M phrases, IVF4096,PQ96, batch 64, nprobe 256).
// Streams 4096 lists of 763 code blocks (3 KB each, 9.6 GB) through the scan's own access pattern -- one persistent CTA per SM
// pulling (list, item) units from an atomic queue and claiming its next unit when it starts the current one; per warp one block per
// round into registers with ld.global.nc.L1::no_allocate and cp.async.bulk.prefetch.L2 of the block R rounds ahead -- with no
// gathers.  Two unit schedules:
//   (a) items of <= 4 probing queries: ceil(cnt / 4) sibling units per list, adjacent in the queue (cnt ~ Binomial(64, 1/16));
//   (b) each list once.
// (b) is the least time the scan could take at C2; (a) - (b) is the cost of sibling items that re-read a list from HBM.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scan_floor tools/scan_floor.cu && ./scan_floor
#include <cstdio>
#include <cstdint>
#include <random>
#include <vector>
#include <cuda_runtime.h>

#define NLIST 4096
#define NB 763                      // 24 414 vectors per list / 32
#define BLK 3072
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void l2_prefetch_block(const void* p) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(p), "n"(BLK) : "memory");
}

__global__ void floor_kernel(const uint8_t* codes, const int* unit_list, int total_units, int* next_unit, int rounds, unsigned* sink) {
    __shared__ int unit, next;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    unsigned acc = 0;
    if (threadIdx.x == 0) unit = atomicAdd(next_unit, 1);
    __syncthreads();
    while (unit < total_units) {
        if (threadIdx.x == 0) next = atomicAdd(next_unit, 1);          // claim-ahead: the next unit is claimed when this one starts
        const uint4* lbase = reinterpret_cast<const uint4*>(codes + (size_t)unit_list[unit] * NB * BLK);
        unsigned b = warp, bp = warp;
        for (int r = 0; r < rounds && bp < NB; r++, bp += nw)
            if (lane == 0) l2_prefetch_block(lbase + (size_t)bp * (BLK / 16));
        uint4 nxt[6];
        if (b < NB) {
#pragma unroll
            for (int c = 0; c < 6; c++) nxt[c] = ldg_stream(lbase + (size_t)b * (BLK / 16) + lane + c * 32);
        }
        while (b < NB) {
            uint4 cur[6];
#pragma unroll
            for (int c = 0; c < 6; c++) cur[c] = nxt[c];
            if (bp < NB) { if (lane == 0) l2_prefetch_block(lbase + (size_t)bp * (BLK / 16)); bp += nw; }
            b += nw;
            if (b < NB) {
#pragma unroll
                for (int c = 0; c < 6; c++) nxt[c] = ldg_stream(lbase + (size_t)b * (BLK / 16) + lane + c * 32);
            }
#pragma unroll
            for (int c = 0; c < 6; c++) acc ^= cur[c].x ^ cur[c].y ^ cur[c].z ^ cur[c].w;
        }
        __syncthreads();
        if (threadIdx.x == 0) unit = next;
        __syncthreads();
    }
    if (acc == 0x9E3779B9u) sink[0] = acc;      // keeps the loads alive
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const size_t bytes = (size_t)NLIST * NB * BLK;
    uint8_t* codes = nullptr; int *d_units = nullptr, *d_next = nullptr; unsigned* sink = nullptr;
    CK(cudaMalloc(&codes, bytes));
    CK(cudaMemset(codes, 0x5A, bytes));
    CK(cudaMalloc(&d_next, 4)); CK(cudaMalloc(&sink, 4));
    // (a): items per list from a seeded Binomial(64, 1/16) probe count, as the plan would emit them; (b): one unit per list
    std::mt19937 rng(1234);
    std::binomial_distribution<int> probes(64, 1.0 / 16);
    std::vector<int> ua, ub;
    long long probed = 0;
    for (int l = 0; l < NLIST; l++) {
        const int cnt = probes(rng);
        if (cnt == 0) continue;
        probed++;
        ub.push_back(l);
        for (int it = 0; it < (cnt + 3) / 4; it++) ua.push_back(l);
    }
    CK(cudaMalloc(&d_units, ua.size() * 4));
    printf("%s, %d SMs; %lld of %d lists probed, %zu items of <= 4 queries; distinct bytes %.3f GB\n", prop.name, prop.multiProcessorCount,
           probed, NLIST, ua.size(), probed * (double)NB * BLK * 1e-9);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    auto run = [&](const std::vector<int>& units, int threads, int rounds, int reps) -> float {
        CK(cudaMemcpy(d_units, units.data(), units.size() * 4, cudaMemcpyHostToDevice));
        float best = 1e30f;
        for (int i = 0; i < reps + 1; i++) {
            CK(cudaMemset(d_next, 0, 4));
            CK(cudaEventRecord(e0));
            floor_kernel<<<prop.multiProcessorCount, threads>>>(codes, d_units, (int)units.size(), d_next, rounds, sink);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (i > 0 && ms < best) best = ms;          // first launch: warm-up
        }
        return best;
    };
    const double distinct = probed * (double)NB * BLK;
    for (int threads : {512, 256})
        for (int rounds : {2, 4, 6, 8}) {
            const float ta = run(ua, threads, rounds, 5), tb = run(ub, threads, rounds, 5);
            printf("threads %3d, L2 prefetch %d rounds: (a) sibling items %.3f ms  (b) each list once %.3f ms = %.2f TB/s of distinct bytes;"
                   " (a) - (b) %.3f ms\n", threads, rounds, ta, tb, distinct / (tb * 1e-3) * 1e-12, ta - tb);
        }
    return 0;
}
