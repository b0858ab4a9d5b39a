// tools/scan_floor.cu -- microbenchmark: the HBM floor of the quad scan.  Default shape C2 (100 M phrases, IVF4096,PQ96, batch 64,
// nprobe 256); `./scan_floor NLIST BLOCKS_PER_LIST BATCH NPROBE` takes another, e.g. C4 on one GPU (500 M phrases):
//   ./scan_floor 65536 239 1024 256
// Streams NLIST lists of BLOCKS_PER_LIST code blocks (3 KB each) through the scan's own access pattern -- one persistent CTA per SM
// pulling (list, item) units from an atomic queue and claiming its next unit when it starts the current one; per warp one block per
// round into registers with ld.global.nc.L1::no_allocate and cp.async.bulk.prefetch.L2 of the block R rounds ahead -- with no
// gathers.  Probes per list ~ Binomial(BATCH * NPROBE, 1 / NLIST).  Unit schedules:
//   (a) items of <= 4 probing queries: ceil(cnt / 4) sibling units per list, adjacent in the queue;
//   (b) each list once;
//   (c) each list once, plus the packed-table source reads of the unit's min(cnt, 8) queries: 24 KB per query (the compact 8-bit quad
//       table source), from a BATCH x 24 KB area, all issued as 16-byte loads before they are consumed.  Once with the default L2
//       policy everywhere, once with the tables loaded evict_last and the code stream (loads and bulk prefetches) marked evict_first.
// (b) is the least time the scan could take; (a) - (b) is the cost of sibling items that re-read a list from HBM; (c) - (b) is the
// cost of the table reads, and the two (c) columns show whether an L2 priority keeps the tables resident under the code stream.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scan_floor tools/scan_floor.cu && ./scan_floor
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <random>
#include <vector>
#include <cuda_runtime.h>

#define BLK 3072
#define TAB_BYTES (3 * 256 * 32)    // one query's compact 8-bit quad table source
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ uint4 ldg_stream(const uint4* p, unsigned long long pol, bool hint) {
    uint4 r;
    if (hint)
        asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    else
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint4 ldg_table(const uint4* p, unsigned long long pol, bool hint) {
    uint4 r;
    if (hint)
        asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    else
        asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void l2_prefetch_block(const void* p, unsigned long long pol, bool hint) {
    if (hint) asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;" :: "l"(p), "n"(BLK), "l"(pol) : "memory");
    else asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(p), "n"(BLK) : "memory");
}

struct Unit { int list, nq, q0; };      // (c): the unit's queries are q0 .. q0 + nq - 1 (mod batch)

__global__ void __launch_bounds__(512) floor_kernel(const uint8_t* codes, int nb, const Unit* units, int total_units, int* next_unit, int rounds,
                             const uint8_t* tabs, int batch, bool hint, unsigned* sink) {
    __shared__ int unit, next;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    unsigned long long pol_first = 0, pol_last = 0;
    if (hint) {
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_first));
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_last));
    }
    unsigned acc = 0;
    if (threadIdx.x == 0) unit = atomicAdd(next_unit, 1);
    __syncthreads();
    while (unit < total_units) {
        if (threadIdx.x == 0) next = atomicAdd(next_unit, 1);          // claim-ahead: the next unit is claimed when this one starts
        const Unit ud = units[unit];
        const uint4* lbase = reinterpret_cast<const uint4*>(codes + (size_t)ud.list * nb * BLK);
        unsigned b = warp, bp = warp;
        for (int r = 0; r < rounds && bp < (unsigned)nb; r++, bp += nw)
            if (lane == 0) l2_prefetch_block(lbase + (size_t)bp * (BLK / 16), pol_first, hint);
        uint4 nxt[6];
        if (b < (unsigned)nb) {
#pragma unroll
            for (int c = 0; c < 6; c++) nxt[c] = ldg_stream(lbase + (size_t)b * (BLK / 16) + lane + c * 32, pol_first, hint);
        }
        if (tabs) {       // the table build's reads: one table (four queries) at a time, all of its loads in flight
            for (int t0 = 0; t0 < ud.nq; t0 += 4) {
                uint4 v[24];
#pragma unroll
                for (int e = 0; e < 24; e++) {
                    const int i = threadIdx.x + e * 256;                 // 6144 16-byte chunks per table of four queries
                    const int qi = t0 + (i / 1536);
                    const int q = (ud.q0 + (qi < ud.nq ? qi : 0)) % batch;
                    v[e] = ldg_table(reinterpret_cast<const uint4*>(tabs + (size_t)q * TAB_BYTES) + (i % 1536), pol_last, hint);
                }
#pragma unroll
                for (int e = 0; e < 24; e++) acc ^= v[e].x ^ v[e].y ^ v[e].z ^ v[e].w;
            }
        }
        while (b < (unsigned)nb) {
            uint4 cur[6];
#pragma unroll
            for (int c = 0; c < 6; c++) cur[c] = nxt[c];
            if (bp < (unsigned)nb) { if (lane == 0) l2_prefetch_block(lbase + (size_t)bp * (BLK / 16), pol_first, hint); bp += nw; }
            b += nw;
            if (b < (unsigned)nb) {
#pragma unroll
                for (int c = 0; c < 6; c++) nxt[c] = ldg_stream(lbase + (size_t)b * (BLK / 16) + lane + c * 32, pol_first, hint);
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

int main(int argc, char** argv) {
    const int nlist = argc > 1 ? atoi(argv[1]) : 4096;
    const int nb = argc > 2 ? atoi(argv[2]) : 763;               // C2: 24 414 vectors per list / 32
    const int batch = argc > 3 ? atoi(argv[3]) : 64;
    const int nprobe = argc > 4 ? atoi(argv[4]) : 256;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const size_t bytes = (size_t)nlist * nb * BLK;
    uint8_t *codes = nullptr, *tabs = nullptr; Unit* d_units = nullptr; int* d_next = nullptr; unsigned* sink = nullptr;
    CK(cudaMalloc(&codes, bytes));
    CK(cudaMemset(codes, 0x5A, bytes));
    CK(cudaMalloc(&tabs, (size_t)batch * TAB_BYTES));
    CK(cudaMemset(tabs, 0x3C, (size_t)batch * TAB_BYTES));
    CK(cudaMalloc(&d_next, 4)); CK(cudaMalloc(&sink, 4));
    std::mt19937 rng(1234);
    std::binomial_distribution<int> probes(batch * nprobe, 1.0 / nlist);
    std::uniform_int_distribution<int> qpick(0, batch - 1);
    std::vector<Unit> ua, ub;
    long long probed = 0, table_bytes = 0;
    for (int l = 0; l < nlist; l++) {
        const int cnt = probes(rng);
        if (cnt == 0) continue;
        probed++;
        const int nq = cnt < 8 ? cnt : 8;
        ub.push_back({l, nq, qpick(rng)});
        table_bytes += (long long)((nq + 3) / 4) * 4 * TAB_BYTES;
        for (int it = 0; it < (cnt + 3) / 4; it++) ua.push_back({l, 0, 0});
    }
    CK(cudaMalloc(&d_units, ua.size() * sizeof(Unit)));
    const double distinct = probed * (double)nb * BLK;
    printf("%s, %d SMs, L2 %d MB; nlist %d, %d blocks per list, batch %d, nprobe %d; %lld lists probed, %zu items of <= 4 queries; "
           "distinct bytes %.3f GB; (c) table reads %.3f GB from a %.1f MB area\n", prop.name, prop.multiProcessorCount, prop.l2CacheSize >> 20,
           nlist, nb, batch, nprobe, probed, ua.size(), distinct * 1e-9, table_bytes * 1e-9, batch * (double)TAB_BYTES / (1 << 20));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    auto run = [&](const std::vector<Unit>& units, int threads, int rounds, bool tables, bool hint, int reps) -> float {
        CK(cudaMemcpy(d_units, units.data(), units.size() * sizeof(Unit), cudaMemcpyHostToDevice));
        float best = 1e30f;
        for (int i = 0; i < reps + 1; i++) {
            CK(cudaMemset(d_next, 0, 4));
            CK(cudaEventRecord(e0));
            floor_kernel<<<prop.multiProcessorCount, threads>>>(codes, nb, d_units, (int)units.size(), d_next, rounds, tables ? tabs : nullptr,
                                                                 batch, hint, sink);
            CK(cudaGetLastError());
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (i > 0 && ms < best) best = ms;          // first launch: warm-up
        }
        return best;
    };
    for (int threads : {512, 256})
        for (int rounds : {2, 4, 6, 8}) {
            const float ta = run(ua, threads, rounds, false, false, 5), tb = run(ub, threads, rounds, false, false, 5);
            printf("threads %3d, L2 prefetch %d rounds: (a) sibling items %.3f ms  (b) each list once %.3f ms = %.2f TB/s of distinct bytes;"
                   " (a) - (b) %.3f ms\n", threads, rounds, ta, tb, distinct / (tb * 1e-3) * 1e-12, ta - tb);
        }
    // (c) at the quad kernel's own shape: 256 threads (the table loop assumes it), 2 rounds
    const float tb = run(ub, 256, 2, false, false, 5), tcd = run(ub, 256, 2, true, false, 5), tch = run(ub, 256, 2, true, true, 5);
    printf("threads 256, L2 prefetch 2 rounds: (b) %.3f ms  (c) default policy %.3f ms (+%.3f)  (c) tables evict_last, codes evict_first "
           "%.3f ms (+%.3f)\n", tb, tcd, tcd - tb, tch, tch - tb);
    return 0;
}
