// common.cuh -- shared device/host helpers for libdph_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#define DPH_D 768
#define DPH_M 96
#define DPH_KSUB 256
#define DPH_DSUB 8
#define DPH_CODE 96          // bytes per PQ code row
#define DPH_BLK_VECS 32      // vectors per interleaved code block
#define DPH_BLK_BYTES 3072   // 32 * 96
#define DPH_NEUTRAL (-3.402823466e+38f)  // faiss CMin<float>::neutral() == -FLT_MAX

#define DPH_API extern "C" __attribute__((visibility("default")))
void dph_set_error(const std::string& msg);

#define DPH_CUDA(call)                                                                              \
    do {                                                                                            \
        cudaError_t e__ = (call);                                                                   \
        if (e__ != cudaSuccess) {                                                                   \
            dph_set_error(std::string(#call) + ": " + cudaGetErrorString(e__) + " @" + __FILE__ + ":" + \
                          std::to_string(__LINE__));                                                \
            return 1;                                                                               \
        }                                                                                           \
    } while (0)
#define DPH_CHECK(cond, msg)                                                        \
    do {                                                                            \
        if (!(cond)) { dph_set_error(std::string(msg) + " (" #cond ")"); return 1; } \
    } while (0)
#define DPH_TRY(call)            \
    do {                         \
        int r__ = (call);        \
        if (r__) return r__;     \
    } while (0)

// Once-per-device latch for cudaFuncSetAttribute: function attributes live in the per-device context, so a process that drives
// several GPUs has to raise the dynamic shared-memory limit on each of them.
struct DphPerDeviceOnce {
    bool done[64] = {};
    bool first() {
        int d = 0;
        cudaGetDevice(&d);
        d &= 63;
        if (done[d]) return false;
        done[d] = true;
        return true;
    }
};

// Component-wise float2 FMA / add: two independent IEEE fp32 operations (Hopper has no packed f32x2 instructions), so each
// component follows exactly the rounding chain of a scalar accumulator.
__device__ __forceinline__ float2 dph_ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 dph_fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// ---- counter-based generator: bit-identical to oracle/ivfpq_ref.c (mix64 / rnd64 / approx_normal) ----
__host__ __device__ __forceinline__ uint64_t dph_mix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__host__ __device__ __forceinline__ uint64_t dph_rnd64(uint64_t seed, uint64_t stream, uint64_t a, uint64_t b) {
    return dph_mix64(dph_mix64(dph_mix64(seed ^ (stream * 0xA24BAED4963EE407ull)) + a) + b);
}
__host__ __device__ __forceinline__ float dph_approx_normal(uint64_t u, float sigma_over_std) {
    int32_t s = (int32_t)(u & 0xFFFF) + (int32_t)((u >> 16) & 0xFFFF) + (int32_t)((u >> 32) & 0xFFFF) + (int32_t)(u >> 48) - 131070;
    return (float)s * sigma_over_std;
}
#define DPH_IH4_STD 37837.227f
enum { DPH_STREAM_CODES = 1, DPH_STREAM_CENTROIDS = 2, DPH_STREAM_PQ = 3 };

// ---- order-preserving float <-> uint32 key (larger float -> larger key) ----
__host__ __device__ __forceinline__ uint32_t dph_fkey(float f) {
    uint32_t b;
#ifdef __CUDA_ARCH__
    b = __float_as_uint(f);
#else
    memcpy(&b, &f, 4);
#endif
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float dph_fkey_inv(uint32_t k) {
    uint32_t b = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
#ifdef __CUDA_ARCH__
    return __uint_as_float(b);
#else
    float f; memcpy(&f, &b, 4); return f;
#endif
}
// candidate key: score desc, then scan position asc  (== larger key first)
__host__ __device__ __forceinline__ uint64_t dph_ckey(float score, uint32_t gidx) {
    return ((uint64_t)dph_fkey(score) << 32) | (uint64_t)(0xFFFFFFFFu - gidx);
}
__host__ __device__ __forceinline__ float dph_ckey_score(uint64_t k) { return dph_fkey_inv((uint32_t)(k >> 32)); }
__host__ __device__ __forceinline__ uint32_t dph_ckey_gidx(uint64_t k) { return 0xFFFFFFFFu - (uint32_t)k; }

// ---- interleaved code-block layout -------------------------------------------------------------
// A block holds 32 vectors x 96 code bytes.  Lane l of a warp owns vector l of the block and reads
// its 96 bytes as 6 coalesced 16-byte chunks:  byte address  c*512 + l*16 + b  (c<6, b<16).
// Position t = c*16+b (0..95) holds sub-quantizer  m = 32*(t/32) + ((l + t%32) & 31):  the row is
// stored ROTATED by the lane number inside each 32-wide segment, so that at scan step t the 32 lanes
// of a warp look up 32 *different* sub-quantizers -> 32 different shared-memory banks (see scan.cu).
__host__ __device__ __forceinline__ int dph_blk_addr(int lane, int m) {
    int seg = m >> 5, s = ((m & 31) - lane) & 31;
    int t = seg * 32 + s;
    return (t >> 4) * 512 + lane * 16 + (t & 15);
}
// The inverse: the sub-quantizer held at position t (0..95) of lane `lane`'s row.
__host__ __device__ __forceinline__ int dph_blk_sub(int lane, int t) { return (t & ~31) + ((lane + (t & 31)) & 31); }

// Segment descriptor produced by the plan kernel: one per (query, probe rank); 32 bytes.
struct __align__(16) DphSeg {
    long long blk;      // first code block of the list in this shard's code array (-1: not in shard)
    int len;            // list length (vectors)
    unsigned gstart;    // canonical scan position of the list's first vector for this query
    float dis0;         // <xr, centroid>
    unsigned wrel;      // first in-shard work block of this segment, relative to the query's first block
    unsigned wend;      // one past the last
    int list;           // list number (or -1)
};

struct DphWork {       // device scalars written by the plan kernel
    long long total_blocks;
};
struct DphGroupWork {  // grouped modes (pair, quad): the work queue of (list, block segment, item) units the scan CTAs pull from
    long long total_blocks;         // sum over items of the list's blocks
    long long per;                  // blocks per segment (a list longer than this is cut into several units per item)
    int total_units;
    int next_unit;                  // queue head, advanced with atomicAdd by the scan CTAs; reset by the plan
};
// Quad mode: one fully resolved work item (list segment x group of <= 8 probing queries), written by the plan so that a scan CTA
// starts an item from ONE 160-byte read (prefetched during the previous item) instead of a chain of dependent look-ups.
#define DPH_QUAD_ITEM_Q 8           // queries per quad-mode work item: two packed tables of four
struct __align__(16) DphUnit {
    long long blk;                  // first code block of the list in this shard's code array
    int len;                        // list length (vectors)
    unsigned bi0, bend;             // block range of this segment inside the list
    int nq;                         // queries in the group (1..8); the unused slots repeat slot 0
    int list, pad;
    unsigned q[DPH_QUAD_ITEM_Q];    // query numbers
    unsigned gs[DPH_QUAD_ITEM_Q];   // canonical scan position of the list's first vector, per query
    float base[DPH_QUAD_ITEM_Q];    // <xr, centroid> + the query's quantisation offset
    float step[DPH_QUAD_ITEM_Q];    // the query's quantisation step
};
#define DPH_GROUP_SEG_MIN 128       // shortest segment worth rebuilding the packed 192 KB LUT for
#define DPH_GROUP_UNITS_PER_CTA 16  // lists are cut only when the batch has fewer than this many whole-list units per CTA
