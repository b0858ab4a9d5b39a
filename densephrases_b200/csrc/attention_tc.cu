// attention_tc.cu -- BERT self-attention for query-length sequences (S <= 64: max_query_length 24 / 32 / 64, options.py:38,
// reference Makefile:441) on the Hopper tensor cores.  Same arithmetic as HF BertSelfAttention behind Encoder.embed_query
// (reference densephrases/encoder.py:101-118): softmax(Q K^T / 8 + (1 - mask) * -10000) V per head, fp32 softmax; the two
// contractions run as wgmma tf32 with fp32 accumulation in registers (torch 1.9 -- the reference's pin -- also ran the attention
// matmuls in TF32 on Ampere+).
// attention_tc_bx_kernel (further down) is the fp32-accurate variant used by the 3xTF32 / bf16x3 encoder modes: Q, K, P and V^T are
// carried as bf16 (hi, lo) planes and every contraction is hi.lo + lo.hi + hi.hi (three bf16 wgmmas, ~2^-17 relative).
//
// One CTA (256 threads = two warpgroups) handles TWO heads of one sequence of one tower; warpgroup hh owns head h0 + hh:
//   rows 0..63 of every operand tile = tokens of head h0, rows 64..127 = tokens of head h0+1.
//   1. TMA (SWIZZLE_128B boxes of 32 floats x 64 rows out of the [T, 2304] QKV activation) stages Q and K of both heads as two
//      K-major [128 x 64] operands; meanwhile the threads stage V TRANSPOSED ([d][key], the K-major B operand of P V) with the
//      same 128-byte swizzle written by hand, one warp per (head, 32-key block, half of d), conflict-free.
//   2. S = Q K^T : warpgroup hh issues m64n64 wgmmas over its head's 64 query rows and 64 key rows (k = 64).
//   3. Scale + mask + softmax on the register fragment (a row lives in the 4 lanes of a quad: shuffles), P written back to shared
//      memory (over the head's dead Q rows) in the swizzled K-major layout.
//   4. O = P V : P [64 x 64 keys] against V^T of the head [64 d x 64 keys].
//   5. The fragment -> 256-byte row segments of the context activation.
// ~97 KB shared memory per CTA -> two CTAs per SM.
#include "wgmma.cuh"
#include <cuda_bf16.h>

#define AT_H 768
#define AT_DH 64
#define AT_TILE (128 * 128)            // bytes of one [128 rows x 32 floats] swizzled operand block
#define AT_VT_TILE (64 * 128)          // bytes of one [64 d x 32 keys] block of V^T
#define AT_SMEM_QK 0                   // Q kb0, Q kb1, K kb0, K kb1 (P kb0, kb1 alias Q after S is complete)
#define AT_SMEM_VT (4 * AT_TILE)       // [head][kb] : 4 blocks
#define AT_SMEM_TAIL (AT_SMEM_VT + 4 * AT_VT_TILE)
#define AT_SMEM_BYTES (AT_SMEM_TAIL + 64 * 4 + 64 + 1024)

struct AttnTcMaps { CUtensorMap qkv[2]; };
struct AttnTcArgs { const float* qkv[2]; float* ctx[2]; const long long* mask; int S;
                    unsigned short* ctx_hi[2]; unsigned short* ctx_lo[2]; };       // bx kernel only, nullable: bf16 (hi, lo) planes of the context

// x -> (hi, lo) bf16 bit patterns with x = hi + lo up to 2^-18 |x|; two elements per 32-bit word (element 0 in the low half):
// one packed convert for the hi parts, one for the remainders
__device__ __forceinline__ void bx_split2(float x0, float x1, unsigned& hi, unsigned& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
    const float2 hf = __bfloat1622float2(h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<const unsigned*>(&h);
    lo = *reinterpret_cast<const unsigned*>(&l);
}

// Softmax of the S fragment of one warpgroup (m64n64 layout, see wgmma.cuh): s[4j + c] is query row r = 16 warp + lane/4 + 8(c/2),
// key 8j + 2(lane%4) + c%2.  Scale, additive key mask, keys >= S excluded; on return s holds the probabilities.
__device__ __forceinline__ void at_softmax(float (&s)[32], const float* mb, int S, int lane) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
        float mx = -3.0e38f;
#pragma unroll
        for (int j = 0; j < 8; j++)
#pragma unroll
            for (int c = 0; c < 2; c++) {
                const int key = 8 * j + 2 * (lane & 3) + c;
                float& v = s[4 * j + 2 * h + c];
                v = v * 0.125f + mb[key];
                if (key < S) mx = fmaxf(mx, v);
            }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; j++)
#pragma unroll
            for (int c = 0; c < 2; c++) {
                const int key = 8 * j + 2 * (lane & 3) + c;
                float& v = s[4 * j + 2 * h + c];
                v = (key < S) ? expf(v - mx) : 0.f;
                sum += v;
            }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        const float inv = 1.0f / sum;
#pragma unroll
        for (int j = 0; j < 8; j++) { s[4 * j + 2 * h] *= inv; s[4 * j + 2 * h + 1] *= inv; }
    }
}

__global__ void __launch_bounds__(256, 2) attention_tc_kernel(const __grid_constant__ AttnTcMaps maps, const AttnTcArgs a) {
    extern __shared__ __align__(1024) unsigned char atsm[];
    // swizzle atoms need 1024-byte alignment: the window is rounded up here (the launch reserves 1 KB of slack)
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int hh = tid >> 7, wq = warp & 3;                     // warpgroup = head of the pair, warp inside the warpgroup
    const int hp = blockIdx.x, b = blockIdx.y, tw = blockIdx.z;
    const int S = a.S, h0 = hp * 2;
    unsigned char* base = (unsigned char*)((((unsigned long long)atsm) + 1023ull) & ~1023ull);
    const unsigned sbase = smem_u32(base);
    float* mb = reinterpret_cast<float*>(base + AT_SMEM_TAIL);                         // [64] additive key mask
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(base + AT_SMEM_TAIL + 256);
    const unsigned bar_tma = smem_u32(bars);
    const CUtensorMap* map = &maps.qkv[tw];
    const long long row0 = (long long)b * S;

    if (tid == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
        mbar_init(bar_tma, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(bar_tma, 4 * AT_TILE);
#pragma unroll
        for (int op = 0; op < 2; op++)              // 0: Q (columns 0..767), 1: K (columns 768..1535)
#pragma unroll
            for (int kb = 0; kb < 2; kb++)
#pragma unroll
                for (int h = 0; h < 2; h++)
                    tma_load_2d(sbase + AT_SMEM_QK + (op * 2 + kb) * AT_TILE + h * (64 * 128), map, op * AT_H + (h0 + h) * AT_DH + kb * 32, (int)row0, bar_tma);
    }
    // V^T, hand-swizzled: warp w stages block (head w>>2, keys 32((w>>1)&1) .. +31), d in [32 (w&1), +32); lane = key, so the 32
    // lanes of one store fill one 128-byte row (d fixed) -- every bank once.  Element (d, kk) of a block: d*128 + ((kk>>2 ^ d&7) << 4) + (kk&3)*4.
    {
        const int vh = warp >> 2, kbk = (warp >> 1) & 1, dh = warp & 1, j = kbk * 32 + lane;
        const bool ok = j < S;
        const float4* src = reinterpret_cast<const float4*>(a.qkv[tw] + (row0 + j) * (3 * AT_H) + 2 * AT_H + (h0 + vh) * AT_DH);
        unsigned char* blk = base + AT_SMEM_VT + (vh * 2 + kbk) * AT_VT_TILE;
        const unsigned kk = (unsigned)lane;
#pragma unroll 4
        for (int d4 = dh * 8; d4 < dh * 8 + 8; d4++) {
            const float4 v = ok ? __ldg(src + d4) : make_float4(0.f, 0.f, 0.f, 0.f);
            const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const unsigned d = (unsigned)(d4 * 4 + t);
                *reinterpret_cast<float*>(blk + d * 128 + ((((kk >> 2) ^ (d & 7u)) << 4) | ((kk & 3u) << 2))) = e[t];
            }
        }
        if (tid < 64) mb[tid] = (tid < S) ? (1.0f - (float)a.mask[row0 + tid]) * -10000.0f : 0.f;
    }
    fence_proxy_async_smem();                       // generic-proxy stores above -> visible to the tensor core's async-proxy reads
    __syncthreads();
    mbar_wait(bar_tma, 0);

    float s[32];
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 2; kb++)
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const unsigned off = kb * AT_TILE + hh * (64 * 128) + k * 32;
            wgmma_tf32<64>(s, make_sw128_desc(sbase + AT_SMEM_QK + off), make_sw128_desc(sbase + AT_SMEM_QK + 2 * AT_TILE + off), (kb | k) ? 1 : 0);
        }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    at_softmax(s, mb, S, lane);
    // P rows of this head -> blocks kb = 0,1 over the head's Q rows (its S is complete => the tensor core is done reading them)
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const unsigned r = (unsigned)(hh * 64 + wq * 16 + (lane >> 2) + 8 * h);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const unsigned key = (unsigned)(8 * j + 2 * (lane & 3)), kb = key >> 5, c = (key & 31u) >> 2;
            *reinterpret_cast<float2*>(base + AT_SMEM_QK + kb * AT_TILE + r * 128 + ((c ^ (r & 7u)) << 4) + (key & 3u) * 4) =
                make_float2(s[4 * j + 2 * h], s[4 * j + 2 * h + 1]);
        }
    }
    fence_proxy_async_smem();
    warpgroup_bar(1 + hh);

    float o[32];
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 2; kb++)
#pragma unroll
        for (int k = 0; k < 4; k++)
            wgmma_tf32<64>(o, make_sw128_desc(sbase + AT_SMEM_QK + kb * AT_TILE + hh * (64 * 128) + k * 32),
                           make_sw128_desc(sbase + AT_SMEM_VT + (hh * 2 + kb) * AT_VT_TILE + k * 32), (kb | k) ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int i = wq * 16 + (lane >> 2) + 8 * h;
        if (i >= S) continue;
        float* out = a.ctx[tw] + (row0 + i) * AT_H + (h0 + hh) * AT_DH + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 8; j++) *reinterpret_cast<float2*>(out + 8 * j) = make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
    }
}


// =================================================================================================
// fp32-accurate variant: bf16 (hi, lo) planes, three bf16 wgmmas per contraction.  Same work split as above (two heads per CTA,
// one warpgroup per head), three 32 KB shared-memory regions that are reused as the data moves on, so that the CTA still needs
// only ~97 KB and TWO CTAs share an SM:
//   R0: Q as fp32 (TMA landing, 2 k-block tiles)        -> K planes  [K_hi 16 KB | K_lo 16 KB]
//   R1: K as fp32 (TMA landing)                         -> V^T planes [h0 hi | h1 hi | h0 lo | h1 lo] (8 KB each)
//   R2: Q planes [Q_hi 16 KB | Q_lo 16 KB]              -> P planes  [P_hi | P_lo]
// A plane tile is [128 rows x 64 bf16] = 128-byte rows, SWIZZLE_128B, K-major: logical 16-byte chunk q of row r sits at
// r*128 + ((q ^ (r & 7)) << 4).  The fp32 -> planes conversion of row r is split over two threads of the row's warpgroup (each
// reads two fp32 chunks of the TMA tile per output chunk and writes one bf16 chunk per plane).
// =================================================================================================
#define ATB_R0 0
#define ATB_R1 (32 * 1024)
#define ATB_R2 (64 * 1024)
#define ATB_TAIL (96 * 1024)
#define ATB_SMEM_BYTES (ATB_TAIL + 64 * 4 + 64 + 1024)
#define ATB_PLANE (16 * 1024)

// fp32 TMA tiles (2 k-blocks of [128 x 32 floats]) at `src` -> bf16 planes [128 x 64] at dst_hi / dst_lo: row r, chunks q0 .. q0+3
__device__ __forceinline__ void atb_convert_rows(const unsigned char* src, unsigned char* dst_hi, unsigned char* dst_lo, unsigned r, unsigned q0) {
#pragma unroll
    for (unsigned q = q0; q < q0 + 4; q++) {
        const unsigned kb = q >> 2, c0 = (q & 3u) * 2u;
        const float4 a = *reinterpret_cast<const float4*>(src + kb * AT_TILE + r * 128 + (((c0) ^ (r & 7u)) << 4));
        const float4 b = *reinterpret_cast<const float4*>(src + kb * AT_TILE + r * 128 + (((c0 + 1u) ^ (r & 7u)) << 4));
        uint4 h, l;
        bx_split2(a.x, a.y, h.x, l.x); bx_split2(a.z, a.w, h.y, l.y); bx_split2(b.x, b.y, h.z, l.z); bx_split2(b.z, b.w, h.w, l.w);
        const unsigned off = r * 128 + ((q ^ (r & 7u)) << 4);
        *reinterpret_cast<uint4*>(dst_hi + off) = h;
        *reinterpret_cast<uint4*>(dst_lo + off) = l;
    }
}

__global__ void __launch_bounds__(256, 2) attention_tc_bx_kernel(const __grid_constant__ AttnTcMaps maps, const AttnTcArgs a) {
    extern __shared__ __align__(1024) unsigned char atsm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int hh = tid >> 7, wq = warp & 3;
    const int hp = blockIdx.x, b = blockIdx.y, tw = blockIdx.z;
    const int S = a.S, h0 = hp * 2;
    unsigned char* base = (unsigned char*)((((unsigned long long)atsm) + 1023ull) & ~1023ull);
    const unsigned sbase = smem_u32(base);
    float* mb = reinterpret_cast<float*>(base + ATB_TAIL);
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(base + ATB_TAIL + 256);
    const unsigned bar_tma = smem_u32(bars);
    const CUtensorMap* map = &maps.qkv[tw];
    const long long row0 = (long long)b * S;

    if (tid == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
        mbar_init(bar_tma, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(bar_tma, 4 * AT_TILE);
#pragma unroll
        for (int op = 0; op < 2; op++)              // 0: Q -> R0, 1: K -> R1
#pragma unroll
            for (int kb = 0; kb < 2; kb++)
#pragma unroll
                for (int h = 0; h < 2; h++)
                    tma_load_2d(sbase + (op ? ATB_R1 : ATB_R0) + kb * AT_TILE + h * (64 * 128), map, op * AT_H + (h0 + h) * AT_DH + kb * 32, (int)row0, bar_tma);
    }
    // V of this thread's (head, key, half of d) while the TMA is in flight: warp w -> head w>>2, keys 32((w>>1)&1) .. +31, d in [32 (w&1), +32)
    const int vhh = warp >> 2, vj = ((warp >> 1) & 1) * 32 + lane, vdh = warp & 1;
    float4 vreg[8];
    {
        const bool ok = vj < S;
        const float4* src = reinterpret_cast<const float4*>(a.qkv[tw] + (row0 + vj) * (3 * AT_H) + 2 * AT_H + (h0 + vhh) * AT_DH) + vdh * 8;
#pragma unroll
        for (int d4 = 0; d4 < 8; d4++) vreg[d4] = ok ? __ldg(src + d4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid < 64) mb[tid] = (tid < S) ? (1.0f - (float)a.mask[row0 + tid]) * -10000.0f : 0.f;
    const unsigned crow = (unsigned)(tid >> 1), cq0 = (unsigned)(tid & 1) * 4u;          // conversion: row, first 16-byte chunk
    mbar_wait(bar_tma, 0);
    atb_convert_rows(base + ATB_R0, base + ATB_R2, base + ATB_R2 + ATB_PLANE, crow, cq0);             // Q: R0 -> R2
    __syncthreads();                                                                                   // every row of R0 has been read
    atb_convert_rows(base + ATB_R1, base + ATB_R0, base + ATB_R0 + ATB_PLANE, crow, cq0);             // K: R1 -> R0
    __syncthreads();                                                                                   // every row of R1 has been read
    {   // V^T planes into R1: element (d, key) of head vhh at  vhh*8K + d*128 + (((key >> 3) ^ (d & 7)) << 4) + (key & 7)*2
        unsigned char* vh = base + ATB_R1 + vhh * (8 * 1024);
        unsigned char* vl = vh + 16 * 1024;
        const unsigned kk = (unsigned)vj;
#pragma unroll
        for (int d4 = 0; d4 < 8; d4++) {
            const float e[4] = {vreg[d4].x, vreg[d4].y, vreg[d4].z, vreg[d4].w};
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const unsigned d = (unsigned)((vdh * 8 + d4) * 4 + t);
                const unsigned off = d * 128 + ((((kk >> 3) ^ (d & 7u)) << 4) | ((kk & 7u) << 1));
                const __nv_bfloat16 hb = __float2bfloat16_rn(e[t]);
                *reinterpret_cast<__nv_bfloat16*>(vh + off) = hb;
                *reinterpret_cast<__nv_bfloat16*>(vl + off) = __float2bfloat16_rn(e[t] - __bfloat162float(hb));
            }
        }
    }
    fence_proxy_async_smem();
    __syncthreads();

    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) {           // k = 16 bf16 = 32 bytes per wgmma
        const unsigned off = hh * (64 * 128) + k * 32;
        const unsigned long long qh = make_sw128_desc(sbase + ATB_R2 + off), ql = make_sw128_desc(sbase + ATB_R2 + ATB_PLANE + off);
        const unsigned long long kh = make_sw128_desc(sbase + ATB_R0 + off), kl = make_sw128_desc(sbase + ATB_R0 + ATB_PLANE + off);
        wgmma_bf16<64>(s, qh, kl, k ? 1 : 0);
        wgmma_bf16<64>(s, ql, kh, 1);
        wgmma_bf16<64>(s, qh, kh, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    at_softmax(s, mb, S, lane);
    // P planes over the head's Q plane rows (its S is complete => the tensor core is done with them)
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const unsigned r = (unsigned)(hh * 64 + wq * 16 + (lane >> 2) + 8 * h);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            unsigned ph, pl;
            bx_split2(s[4 * j + 2 * h], s[4 * j + 2 * h + 1], ph, pl);
            const unsigned off = r * 128 + ((((unsigned)j) ^ (r & 7u)) << 4) + (lane & 3) * 4;
            *reinterpret_cast<unsigned*>(base + ATB_R2 + off) = ph;
            *reinterpret_cast<unsigned*>(base + ATB_R2 + ATB_PLANE + off) = pl;
        }
    }
    fence_proxy_async_smem();
    warpgroup_bar(1 + hh);

    float o[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const unsigned off = hh * (64 * 128) + k * 32;
        const unsigned long long ph = make_sw128_desc(sbase + ATB_R2 + off), pl = make_sw128_desc(sbase + ATB_R2 + ATB_PLANE + off);
        const unsigned long long vhd = make_sw128_desc(sbase + ATB_R1 + hh * (8 * 1024) + k * 32), vld = make_sw128_desc(sbase + ATB_R1 + 16 * 1024 + hh * (8 * 1024) + k * 32);
        wgmma_bf16<64>(o, ph, vld, k ? 1 : 0);
        wgmma_bf16<64>(o, pl, vhd, 1);
        wgmma_bf16<64>(o, ph, vhd, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int i = wq * 16 + (lane >> 2) + 8 * h;
        if (i >= S) continue;
        const long long at = (row0 + i) * AT_H + (h0 + hh) * AT_DH + 2 * (lane & 3);
        float* out = a.ctx[tw] + at;
#pragma unroll
        for (int j = 0; j < 8; j++) *reinterpret_cast<float2*>(out + 8 * j) = make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
        if (a.ctx_hi[tw]) {               // the same row segment as (hi, lo) bf16 planes for the bf16x3 output projection
#pragma unroll
            for (int j = 0; j < 8; j++) {
                unsigned ph, pl;
                bx_split2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1], ph, pl);
                *reinterpret_cast<unsigned*>(a.ctx_hi[tw] + at + 8 * j) = ph;
                *reinterpret_cast<unsigned*>(a.ctx_lo[tw] + at + 8 * j) = pl;
            }
        }
    }
}

// towers (1 or 2) independent problems on the same mask; qkv[t]: [T, 2304] fp32 (Q | K | V, heads contiguous inside each),
// ctx[t]: [T, 768]; mask int64 [B, S]; S <= 64, 12 heads.
int dph_launch_attention_tc(int towers, const float* const* qkv, float* const* ctx, const long long* mask, int B, int S, long long T, cudaStream_t st,
                            int split, unsigned short* const* ctx_hi, unsigned short* const* ctx_lo) {
    DPH_CHECK(towers >= 1 && towers <= 2, "attention_tc: one or two towers");
    DPH_CHECK(S >= 1 && S <= 64 && B >= 1 && B <= 65535 && T >= (long long)B * S && T <= INT32_MAX, "attention_tc: S must be 1..64");
    static DphPerDeviceOnce once;
    if (once.first()) {
        DPH_CUDA(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM_BYTES));
        DPH_CUDA(cudaFuncSetAttribute(attention_tc_bx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATB_SMEM_BYTES));
    }
    AttnTcMaps maps{};
    AttnTcArgs a{};
    for (int t = 0; t < towers; t++) {
        DPH_TRY(dph_make_map_f32(&maps.qkv[t], qkv[t], T, 3 * AT_H, 3 * AT_H, 64));
        a.qkv[t] = qkv[t]; a.ctx[t] = ctx[t];
        a.ctx_hi[t] = ctx_hi ? ctx_hi[t] : nullptr; a.ctx_lo[t] = ctx_lo ? ctx_lo[t] : nullptr;
    }
    a.mask = mask; a.S = S;
    if (split) attention_tc_bx_kernel<<<dim3(6, (unsigned)B, (unsigned)towers), 256, ATB_SMEM_BYTES, st>>>(maps, a);
    else attention_tc_kernel<<<dim3(6, (unsigned)B, (unsigned)towers), 256, AT_SMEM_BYTES, st>>>(maps, a);
    DPH_CUDA(cudaGetLastError());
    return 0;
}
