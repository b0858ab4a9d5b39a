// attention_flash.cu -- BERT self-attention for context-length sequences (64 < S <= 512: max_seq_length 384 of the phrase dumps,
// options.py:33, and 512 of the reference's dump recipe) on the Hopper tensor cores.  Same arithmetic as attention_tc.cu:
// softmax(Q K^T / 8 + (1 - mask) * -10000) V per head, fp32 softmax; the keys are streamed in blocks of 64 with an online
// (running max, running sum) softmax, so shared memory does not grow with S.
//
// One CTA (128 threads = one warpgroup) owns a 64-row query tile of one head of one sequence:
//   - K blocks arrive by TMA (two SWIZZLE_128B boxes of 32 floats x 64 keys out of the [T, 2304] QKV activation) into a
//     two-stage mbarrier ring: block j+2 is in flight while block j is used.
//   - V blocks are read into registers one block ahead and written TRANSPOSED ([d][key], the K-major B operand of P V) with
//     the 128-byte swizzle by hand: warp w owns keys 32 (w >> 1) .. +31 (lane = key) and d in [32 (w & 1), +32).
//   - per block: S = Q K^T (m64n64 wgmma), scale + mask, new row max, rescale of the running sum and of the O accumulator,
//     P = exp(S - max) to shared memory (K-major), O += P V^T.  After the last block O is divided by the row sum.
// Keys >= S (the tail of the last block) get probability exactly 0; masked keys get the reference's -10000 bias.
//
// Two variants, as in attention_tc.cu:
//   BX = false: Q, K, P, V^T as fp32 read by wgmma tf32 (the 1xTF32 encoder mode);                               ~83 KB smem
//   BX = true : Q, K, P, V^T as bf16 (hi, lo) planes, three bf16 wgmmas per contraction (hi.lo + lo.hi + hi.hi, ~2^-17 relative)
//               for the fp32-accurate modes; K lands as fp32 and is split by the threads.  Optionally writes the context as
//               (hi, lo) planes too, for the bf16x3 output projection.                                               ~99 KB smem
// Either way two CTAs share an SM.
#include "wgmma.cuh"
#include <cuda_bf16.h>

#define AF_H 768
#define AF_DH 64
#define AF_HEADS 12
#define AF_MAX_S 512
#define AF_BOX (64 * 128)              // one [64 rows x 32 floats] fp32 box, or one [64 rows x 64 bf16] plane: 8 KB, 128-byte rows
#define AF_KSTAGE (2 * AF_BOX)          // one K block (64 keys x 64 d) as fp32
#define AF_OFF_Q 0                      // fp32: 2 boxes (d 0..31, 32..63); bx: hi plane | lo plane
#define AF_OFF_K (2 * AF_BOX)           // K ring, 2 stages of fp32
#define AF_OFF_KP (6 * AF_BOX)          // bx only: K planes hi | lo
#define AF_TAIL_BYTES (AF_MAX_S * 4 + 64)
template <bool BX> struct AfLayout {
    static constexpr unsigned P = BX ? 8 * AF_BOX : 6 * AF_BOX;        // fp32: 2 boxes (keys 0..31, 32..63); bx: hi | lo plane
    static constexpr unsigned VT = P + 2 * AF_BOX;                      // fp32: 2 boxes [64 d x 32 keys]; bx: hi | lo plane [64 d x 64 keys]
    static constexpr unsigned TAIL = VT + 2 * AF_BOX;                   // additive mask [512] + mbarriers
    static constexpr unsigned SMEM = TAIL + AF_TAIL_BYTES + 1024;       // + slack for the 1024-byte alignment of the window
};

struct AttnFlashArgs { const float* qkv; float* ctx; const long long* mask; int S;
                       unsigned short* ctx_hi; unsigned short* ctx_lo; };       // nullable (bx only): bf16 (hi, lo) planes of the context

__device__ __forceinline__ void af_split2(float x0, float x1, unsigned& hi, unsigned& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
    const float2 hf = __bfloat1622float2(h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<const unsigned*>(&h);
    lo = *reinterpret_cast<const unsigned*>(&l);
}
// 16 consecutive floats of one row (a, b: chunks 2q', 2q'+1 as float4 pairs) -> one 16-byte chunk per plane
__device__ __forceinline__ void af_split_chunk(float4 a, float4 b, uint4& h, uint4& l) {
    af_split2(a.x, a.y, h.x, l.x); af_split2(a.z, a.w, h.y, l.y); af_split2(b.x, b.y, h.z, l.z); af_split2(b.z, b.w, h.w, l.w);
}

template <bool BX>
__global__ void __launch_bounds__(128) attention_flash_kernel(const __grid_constant__ CUtensorMap map, const AttnFlashArgs a) {
    using Lay = AfLayout<BX>;
    extern __shared__ __align__(1024) unsigned char afsm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int S = a.S, h = blockIdx.x % AF_HEADS, q0 = (blockIdx.x / AF_HEADS) * 64, b = blockIdx.y;
    const int nkb = (S + 63) >> 6;
    unsigned char* base = (unsigned char*)((((unsigned long long)afsm) + 1023ull) & ~1023ull);
    const unsigned sbase = smem_u32(base);
    float* mb = reinterpret_cast<float*>(base + Lay::TAIL);                                   // [nkb * 64] additive key mask
    const unsigned bar_full = smem_u32(base + Lay::TAIL + AF_MAX_S * 4);                      // [2]: K ring stages
    const unsigned bar_q = bar_full + 16;
    const long long row0 = (long long)b * S;

    if (tid == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map) : "memory");
        mbar_init(bar_full, 1); mbar_init(bar_full + 8, 1); mbar_init(bar_q, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
        if (!BX) {
            mbar_expect_tx(bar_q, 2 * AF_BOX);
            for (int kb = 0; kb < 2; kb++) tma_load_2d(sbase + AF_OFF_Q + kb * AF_BOX, &map, h * AF_DH + kb * 32, (int)(row0 + q0), bar_q);
        }
        for (int j = 0; j < 2 && j < nkb; j++) {
            mbar_expect_tx(bar_full + 8 * j, AF_KSTAGE);
            for (int kb = 0; kb < 2; kb++)
                tma_load_2d(sbase + AF_OFF_K + j * AF_KSTAGE + kb * AF_BOX, &map, AF_H + h * AF_DH + kb * 32, (int)(row0 + j * 64), bar_full + 8 * j);
        }
    }
    for (int i = tid; i < nkb * 64; i += 128) mb[i] = (i < S) ? (1.0f - (float)a.mask[row0 + i]) * -10000.0f : 0.f;

    // V of block j: this thread's key and half of d, into registers; zeros past S
    const int vk = (warp >> 1) * 32 + lane, vdh = warp & 1;
    float4 vr[8];
    auto load_v = [&](int j) {
        const int key = j * 64 + vk;
        const float4* src = reinterpret_cast<const float4*>(a.qkv + (row0 + key) * (3 * AF_H) + 2 * AF_H + h * AF_DH) + vdh * 8;
#pragma unroll
        for (int i = 0; i < 8; i++) vr[i] = key < S ? __ldg(src + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    auto store_vt = [&]() {
        const unsigned kk = (unsigned)vk;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const float e[4] = {vr[i].x, vr[i].y, vr[i].z, vr[i].w};
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const unsigned d = (unsigned)((vdh * 8 + i) * 4 + t);
                if (!BX) {      // box kk >> 5 of [64 d x 32 keys] fp32: element (d, k) at d*128 + (((k>>2) ^ (d&7)) << 4) + (k&3)*4
                    const unsigned k = kk & 31u;
                    *reinterpret_cast<float*>(base + Lay::VT + (kk >> 5) * AF_BOX + d * 128 + ((((k >> 2) ^ (d & 7u)) << 4) | ((k & 3u) << 2))) = e[t];
                } else {        // [64 d x 64 keys] bf16 planes: element (d, k) at d*128 + (((k>>3) ^ (d&7)) << 4) + (k&7)*2
                    const unsigned off = d * 128 + ((((kk >> 3) ^ (d & 7u)) << 4) | ((kk & 7u) << 1));
                    const __nv_bfloat16 hb = __float2bfloat16_rn(e[t]);
                    *reinterpret_cast<__nv_bfloat16*>(base + Lay::VT + off) = hb;
                    *reinterpret_cast<__nv_bfloat16*>(base + Lay::VT + AF_BOX + off) = __float2bfloat16_rn(e[t] - __bfloat162float(hb));
                }
            }
        }
    };
    load_v(0);
    if (BX) {   // Q planes straight from global: row r = tid / 2, d in [32 (tid & 1), +32) -> plane chunks 4 (tid & 1) .. +3
        const unsigned r = (unsigned)(tid >> 1), hf = (unsigned)(tid & 1);
        const bool ok = q0 + (int)r < S;
        const float4* src = reinterpret_cast<const float4*>(a.qkv + (row0 + q0 + r) * (3 * AF_H) + h * AF_DH) + hf * 8;
#pragma unroll
        for (unsigned c = 0; c < 4; c++) {
            const float4 x = ok ? __ldg(src + 2 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 y = ok ? __ldg(src + 2 * c + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
            uint4 hi, lo;
            af_split_chunk(x, y, hi, lo);
            const unsigned q = hf * 4 + c, off = r * 128 + ((q ^ (r & 7u)) << 4);
            *reinterpret_cast<uint4*>(base + AF_OFF_Q + off) = hi;
            *reinterpret_cast<uint4*>(base + AF_OFF_Q + AF_BOX + off) = lo;
        }
    }
    store_vt();
    if (!BX) mbar_wait(bar_q, 0);

    float o[32];
#pragma unroll
    for (int i = 0; i < 32; i++) o[i] = 0.f;
    float m[2] = {-3.0e38f, -3.0e38f}, l[2] = {0.f, 0.f};      // running row max; this thread's partial running row sum
    for (int j = 0; j < nkb; j++) {
        if (j + 1 < nkb) load_v(j + 1);
        const unsigned stage = AF_OFF_K + (j & 1) * AF_KSTAGE;
        mbar_wait(bar_full + 8 * (j & 1), (j >> 1) & 1);
        if (BX) {   // K stage (fp32, 2 boxes) -> K planes: row r = tid / 2, plane chunks 4 (tid & 1) .. +3
            const unsigned r = (unsigned)(tid >> 1);
#pragma unroll
            for (unsigned q = (unsigned)(tid & 1) * 4; q < (unsigned)(tid & 1) * 4 + 4; q++) {
                const unsigned kb = q >> 2, c0 = (q & 3u) * 2u;
                const unsigned char* src = base + stage + kb * AF_BOX + r * 128;
                const float4 x = *reinterpret_cast<const float4*>(src + ((c0 ^ (r & 7u)) << 4));
                const float4 y = *reinterpret_cast<const float4*>(src + (((c0 + 1u) ^ (r & 7u)) << 4));
                uint4 hi, lo;
                af_split_chunk(x, y, hi, lo);
                const unsigned off = r * 128 + ((q ^ (r & 7u)) << 4);
                *reinterpret_cast<uint4*>(base + AF_OFF_KP + off) = hi;
                *reinterpret_cast<uint4*>(base + AF_OFF_KP + AF_BOX + off) = lo;
            }
        }
        fence_proxy_async_smem();           // V^T (and Q / K planes) stores -> visible to the tensor core
        __syncthreads();

        float s[32];
        wgmma_fence();
        if (!BX) {
#pragma unroll
            for (int kb = 0; kb < 2; kb++)
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const unsigned off = kb * AF_BOX + k * 32;
                    wgmma_tf32<64>(s, make_sw128_desc(sbase + AF_OFF_Q + off), make_sw128_desc(sbase + stage + off), (kb | k) ? 1 : 0);
                }
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const unsigned off = k * 32;
                const unsigned long long qh = make_sw128_desc(sbase + AF_OFF_Q + off), ql = make_sw128_desc(sbase + AF_OFF_Q + AF_BOX + off);
                const unsigned long long kh = make_sw128_desc(sbase + AF_OFF_KP + off), kl = make_sw128_desc(sbase + AF_OFF_KP + AF_BOX + off);
                wgmma_bf16<64>(s, qh, kl, k ? 1 : 0);
                wgmma_bf16<64>(s, ql, kh, 1);
                wgmma_bf16<64>(s, qh, kh, 1);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(s);
        // online softmax; s[4jj + 2hr + c] is query row 16 warp + lane/4 + 8 hr, key 64 j + 8 jj + 2 (lane % 4) + c
#pragma unroll
        for (int hr = 0; hr < 2; hr++) {
            float mx = m[hr];
#pragma unroll
            for (int jj = 0; jj < 8; jj++)
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    const int key = j * 64 + 8 * jj + 2 * (lane & 3) + c;
                    float& v = s[4 * jj + 2 * hr + c];
                    v = v * 0.125f + mb[key];
                    if (key < S) mx = fmaxf(mx, v);
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float corr = expf(m[hr] - mx);
            m[hr] = mx;
            float sum = 0.f;
#pragma unroll
            for (int jj = 0; jj < 8; jj++)
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    const int key = j * 64 + 8 * jj + 2 * (lane & 3) + c;
                    float& v = s[4 * jj + 2 * hr + c];
                    v = (key < S) ? expf(v - mx) : 0.f;
                    sum += v;
                }
            l[hr] = l[hr] * corr + sum;
#pragma unroll
            for (int jj = 0; jj < 8; jj++) { o[4 * jj + 2 * hr] *= corr; o[4 * jj + 2 * hr + 1] *= corr; }
        }
        // P -> shared memory, K-major [64 rows x 64 keys]
#pragma unroll
        for (int hr = 0; hr < 2; hr++) {
            const unsigned r = (unsigned)(warp * 16 + (lane >> 2) + 8 * hr);
#pragma unroll
            for (int jj = 0; jj < 8; jj++) {
                if (!BX) {
                    const unsigned key = (unsigned)(8 * jj + 2 * (lane & 3)), kb = key >> 5, c = (key & 31u) >> 2;
                    *reinterpret_cast<float2*>(base + Lay::P + kb * AF_BOX + r * 128 + ((c ^ (r & 7u)) << 4) + (key & 3u) * 4) =
                        make_float2(s[4 * jj + 2 * hr], s[4 * jj + 2 * hr + 1]);
                } else {
                    unsigned ph, pl;
                    af_split2(s[4 * jj + 2 * hr], s[4 * jj + 2 * hr + 1], ph, pl);
                    const unsigned off = r * 128 + ((((unsigned)jj) ^ (r & 7u)) << 4) + (lane & 3) * 4;
                    *reinterpret_cast<unsigned*>(base + Lay::P + off) = ph;
                    *reinterpret_cast<unsigned*>(base + Lay::P + AF_BOX + off) = pl;
                }
            }
        }
        fence_proxy_async_smem();
        __syncthreads();                    // P complete; every thread is past S = Q K^T (and the K split): the stage is free
        if (tid == 0 && j + 2 < nkb) {
            mbar_expect_tx(bar_full + 8 * (j & 1), AF_KSTAGE);
            for (int kb = 0; kb < 2; kb++)
                tma_load_2d(sbase + stage + kb * AF_BOX, &map, AF_H + h * AF_DH + kb * 32, (int)(row0 + (j + 2) * 64), bar_full + 8 * (j & 1));
        }
        wgmma_fence();
        if (!BX) {
#pragma unroll
            for (int kb = 0; kb < 2; kb++)
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const unsigned off = kb * AF_BOX + k * 32;
                    wgmma_tf32<64>(o, make_sw128_desc(sbase + Lay::P + off), make_sw128_desc(sbase + Lay::VT + off), 1);
                }
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const unsigned off = k * 32;
                const unsigned long long ph = make_sw128_desc(sbase + Lay::P + off), pl = make_sw128_desc(sbase + Lay::P + AF_BOX + off);
                const unsigned long long vh = make_sw128_desc(sbase + Lay::VT + off), vl = make_sw128_desc(sbase + Lay::VT + AF_BOX + off);
                wgmma_bf16<64>(o, ph, vl, 1);
                wgmma_bf16<64>(o, pl, vh, 1);
                wgmma_bf16<64>(o, ph, vh, 1);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(o);
        __syncthreads();                    // P and V^T buffers are free
        if (j + 1 < nkb) store_vt();
    }
#pragma unroll
    for (int hr = 0; hr < 2; hr++) {
        float sum = l[hr];
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        const float inv = 1.0f / sum;
        const int q = q0 + warp * 16 + (lane >> 2) + 8 * hr;
        if (q >= S) continue;
        const long long at = (row0 + q) * AF_H + h * AF_DH + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < 8; jj++) {
            const float x0 = o[4 * jj + 2 * hr] * inv, x1 = o[4 * jj + 2 * hr + 1] * inv;
            *reinterpret_cast<float2*>(a.ctx + at + 8 * jj) = make_float2(x0, x1);
            if (BX && a.ctx_hi) {
                unsigned ph, pl;
                af_split2(x0, x1, ph, pl);
                *reinterpret_cast<unsigned*>(a.ctx_hi + at + 8 * jj) = ph;
                *reinterpret_cast<unsigned*>(a.ctx_lo + at + 8 * jj) = pl;
            }
        }
    }
}

// qkv: [T, 2304] fp32 (Q | K | V, heads contiguous inside each), ctx: [T, 768]; mask int64 [B, S]; 1 <= S <= 512, 12 heads.
// split: bf16 (hi, lo) plane variant; ctx_hi / ctx_lo (nullable, split only): the context's planes as well.
int dph_launch_attention_flash(const float* qkv, float* ctx, const long long* mask, int B, int S, long long T, cudaStream_t st, int split,
                               unsigned short* ctx_hi, unsigned short* ctx_lo) {
    DPH_CHECK(S >= 1 && S <= AF_MAX_S && B >= 1 && B <= 65535 && T >= (long long)B * S && T <= INT32_MAX, "attention_flash: S must be 1..512");
    static DphPerDeviceOnce once;
    if (once.first()) {
        DPH_CUDA(cudaFuncSetAttribute(attention_flash_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AfLayout<false>::SMEM));
        DPH_CUDA(cudaFuncSetAttribute(attention_flash_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AfLayout<true>::SMEM));
    }
    CUtensorMap map;
    DPH_TRY(dph_make_map_f32(&map, qkv, T, 3 * AF_H, 3 * AF_H, 64));
    AttnFlashArgs a;
    a.qkv = qkv; a.ctx = ctx; a.mask = mask; a.S = S;
    a.ctx_hi = split ? ctx_hi : nullptr; a.ctx_lo = split ? ctx_lo : nullptr;
    const dim3 grid((unsigned)(AF_HEADS * ((S + 63) / 64)), (unsigned)B, 1);
    if (split) attention_flash_kernel<true><<<grid, 128, AfLayout<true>::SMEM, st>>>(map, a);
    else attention_flash_kernel<false><<<grid, 128, AfLayout<false>::SMEM, st>>>(map, a);
    DPH_CUDA(cudaGetLastError());
    return 0;
}
