// prep.cu -- query preparation kernels of the IVF-PQ search (everything before the code scan):
//   * sgemm_nt_seq : out = X W^T with ONE sequential fp32 FMA chain per output (k ascending) -- used for the
//                    OPQ rotation (faiss LinearTransform::apply) and the coarse scores (IndexFlatIP::search),
//                    replacing the sgemm faiss calls at reference densephrases/index.py:200.
//   * coarse_select: top-nprobe lists per query, (score desc, list asc).
//   * lut          : PQ inner-product tables (faiss ProductQuantizer::compute_inner_prod_table) in two layouts.
//   * plan         : per (query, probe) segment descriptors + work partition for the scan kernel.
#include "index_internal.cuh"
#include "select.cuh"

// =================================================================================================
// sgemm_nt_seq: X [n,K] row-major, W [m,K] row-major, out [n,m].  128x128 tile, 256 threads, 8x8 micro-tile,
// BK = 8, double-buffered smem.  Each accumulator is updated by exactly one FFMA per k, k ascending, starting
// from +0 -> bit-identical to `acc = fmaf(x[t], w[t], acc)` on the host (oracle/ivfpq_ref.c:dot_seq).
// =================================================================================================
#define GBM 128
#define GBN 128
#define GBK 8
__global__ void __launch_bounds__(256) sgemm_nt_seq_kernel(const float* __restrict__ X, long long n, const float* __restrict__ W,
                                                            long long m, int K, float* __restrict__ out) {
    __shared__ __align__(16) float As[2][GBK][GBM];
    __shared__ __align__(16) float Bs[2][GBK][GBN];
    const int tid = threadIdx.x;
    const long long row0 = (long long)blockIdx.y * GBM, col0 = (long long)blockIdx.x * GBN;
    const int lr = tid & 127, lk4 = tid >> 7;          // tile row, which float4 along K (0..1)
    const long long arow = row0 + lr, brow = col0 + lr;
    const bool aok = arow < n, bok = brow < m;
    const float4* ap = reinterpret_cast<const float4*>(X + (aok ? arow : 0) * K) + lk4;
    const float4* bp = reinterpret_cast<const float4*>(W + (bok ? brow : 0) * K) + lk4;
    const int tx = tid & 15, ty = tid >> 4;
    // accumulators as float2 pairs along the output column (dph_ffma2: two independent IEEE fp32 FMAs): every output sees
    // exactly one fused multiply-add per k, k ascending (bit-identical to the scalar chain).
    float2 acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = make_float2(0.0f, 0.0f);
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 ra = aok ? __ldg(ap) : z4, rb = bok ? __ldg(bp) : z4;
    const int ktiles = K / GBK;
    int buf = 0;
    As[0][lk4 * 4 + 0][lr] = ra.x; As[0][lk4 * 4 + 1][lr] = ra.y; As[0][lk4 * 4 + 2][lr] = ra.z; As[0][lk4 * 4 + 3][lr] = ra.w;
    Bs[0][lk4 * 4 + 0][lr] = rb.x; Bs[0][lk4 * 4 + 1][lr] = rb.y; Bs[0][lk4 * 4 + 2][lr] = rb.z; Bs[0][lk4 * 4 + 3][lr] = rb.w;
    __syncthreads();
    for (int kt = 0; kt < ktiles; kt++) {
        if (kt + 1 < ktiles) {
            ra = aok ? __ldg(ap + (kt + 1) * 2) : z4;
            rb = bok ? __ldg(bp + (kt + 1) * 2) : z4;
        }
#pragma unroll
        for (int k = 0; k < GBK; k++) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
            float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float2 b[4] = {make_float2(b0.x, b0.y), make_float2(b0.z, b0.w), make_float2(b1.x, b1.y), make_float2(b1.z, b1.w)};
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const float2 a2 = make_float2(a[i], a[i]);
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = dph_ffma2(a2, b[j], acc[i][j]);
            }
        }
        if (kt + 1 < ktiles) {
            int nb = buf ^ 1;
            As[nb][lk4 * 4 + 0][lr] = ra.x; As[nb][lk4 * 4 + 1][lr] = ra.y; As[nb][lk4 * 4 + 2][lr] = ra.z; As[nb][lk4 * 4 + 3][lr] = ra.w;
            Bs[nb][lk4 * 4 + 0][lr] = rb.x; Bs[nb][lk4 * 4 + 1][lr] = rb.y; Bs[nb][lk4 * 4 + 2][lr] = rb.z; Bs[nb][lk4 * 4 + 3][lr] = rb.w;
            __syncthreads();
            buf = nb;
        }
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        long long r = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (r >= n) continue;
#pragma unroll
        for (int jh = 0; jh < 2; jh++) {
            long long c = col0 + jh * 64 + tx * 4;
            float* o = out + r * m + c;
            if (c + 3 < m && ((m & 3) == 0)) {
                *reinterpret_cast<float4*>(o) = make_float4(acc[i][jh * 2].x, acc[i][jh * 2].y, acc[i][jh * 2 + 1].x, acc[i][jh * 2 + 1].y);
            } else {
                const float v[4] = {acc[i][jh * 2].x, acc[i][jh * 2].y, acc[i][jh * 2 + 1].x, acc[i][jh * 2 + 1].y};
#pragma unroll
                for (int j = 0; j < 4; j++)
                    if (c + j < m) o[j] = v[j];
            }
        }
    }
}

// Same contract, 64x64 tile / 4x4 micro-tile / 32-deep k tiles: 4x the CTAs, a 4x shorter per-k-step dependency chain and a
// quarter of the (latency-bound) global-load round trips -- used when the 128x128 grid cannot fill the GPU (small query
// batches; the sequential-k definition forbids split-K).
#define GSK 32
__global__ void __launch_bounds__(256) sgemm_nt_seq_small_kernel(const float* __restrict__ X, long long n, const float* __restrict__ W,
                                                                  long long m, int K, float* __restrict__ out) {
    __shared__ __align__(16) float As[2][GSK][64];
    __shared__ __align__(16) float Bs[2][GSK][64];
    const int tid = threadIdx.x;
    const long long row0 = (long long)blockIdx.y * 64, col0 = (long long)blockIdx.x * 64;
    const int lr = tid & 63, q4 = tid >> 6;                 // tile row, float4 slot along K (q4 and q4 + 4 of 8)
    const long long arow = row0 + lr, brow = col0 + lr;
    const bool aok = arow < n, bok = brow < m;
    const float4* ap = reinterpret_cast<const float4*>(X + (aok ? arow : 0) * K) + q4;
    const float4* bp = reinterpret_cast<const float4*>(W + (bok ? brow : 0) * K) + q4;
    const int tx = tid & 15, ty = tid >> 4;
    float2 acc[4][2];                        // float2 pairs along the output column (see sgemm_nt_seq_kernel)
#pragma unroll
    for (int i = 0; i < 4; i++) { acc[i][0] = make_float2(0.0f, 0.0f); acc[i][1] = make_float2(0.0f, 0.0f); }
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 ra0 = aok ? __ldg(ap) : z4, ra1 = aok ? __ldg(ap + 4) : z4, rb0 = bok ? __ldg(bp) : z4, rb1 = bok ? __ldg(bp + 4) : z4;
    const int ktiles = K / GSK;
    int buf = 0;
    auto stash = [&](int b) {
        As[b][q4 * 4 + 0][lr] = ra0.x; As[b][q4 * 4 + 1][lr] = ra0.y; As[b][q4 * 4 + 2][lr] = ra0.z; As[b][q4 * 4 + 3][lr] = ra0.w;
        As[b][16 + q4 * 4 + 0][lr] = ra1.x; As[b][16 + q4 * 4 + 1][lr] = ra1.y; As[b][16 + q4 * 4 + 2][lr] = ra1.z; As[b][16 + q4 * 4 + 3][lr] = ra1.w;
        Bs[b][q4 * 4 + 0][lr] = rb0.x; Bs[b][q4 * 4 + 1][lr] = rb0.y; Bs[b][q4 * 4 + 2][lr] = rb0.z; Bs[b][q4 * 4 + 3][lr] = rb0.w;
        Bs[b][16 + q4 * 4 + 0][lr] = rb1.x; Bs[b][16 + q4 * 4 + 1][lr] = rb1.y; Bs[b][16 + q4 * 4 + 2][lr] = rb1.z; Bs[b][16 + q4 * 4 + 3][lr] = rb1.w;
    };
    stash(0);
    __syncthreads();
    for (int kt = 0; kt < ktiles; kt++) {
        if (kt + 1 < ktiles) {
            const int o = (kt + 1) * 8;
            ra0 = aok ? __ldg(ap + o) : z4; ra1 = aok ? __ldg(ap + o + 4) : z4;
            rb0 = bok ? __ldg(bp + o) : z4; rb1 = bok ? __ldg(bp + o + 4) : z4;
        }
#pragma unroll
        for (int k = 0; k < GSK; k++) {
            const float4 a4 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w};
            const float2 b01 = make_float2(b4.x, b4.y), b23 = make_float2(b4.z, b4.w);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float2 a2 = make_float2(a[i], a[i]);
                acc[i][0] = dph_ffma2(a2, b01, acc[i][0]);
                acc[i][1] = dph_ffma2(a2, b23, acc[i][1]);
            }
        }
        if (kt + 1 < ktiles) {
            stash(buf ^ 1);
            __syncthreads();
            buf ^= 1;
        }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const long long rr = row0 + ty * 4 + i;
        if (rr >= n) continue;
        const long long c = col0 + tx * 4;
        float* o = out + rr * m + c;
        const float v[4] = {acc[i][0].x, acc[i][0].y, acc[i][1].x, acc[i][1].y};
        if (c + 3 < m && ((m & 3) == 0)) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        else {
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (c + j < m) o[j] = v[j];
        }
    }
}

// Few query rows (the usual case: 64 ... 2048 vectors per batch): (16 TM) x 64 tiles, TM x 4 micro-tile, 256 threads.  The k chain
// of every output is sequential by definition, so the only parallelism is across outputs: small row tiles put the batch on many
// SMs (n = 64, m = 768: 48 CTAs instead of 12) and keep several CTAs resident per SM so that the LDS -> FFMA latency of one
// warp is covered by the others.  Same arithmetic as the kernels above (one FFMA per k per output, k ascending, from +0).
#define GRK 64                      // k tile of the row-tiled kernels: half as many global round trips and barriers as 32
template <int TM>
__global__ void __launch_bounds__(256) sgemm_nt_seq_rows_kernel(const float* __restrict__ X, long long n, const float* __restrict__ W,
                                                                 long long m, int K, float* __restrict__ out) {
    constexpr int BM = 16 * TM;
    constexpr int KQ = GRK / 4;                            // float4 slots along k per row and tile
    __shared__ __align__(16) float As[2][GRK][BM];
    __shared__ __align__(16) float Bs[2][GRK][64];
    const int tid = threadIdx.x;
    const long long row0 = (long long)blockIdx.y * BM, col0 = (long long)blockIdx.x * 64;
    // thread -> (row = tid % rows, first float4 slot = tid / rows), further slots STEP apart
    constexpr int A_STEP = 256 / BM, A_PER = KQ / A_STEP;  // TM = 1: 16 / 16 = 1;  TM = 2: 16 / 8 = 2
    constexpr int B_STEP = 4, B_PER = KQ / B_STEP;         // 4
    static_assert(A_PER >= 1 && A_PER * A_STEP == KQ, "tile shape");
    const int ar = tid % BM, aq = tid / BM;
    const int br = tid & 63, bq = tid >> 6;
    const bool aok = (row0 + ar) < n, bok = (col0 + br) < m;
    const float4* ap = reinterpret_cast<const float4*>(X + (aok ? (row0 + ar) : 0) * K);
    const float4* bp = reinterpret_cast<const float4*>(W + (bok ? (col0 + br) : 0) * K);
    const int tx = tid & 15, ty = tid >> 4;
    float2 acc[TM][2];                       // float2 pairs along the output column, advanced by dph_ffma2 (see sgemm_nt_seq_kernel)
#pragma unroll
    for (int i = 0; i < TM; i++) { acc[i][0] = make_float2(0.0f, 0.0f); acc[i][1] = make_float2(0.0f, 0.0f); }
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 ra[A_PER], rb[B_PER];
    auto fetch = [&](int kt) {
#pragma unroll
        for (int i = 0; i < A_PER; i++) ra[i] = aok ? __ldg(ap + kt * KQ + aq + i * A_STEP) : z4;
#pragma unroll
        for (int i = 0; i < B_PER; i++) rb[i] = bok ? __ldg(bp + kt * KQ + bq + i * B_STEP) : z4;
    };
    auto stash = [&](int b) {
#pragma unroll
        for (int i = 0; i < A_PER; i++) {
            const int q = aq + i * A_STEP;
            As[b][q * 4 + 0][ar] = ra[i].x; As[b][q * 4 + 1][ar] = ra[i].y; As[b][q * 4 + 2][ar] = ra[i].z; As[b][q * 4 + 3][ar] = ra[i].w;
        }
#pragma unroll
        for (int i = 0; i < B_PER; i++) {
            const int q = bq + i * B_STEP;
            Bs[b][q * 4 + 0][br] = rb[i].x; Bs[b][q * 4 + 1][br] = rb[i].y; Bs[b][q * 4 + 2][br] = rb[i].z; Bs[b][q * 4 + 3][br] = rb[i].w;
        }
    };
    const int ktiles = K / GRK;
    fetch(0);
    stash(0);
    __syncthreads();
    int buf = 0;
    for (int kt = 0; kt < ktiles; kt++) {
        if (kt + 1 < ktiles) fetch(kt + 1);
#pragma unroll
        for (int k = 0; k < GRK; k++) {
            float a[TM];
#pragma unroll
            for (int i = 0; i < TM; i++) a[i] = As[buf][k][ty * TM + i];
            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float2 b01 = make_float2(b4.x, b4.y), b23 = make_float2(b4.z, b4.w);
#pragma unroll
            for (int i = 0; i < TM; i++) {
                const float2 a2 = make_float2(a[i], a[i]);
                acc[i][0] = dph_ffma2(a2, b01, acc[i][0]);
                acc[i][1] = dph_ffma2(a2, b23, acc[i][1]);
            }
        }
        if (kt + 1 < ktiles) {
            stash(buf ^ 1);
            __syncthreads();
            buf ^= 1;
        }
    }
#pragma unroll
    for (int i = 0; i < TM; i++) {
        const long long rr = row0 + ty * TM + i;
        if (rr >= n) continue;
        const long long c = col0 + tx * 4;
        float* o = out + rr * m + c;
        const float v[4] = {acc[i][0].x, acc[i][0].y, acc[i][1].x, acc[i][1].y};
        if (c + 3 < m && ((m & 3) == 0)) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        else {
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (c + j < m) o[j] = v[j];
        }
    }
}

int dph_launch_sgemm_nt_seq(const float* X, int64_t n, const float* W, int64_t m, int K, float* out, cudaStream_t st) {
    DPH_CHECK(K % GSK == 0, "sgemm_nt_seq: K must be a multiple of 32");
    if (n == 0 || m == 0) return 0;
    const bool k64 = (K % GRK) == 0;                       // the row-tiled kernels step k by 64
    dim3 grid((unsigned)((m + GBN - 1) / GBN), (unsigned)((n + GBM - 1) / GBM));
    int dev = 0, num_sms = 0;
    DPH_CUDA(cudaGetDevice(&dev));
    DPH_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    if ((long long)grid.x * grid.y >= 2 * num_sms) {
        sgemm_nt_seq_kernel<<<grid, 256, 0, st>>>(X, n, W, m, K, out);
        DPH_CUDA(cudaGetLastError());
        return 0;
    }
    // pick the LARGEST tile that still gives >= 128 CTAs: with fewer CTAs than SMs the smaller tiles' extra parallelism outweighs
    // their lower reuse
    const long long ct = (m + 63) / 64;
    if (!k64 || ct * ((n + 63) / 64) >= 128) {
        sgemm_nt_seq_small_kernel<<<dim3((unsigned)ct, (unsigned)((n + 63) / 64)), 256, 0, st>>>(X, n, W, m, K, out);
    } else if (ct * ((n + 31) / 32) >= 128) {
        sgemm_nt_seq_rows_kernel<2><<<dim3((unsigned)ct, (unsigned)((n + 31) / 32)), 256, 0, st>>>(X, n, W, m, K, out);
    } else {
        sgemm_nt_seq_rows_kernel<1><<<dim3((unsigned)ct, (unsigned)((n + 15) / 16)), 256, 0, st>>>(X, n, W, m, K, out);
    }
    DPH_CUDA(cudaGetLastError());
    return 0;
}

// =================================================================================================
// coarse_select: one CTA per query.  key = (fkey(score) << 32) | (~list)  -> distinct, order = score desc,
// list asc.  Radix-select the nprobe-th key over the S row, gather, bitonic sort, write.
// (faiss IndexFlatIP::search keeps the same SET unless scores tie exactly at the boundary; order among exact
//  ties is heap-dependent in faiss and canonicalised here.)
// =================================================================================================
__global__ void __launch_bounds__(256) coarse_select_kernel(const float* __restrict__ S, long long nlist, int nprobe,
                                                             int* __restrict__ key, float* __restrict__ cd,
                                                             unsigned long long* __restrict__ keys64, unsigned list_base, const int* __restrict__ only_rows,
                                                             long long ld) {
    if (only_rows && only_rows[blockIdx.x] == 0) return;
    __shared__ SelectScratch sc;
    __shared__ unsigned long long sel[DPH_MAX_NPROBE];
    __shared__ int cnt;
    const long long q = blockIdx.x;
    const float* row = S + q * ld;
    const int tid = threadIdx.x;
    const int take = (int)(nlist < nprobe ? nlist : nprobe);
    auto get = [&](int i) { return ((unsigned long long)dph_fkey(__ldg(row + i)) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i); };
    unsigned long long pivot = 0;
    if (nlist > nprobe) pivot = block_radix_select(get, (int)nlist, take, &sc);
    if (tid == 0) cnt = 0;
    const int p2 = dph_next_pow2(take);
    for (int i = tid; i < p2; i += blockDim.x) sel[i] = 0ull;
    __syncthreads();
    for (int i = tid; i < nlist; i += blockDim.x) {
        unsigned long long k = get(i);
        if (k >= pivot) { int p = atomicAdd(&cnt, 1); if (p < DPH_MAX_NPROBE) sel[p] = k; }
    }
    __syncthreads();
    block_bitonic_sort_desc(sel, p2);
    for (int r = tid; r < nprobe; r += blockDim.x) {
        if (keys64) {      // sharded coarse quantizer: (score key, ~global list id); 0 = empty slot
            unsigned long long k = r < take ? sel[r] : 0ull;
            if (k) k = (k & 0xFFFFFFFF00000000ull) | (unsigned long long)(0xFFFFFFFFu - ((0xFFFFFFFFu - (unsigned)k) + list_base));
            keys64[q * nprobe + r] = k;
        } else if (r < take) {
            unsigned long long k = sel[r];
            key[q * nprobe + r] = (int)(0xFFFFFFFFu - (unsigned)k);
            cd[q * nprobe + r] = dph_fkey_inv((unsigned)(k >> 32));
        } else {
            key[q * nprobe + r] = -1;
            cd[q * nprobe + r] = DPH_NEUTRAL;
        }
    }
}

// Merge of the per-shard coarse candidates (all-gathered): keys [W, n, nprobe] -> global top-nprobe per query,
// (score desc, list asc) -- bit-identical to selecting over all lists at once, because every shard computes the
// same sequential-FMA scores for its own lists.
__global__ void __launch_bounds__(256) coarse_merge_kernel(const unsigned long long* __restrict__ keys, int W, long long n, int nprobe,
                                                            int* __restrict__ key, float* __restrict__ cd, unsigned long long* __restrict__ keys64) {
    // W * nprobe candidate keys (distinct: the list id is part of the key; 0 = empty slot) -> the nprobe largest, sorted.
    // Radix-select the nprobe-th key, gather, sort only the winners (a full bitonic sort of 8 x 256 keys was 90 us per 1024 queries).
    extern __shared__ unsigned long long cm[];              // [tot] candidates, then [p2s] winners
    __shared__ SelectScratch sc;
    __shared__ int s_nz, s_cnt;
    const long long q = blockIdx.x;
    const int tot = W * nprobe, p2s = dph_next_pow2(nprobe);
    unsigned long long* sel = cm + tot;
    if (threadIdx.x == 0) { s_nz = 0; s_cnt = 0; }
    __syncthreads();
    int nz = 0;
    for (int i = threadIdx.x; i < tot; i += blockDim.x) {
        const unsigned long long k = keys[((long long)(i / nprobe) * n + q) * nprobe + (i % nprobe)];
        cm[i] = k;
        nz += k != 0ull;
    }
    for (int i = threadIdx.x; i < p2s; i += blockDim.x) sel[i] = 0ull;
    if (nz) atomicAdd(&s_nz, nz);
    __syncthreads();
    unsigned long long pivot = 1ull;                        // fewer real candidates than probes: take them all
    if (s_nz > nprobe) pivot = block_radix_select([&](int i) { return cm[i]; }, tot, nprobe, &sc);
    for (int i = threadIdx.x; i < tot; i += blockDim.x) {
        const unsigned long long k = cm[i];
        if (k >= pivot) { const int p = atomicAdd(&s_cnt, 1); if (p < p2s) sel[p] = k; }
    }
    __syncthreads();
    block_bitonic_sort_desc(sel, p2s);
    for (int r = threadIdx.x; r < nprobe; r += blockDim.x) {
        const unsigned long long k = sel[r];
        if (keys64) { keys64[q * nprobe + r] = k; continue; }       // chunked selection of tensor-core candidates: keys stay packed
        key[q * nprobe + r] = k ? (int)(0xFFFFFFFFu - (unsigned)k) : -1;
        cd[q * nprobe + r] = k ? dph_fkey_inv((unsigned)(k >> 32)) : DPH_NEUTRAL;
    }
}
int dph_launch_coarse_merge(const unsigned long long* keys, int W, int64_t n, int nprobe, int32_t* key, float* cd, cudaStream_t st,
                            unsigned long long* keys64) {
    DPH_CHECK((long long)W * nprobe <= 8192, "coarse merge: world * nprobe must be <= 8192");
    if (n == 0) return 0;
    int p2s = 1; while (p2s < nprobe) p2s <<= 1;
    const size_t smem = (size_t)(W * nprobe + p2s) * 8;
    static DphPerDeviceOnce once;
    if (once.first()) { DPH_CUDA(cudaFuncSetAttribute(coarse_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (8192 + 1024) * 8)); }
    coarse_merge_kernel<<<(unsigned)n, 256, smem, st>>>(keys, W, n, nprobe, key, cd, keys64);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

// Fast path for rows that fit shared memory (nlist <= 16384 per launch row, i.e. every sharded coarse search and C2):
// the row is staged once, keys are normalised to (key - row minimum) so the radix passes start at the first bit that
// actually varies, digits are 11 bits (<= 3 passes), and exact ties at the pivot are resolved by smallest list id.
// Same result as coarse_select_kernel (score desc, list asc).
#define CS_MAX_ROW 16384
#define CS_BINS 2048
// gridDim.y > 1: the row is cut into chunks of `chunk_len` lists, block (q, c) selects inside chunk c and writes row c * n + q of
// keys64 ([chunks, n, nprobe], the layout coarse_merge_kernel reads) with GLOBAL list numbers -- long rows (IVF65536 on one GPU, or
// the query-split coarse quantizer of the sharded search) are selected by many CTAs per query instead of one.
__global__ void __launch_bounds__(256) coarse_select_smem_kernel(const float* __restrict__ S, int nlist_total, int nprobe,
                                                                  int* __restrict__ key, float* __restrict__ cd,
                                                                  unsigned long long* __restrict__ keys64, unsigned list_base, const int* __restrict__ only_rows,
                                                                  long long ld, int chunk_len) {
    if (only_rows && only_rows[blockIdx.x] == 0) return;
    const int chunk0 = (int)blockIdx.y * chunk_len;
    const int nlist = (nlist_total - chunk0) < chunk_len ? (nlist_total - chunk0) : chunk_len;
    list_base += (unsigned)chunk0;
    extern __shared__ unsigned cs_sm[];
    unsigned* row = cs_sm;                         // [nlist] fkey(score)
    unsigned* hist = row + ((nlist + 1) & ~1);     // [2048]   (keeps `sel` 8-byte aligned)
    unsigned long long* sel = reinterpret_cast<unsigned long long*>(hist + CS_BINS);   // [1024]
    __shared__ unsigned s_min, s_max, s_digit, s_rem, s_cnt, s_ties;
    const long long q = blockIdx.x;
    const long long orow = (long long)blockIdx.y * gridDim.x + q;        // output row
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* src = S + q * ld + chunk0;
    unsigned lmin = 0xFFFFFFFFu, lmax = 0u;
    for (int i = tid; i < nlist; i += 256) { const unsigned u = dph_fkey(__ldg(src + i)); row[i] = u; lmin = min(lmin, u); lmax = max(lmax, u); }
    if (tid == 0) { s_min = 0xFFFFFFFFu; s_max = 0u; s_cnt = 0; s_ties = 0; }
    __syncthreads();
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { lmin = min(lmin, __shfl_xor_sync(0xffffffffu, lmin, off)); lmax = max(lmax, __shfl_xor_sync(0xffffffffu, lmax, off)); }
    if (lane == 0) { atomicMin(&s_min, lmin); atomicMax(&s_max, lmax); }
    __syncthreads();
    const int take = nlist < nprobe ? nlist : nprobe;
    const unsigned base = s_min, range = s_max - s_min;
    unsigned pivot = 0;                            // normalised pivot: elements with (u - base) > pivot are taken, == pivot are ties
    unsigned need_ties = 0;
    if (nlist > nprobe) {
        int top = 32 - __clz(range | 1u);          // number of significant bits of the normalised keys
        unsigned prefix = 0, mask = 0, remaining = (unsigned)take;
        for (int hi = top; hi > 0; hi -= 11) {
            const int lo = hi - 11 > 0 ? hi - 11 : 0, width = hi - lo;
            for (int i = tid; i < CS_BINS; i += 256) hist[i] = 0;
            __syncthreads();
            for (int i = tid; i < nlist; i += 256) {
                const unsigned v = row[i] - base;
                if ((v & mask) == prefix) atomicAdd(&hist[(v >> lo) & ((1u << width) - 1u)], 1u);
            }
            __syncthreads();
            {   // suffix scan over 2048 bins: 8 bins per thread, warp scan, then the 8 warp totals
                unsigned loc[8], sum = 0;
#pragma unroll
                for (int b = 0; b < 8; b++) { loc[b] = hist[tid * 8 + b]; sum += loc[b]; }
                unsigned incl = sum;
#pragma unroll
                for (int off = 1; off < 32; off <<= 1) { unsigned v = __shfl_down_sync(0xffffffffu, incl, off); if (lane + off < 32) incl += v; }
                __shared__ unsigned wtot[8];
                if (lane == 0) wtot[warp] = incl;
                __syncthreads();
                unsigned higher = 0;
#pragma unroll
                for (int w = 0; w < 8; w++) higher += (w > warp) ? wtot[w] : 0u;
                const unsigned above = higher + incl - sum;          // elements in bins above this thread's bins
                if (above < remaining && remaining <= above + sum) {
                    unsigned c = above;
#pragma unroll
                    for (int b = 7; b >= 0; b--) {
                        if (c + loc[b] >= remaining) { s_digit = tid * 8 + b; s_rem = remaining - c; break; }
                        c += loc[b];
                    }
                }
            }
            __syncthreads();
            prefix |= s_digit << lo; mask |= ((1u << width) - 1u) << lo; remaining = s_rem;
            __syncthreads();
        }
        pivot = prefix; need_ties = remaining;
    }
    const int p2 = dph_next_pow2(take);
    for (int i = tid; i < p2; i += 256) sel[i] = 0ull;
    __syncthreads();
    // strictly-above elements
    for (int i = tid; i < nlist; i += 256) {
        const unsigned v = row[i] - base;
        if (nlist <= nprobe || v > pivot) { unsigned p = atomicAdd(&s_cnt, 1u); if (p < DPH_MAX_NPROBE) sel[p] = ((unsigned long long)row[i] << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i); }
    }
    __syncthreads();
    if (nlist > nprobe) {      // ties at the pivot: the `need_ties` smallest list ids
        for (int i = tid; i < nlist; i += 256)
            if (row[i] - base == pivot) atomicAdd(&s_ties, 1u);
        __syncthreads();
        const bool all = (s_ties == need_ties);       // the usual case: exactly the needed number of elements sits at the pivot
        for (int i = tid; i < nlist; i += 256) {
            if (row[i] - base == pivot) {
                unsigned rank = 0;
                if (!all) for (int j = 0; j < i; j++) rank += (row[j] - base == pivot) ? 1u : 0u;    // rare: rank among the ties by list id
                if (rank < need_ties) { unsigned p = atomicAdd(&s_cnt, 1u); if (p < DPH_MAX_NPROBE) sel[p] = ((unsigned long long)row[i] << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i); }
            }
        }
        __syncthreads();
    }
    block_bitonic_sort_desc(sel, p2);
    for (int r = tid; r < nprobe; r += 256) {
        if (keys64) {
            unsigned long long k = r < take ? sel[r] : 0ull;
            if (k) k = (k & 0xFFFFFFFF00000000ull) | (unsigned long long)(0xFFFFFFFFu - ((0xFFFFFFFFu - (unsigned)k) + list_base));
            keys64[orow * nprobe + r] = k;
        } else if (r < take) {
            const unsigned long long k = sel[r];
            key[orow * nprobe + r] = (int)(0xFFFFFFFFu - (unsigned)k);
            cd[orow * nprobe + r] = dph_fkey_inv((unsigned)(k >> 32));
        } else { key[orow * nprobe + r] = -1; cd[orow * nprobe + r] = DPH_NEUTRAL; }
    }
}

int dph_launch_coarse_select(const float* S, int64_t n, int64_t nlist, int nprobe, int32_t* key, float* cd, cudaStream_t st,
                             unsigned long long* keys64, unsigned list_base, const int* only_rows, int64_t ld, DevBuf* tmp) {
    if (ld <= 0) ld = nlist;
    DPH_CHECK(nprobe >= 1 && nprobe <= DPH_MAX_NPROBE, "nprobe out of range [1,1024]");
    DPH_CHECK(nlist < (1ll << 31), "nlist too large");
    if (n == 0) return 0;
    if (nlist <= CS_MAX_ROW) {
        const size_t smem = (size_t)((nlist + 1) & ~1) * 4 + CS_BINS * 4 + DPH_MAX_NPROBE * 8;
        static DphPerDeviceOnce once;
        if (once.first()) { DPH_CUDA(cudaFuncSetAttribute(coarse_select_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_MAX_ROW * 4 + CS_BINS * 4 + DPH_MAX_NPROBE * 8)); }
        coarse_select_smem_kernel<<<(unsigned)n, 256, smem, st>>>(S, (int)nlist, nprobe, key, cd, keys64, list_base, only_rows, ld, (int)nlist);
        DPH_CUDA(cudaGetLastError());
        return 0;
    }
    // long rows: chunks of 8192 lists selected by one CTA each, then the per-chunk winners merged per query (same keys, same order:
    // every key carries its global list number, so the merge of the chunk winners IS the selection over the whole row)
    const int chunk_len = 8192;
    const int64_t nchunks = (nlist + chunk_len - 1) / chunk_len;
    if (tmp && !only_rows && nchunks * nprobe <= 8192 && nprobe <= chunk_len) {
        DPH_TRY(tmp->ensure((size_t)nchunks * n * nprobe * 8));
        const size_t smem = (size_t)chunk_len * 4 + CS_BINS * 4 + DPH_MAX_NPROBE * 8;
        static DphPerDeviceOnce once2;
        if (once2.first()) { DPH_CUDA(cudaFuncSetAttribute(coarse_select_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_MAX_ROW * 4 + CS_BINS * 4 + DPH_MAX_NPROBE * 8)); }
        coarse_select_smem_kernel<<<dim3((unsigned)n, (unsigned)nchunks), 256, smem, st>>>(S, (int)nlist, nprobe, nullptr, nullptr, tmp->as<unsigned long long>(),
                                                                                       list_base, nullptr, ld, chunk_len);
        DPH_CUDA(cudaGetLastError());
        return dph_launch_coarse_merge(tmp->as<unsigned long long>(), (int)nchunks, n, nprobe, key, cd, st, keys64);
    }
    coarse_select_kernel<<<(unsigned)n, 256, 0, st>>>(S, nlist, nprobe, key, cd, keys64, list_base, only_rows, ld);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

// =================================================================================================
// lut: grid (ceil(n / 4), 3), 256 threads.  Block (query group, seg) computes LUT[m][j] for m in [32 seg, 32 seg + 32), j = tid, and writes the
// canonical table in the layout of DPH_LUTC_IDX: lut_canon[q][seg][j][m % 32] (index_internal.cuh) -- 96 KB per query, the only
// fp32 table that goes to memory.  lutmax[q][m] = max_j |LUT[m][j]|, lutmin / lutmaxv = min / max over j.
// Each entry is the sequential FMA chain over the 8 sub-dimensions (compute_inner_prod_table).
// =================================================================================================
// A CTA handles one 32-sub-quantizer segment for LQ = 4 queries: every codebook entry it fetches (2 float4 per thread and
// sub-quantizer, from L2) is used for four queries, so the L2 -> SM stream is n/4 x 786 KB instead of n x 786 KB (at 1024 queries per
// batch that stream -- 805 MB -- was what the kernel's 128 us were spent on, not the 100 MB of table writes).
#define LUT_TILE_LD 257                                  // [query][sub-quantizer][code] tile, code rows padded: conflict-free both ways
// LQ = 4 queries x MS = 32 sub-quantizers per CTA (grid.y = 96 / MS).  Eight queries x 16 sub-quantizers (the same 131 KB tile, half
// the codebook stream) was no faster on one shard of C4 (1024 queries; rank step 4.499 vs 4.500 ms at nprobe 256, 1.500 vs 1.479 ms at
// nprobe 32): the kernel is bound by its per-CTA latency chain, not by the codebook stream.
__global__ void __launch_bounds__(256) lut_kernel(const float* __restrict__ xr, const float* __restrict__ pq, long long n,
                                                   float* __restrict__ lut_canon,
                                                   float* __restrict__ lutmax, float* __restrict__ lutmin, float* __restrict__ lutmaxv) {
    constexpr int LQ = 4, MS = 32;
    extern __shared__ __align__(16) float lut_sm[];
    float* __restrict__ tile = lut_sm;                    // [LQ][MS][LUT_TILE_LD]
    __shared__ __align__(16) float xs[LQ * MS * 8];       // a separate object: stores to `tile` cannot alias it, loads can be hoisted
    const long long q0 = (long long)blockIdx.x * LQ;
    const int m0 = blockIdx.y * MS, j = threadIdx.x, lane = j & 31, warp = j >> 5;
    const int nq = (int)((n - q0) < LQ ? (n - q0) : LQ);
    for (int i = j; i < LQ * MS * 8; i += 256) { const int qi = i / (MS * 8); xs[i] = qi < nq ? xr[(q0 + qi) * DPH_D + m0 * 8 + (i % (MS * 8))] : 0.0f; }
    __syncthreads();
    // software pipeline over batches of 8 sub-quantizers: the 16 codebook loads of batch b + 1 are issued before batch b is consumed
    // (loop-carried, so the scheduler cannot sink them next to their uses)
    float4 c0[8], c1[8];
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const float4* cb = reinterpret_cast<const float4*>(pq + ((size_t)(m0 + u) * 256 + j) * 8);
        c0[u] = __ldg(cb); c1[u] = __ldg(cb + 1);
    }
#pragma unroll 1
    for (int ml0 = 0; ml0 < MS; ml0 += 8) {
        float4 n0[8], n1[8];
        if (ml0 + 8 < MS) {
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const float4* cb = reinterpret_cast<const float4*>(pq + ((size_t)(m0 + ml0 + 8 + u) * 256 + j) * 8);
                n0[u] = __ldg(cb); n1[u] = __ldg(cb + 1);
            }
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int ml = ml0 + u;
#pragma unroll
            for (int qi = 0; qi < LQ; qi++) {
                const float4 x0 = *reinterpret_cast<const float4*>(xs + (qi * MS + ml) * 8);
                const float4 x1 = *reinterpret_cast<const float4*>(xs + (qi * MS + ml) * 8 + 4);
                float acc = 0.0f;                        // one sequential FMA chain over the 8 sub-dimensions (compute_inner_prod_table)
                acc = fmaf(x0.x, c0[u].x, acc); acc = fmaf(x0.y, c0[u].y, acc); acc = fmaf(x0.z, c0[u].z, acc); acc = fmaf(x0.w, c0[u].w, acc);
                acc = fmaf(x1.x, c1[u].x, acc); acc = fmaf(x1.y, c1[u].y, acc); acc = fmaf(x1.z, c1[u].z, acc); acc = fmaf(x1.w, c1[u].w, acc);
                tile[(qi * MS + ml) * LUT_TILE_LD + j] = acc;
            }
        }
#pragma unroll
        for (int u = 0; u < 8; u++) { c0[u] = n0[u]; c1[u] = n1[u]; }
    }
    __syncthreads();
    // per (query, sub-quantizer): max |entry|, min, max over the 256 codes -- one warp per pair, 8 entries per lane
    for (int p = warp; p < nq * MS; p += 8) {
        const float* row = tile + p * LUT_TILE_LD;
        float a = 0.0f, lo = row[lane], hi = lo;
#pragma unroll
        for (int e = 0; e < 8; e++) { const float v = row[lane + 32 * e]; a = fmaxf(a, fabsf(v)); lo = fminf(lo, v); hi = fmaxf(hi, v); }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, off));
            lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, off));
            hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, off));
        }
        if (lane == 0) {
            const long long o = (q0 + p / MS) * DPH_M + m0 + (p % MS);
            lutmax[o] = a; lutmin[o] = lo; lutmaxv[o] = hi;
        }
    }
    // canonical table rows [code][m % 32]: consecutive threads -> consecutive m (runs of MS floats; the tile is read column-wise)
    const int seg = m0 >> 5, mo = m0 & 31;
    for (int qi = 0; qi < nq; qi++) {
        float* dst = lut_canon + (size_t)(q0 + qi) * DPH_LUT_CANON_FLOATS + (size_t)seg * (256 * 32) + mo;
        const float* t = tile + qi * MS * LUT_TILE_LD;
        for (int idx = j; idx < 256 * MS; idx += 256) dst[(idx / MS) * 32 + (idx % MS)] = t[(idx % MS) * LUT_TILE_LD + (idx / MS)];
    }
}

// Quantised LUT for the pair-packed scan: qv[m][j] = round((LUT[m][j] - min_m) / step) in [0, 682], one step per query
// (step = max_m range_m / 682) so that 96 entries sum below 2^16 and two queries' tables can share one 32-bit word.
// Written in the scan layout ([3][256][64] u16); qparams[q] = (step, sum_m min_m).
// Quad mode (four queries per gather): the same with 8-bit entries, qv in [0, 255] (96 * 255 < 2^15), T = unsigned char, written as
// the COMPACT source of the quad scan's packed tables: [3][256][32] bytes (DPH_LUTQ8_BYTES per query), no wrap copies.  Byte m of
// row `code` is stored at m ^ ((code & 3) << 2): the table build moves 16-byte chunks of four rows at once, and this swizzle of the
// 4-byte groups inside a chunk makes its 16-byte shared-memory stores conflict-free (scan.cu, scan_quad_kernel).
#define DPH_QMAX 682
#define DPH_QMAX8 255
template <class T, int QMAX>
__global__ void __launch_bounds__(256) lutq_kernel(const float* __restrict__ lut_canon, const float* __restrict__ lutmin,
                                                    const float* __restrict__ lutmaxv, T* __restrict__ lutq,
                                                    float2* __restrict__ qparams) {
    __shared__ float tile[256 * 33];                 // the canonical segment [256 codes][32], rows padded to 33
    __shared__ float s_min[32];
    __shared__ float s_step, s_base;
    const long long q = blockIdx.x;
    const int seg = blockIdx.y, j = threadIdx.x, lane = j & 31;
    if (j < 32) {
        float r = 0.f, b = 0.f;
        for (int m = lane; m < DPH_M; m += 32) { r = fmaxf(r, lutmaxv[q * DPH_M + m] - lutmin[q * DPH_M + m]); b += lutmin[q * DPH_M + m]; }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) { r = fmaxf(r, __shfl_xor_sync(0xffffffffu, r, off)); b += __shfl_xor_sync(0xffffffffu, b, off); }
        if (lane == 0) { s_step = fmaxf(r / (float)QMAX, 1e-30f); s_base = b; }
        s_min[lane] = lutmin[q * DPH_M + seg * 32 + lane];
    }
    const float* src = lut_canon + (size_t)q * DPH_LUT_CANON_FLOATS + (size_t)seg * (256 * 32);
    for (int idx = j; idx < 256 * 32; idx += 256) tile[(idx >> 5) * 33 + (idx & 31)] = __ldg(src + idx);      // coalesced
    __syncthreads();
    const float inv = 1.0f / s_step;
    constexpr bool QUAD = sizeof(T) == 1;
    constexpr int RW = QUAD ? 32 : 64;               // row width in entries
    T* dst = lutq + ((size_t)q * 3 + seg) * (256 * RW);
    for (int idx = j; idx < 256 * RW; idx += 256) {
        const int row = idx / RW, w = idx % RW;
        const int ml = QUAD ? (w ^ ((row & 3) << 2)) : (w & 31);
        int qv = (int)((tile[row * 33 + ml] - s_min[ml]) * inv + 0.5f);
        qv = qv < 0 ? 0 : (qv > QMAX ? QMAX : qv);
        dst[idx] = (w < 63) ? (T)qv : (T)0;
    }
    if (seg == 0 && j == 0) qparams[q] = make_float2(s_step, s_base);
}

int dph_launch_lut(const float* xr, int64_t n, const float* pq, float* lut_canon, float* lutmax, float* lutmin, float* lutmaxv,
                   void* lutq, float2* qparams, cudaStream_t st, int group) {
    if (n == 0) return 0;
    static DphPerDeviceOnce lut_once;
    constexpr int lut_smem = 4 * 32 * LUT_TILE_LD * 4;        // LQ x MS = 128 (query, sub-quantizer) rows
    if (lut_once.first()) DPH_CUDA(cudaFuncSetAttribute(lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lut_smem));
    lut_kernel<<<dim3((unsigned)((n + 3) / 4), 3), 256, lut_smem, st>>>(xr, pq, n, lut_canon, lutmax, lutmin, lutmaxv);
    DPH_CUDA(cudaGetLastError());
    if (lutq) {
        if (group == 4) lutq_kernel<unsigned char, DPH_QMAX8><<<dim3((unsigned)n, 3), 256, 0, st>>>(lut_canon, lutmin, lutmaxv, (unsigned char*)lutq, qparams);
        else lutq_kernel<unsigned short, DPH_QMAX><<<dim3((unsigned)n, 3), 256, 0, st>>>(lut_canon, lutmin, lutmaxv, (unsigned short*)lutq, qparams);
        DPH_CUDA(cudaGetLastError());
    }
    return 0;
}

// =================================================================================================
// plan: (1) plan_segs -- one warp per query: segment descriptors, canonical scan positions, per-query block
// count and the fast filter's error bound eps;  (2) plan_scan -- one CTA: prefix over queries -> qpre[n+1],
// candidate-region offsets, total work; resets the per-batch counters.
// =================================================================================================
struct PlanArgs {
    const int* key; const float* cd; const int* list_len; const long long* blk_off;
    long long list_lo, list_hi; int nprobe; long long n;
    const int* only_flagged;       // nullable: plan work only for queries with flag != 0
    const float* lutmax;
    DphSeg* segs; unsigned* qblocks; int* nseg; float* eps;
    unsigned* gdense;              // nullable: canonical scan position of every (query, probe), dense [n, nprobe] (grouped modes)
    const float2* qparams;         // nullable: quantisation (step, base) -> the grouped filter's extra error term
    const DphQfView* qf;           // QF: the per-query filter's selectors (device memory)
};
// One warp per query.  Writes the COMPACTED list of in-shard, non-empty segments (probe-rank order) to
// segs[q][0..nseg[q]); gstart stays the canonical scan position over ALL probed lists (tie-break key across shards).
// QF (per-query filter, DESIGN.md 3.7): a query with a selector has as much work in a list as its selector has blocks there; a list
// with none is no segment, but its rows still count in the scan positions of the lists after it.
template <bool QF>
__global__ void __launch_bounds__(256) plan_segs_kernel(PlanArgs a) {
    const int lane = threadIdx.x & 31;
    const long long q = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (q >= a.n) return;
    int f = -1;
    if (QF) f = a.qf->assign[q];
    const bool active = a.only_flagged ? (a.only_flagged[q] != 0) : true;
    if (!active) {                                   // fallback plan: nothing to do for queries whose fast filter was proven exact
        if (lane == 0) { a.qblocks[q] = 0u; a.nseg[q] = 0; }
        return;
    }
    unsigned gacc = 0, wacc = 0;
    int sacc = 0;
    float dmax = 0.0f;
    for (int r0 = 0; r0 < a.nprobe; r0 += 32) {
        const int r = r0 + lane;
        int l = -1, len = 0; float d0 = 0.0f; unsigned nb = 0; long long blk = -1;
        if (r < a.nprobe) {
            l = a.key[q * a.nprobe + r];
            d0 = a.cd[q * a.nprobe + r];
            if (l >= 0) {
                len = a.list_len[l];
                dmax = fmaxf(dmax, fabsf(d0));
                if (active && len > 0 && l >= a.list_lo && l < a.list_hi) { nb = (unsigned)((len + 31) >> 5); blk = a.blk_off[l]; }
                if (QF && nb > 0 && f >= 0) { const uint32_t* o = a.qf->off + (long long)f * a.qf->stride + (l - a.qf->lo); nb = o[1] - o[0]; }
            }
        }
        // warp inclusive scans of len and nb
        unsigned gl = (unsigned)len, wl = nb;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            unsigned g2 = __shfl_up_sync(0xffffffffu, gl, off), w2 = __shfl_up_sync(0xffffffffu, wl, off);
            if (lane >= off) { gl += g2; wl += w2; }
        }
        if (a.gdense && r < a.nprobe) a.gdense[q * a.nprobe + r] = gacc + gl - (unsigned)len;
        const unsigned have = __ballot_sync(0xffffffffu, nb > 0);
        if (nb > 0) {
            DphSeg s;
            s.blk = blk; s.len = len; s.gstart = gacc + gl - (unsigned)len; s.dis0 = d0;
            s.wrel = wacc + wl - nb; s.wend = wacc + wl; s.list = l;
            a.segs[q * a.nprobe + sacc + __popc(have & ((1u << lane) - 1u))] = s;
        }
        sacc += __popc(have);
        gacc += __shfl_sync(0xffffffffu, gl, 31);
        wacc += __shfl_sync(0xffffffffu, wl, 31);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) dmax = fmaxf(dmax, __shfl_xor_sync(0xffffffffu, dmax, off));
    float lsum = 0.0f;
    for (int m = lane; m < DPH_M; m += 32) lsum += a.lutmax[q * DPH_M + m];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, off);
    if (lane == 0) {
        a.qblocks[q] = wacc;
        a.nseg[q] = sacc;
        // |approx - canonical| <= 2 * gamma_96 * sum|terms|,  gamma_96 = 96u/(1-96u), u = 2^-24  (Higham 2002, eq. 4.4);
        // inflated by 1.01 for the fp32 evaluation of the bound itself.
        const float gamma96 = 5.7221e-6f;
        float e = 2.0f * gamma96 * (dmax + lsum) * 1.01f;
        // grouped modes: every quantised entry is within 0.5 step of the fp32 entry (+ rounding of the dequantisation) -> 96 * 0.502 * step
        if (a.qparams) e += 96.0f * 0.502f * a.qparams[q].x + 8e-6f * (dmax + lsum);
        a.eps[q] = e;
    }
}

struct PlanScanArgs {
    const unsigned* qblocks; long long n; int keep; int grid;
    long long* qpre; long long* cand_off; int* cand_cnt; unsigned* gthr; DphWork* work;
    const DphGroupWork* groupwork; const int* nseg;   // grouped modes (nullable): a query is flushed once per (list, segment) unit it is part of
};
__global__ void __launch_bounds__(1024) plan_scan_kernel(PlanScanArgs a) {
    __shared__ long long wsum[32];
    __shared__ long long carry, total;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // pass 1: qpre = exclusive prefix of qblocks
    if (tid == 0) carry = 0;
    __syncthreads();
    for (long long base = 0; base < a.n; base += 1024) {
        long long q = base + tid;
        long long v = q < a.n ? (long long)a.qblocks[q] : 0, incl = v;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { long long t = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += t; }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            long long w = wsum[lane], wi = w;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) { long long t = __shfl_up_sync(0xffffffffu, wi, off); if (lane >= off) wi += t; }
            wsum[lane] = wi - w;
        }
        __syncthreads();
        long long excl = carry + wsum[warp] + incl - v;
        if (q < a.n) { a.qpre[q] = excl; a.cand_cnt[q] = 0; a.gthr[q] = 0u; }
        __syncthreads();
        if (tid == 1023) carry = excl + v;
        __syncthreads();
    }
    if (tid == 0) { total = carry; a.qpre[a.n] = carry; a.work->total_blocks = carry; carry = 0; }
    __syncthreads();
    // pass 2: candidate-region offsets; a query spanning `parts` scan CTAs or units may receive parts*keep entries.  The area these
    // regions share is sized by the bound on the batch's sum of parts derived at search.cu: cand_entries.
    const long long T = total;
    const long long per = a.groupwork ? a.groupwork->per : (T / a.grid > 0 ? T / a.grid : 1);
    for (long long base = 0; base < a.n; base += 1024) {
        long long q = base + tid;
        long long v = 0;
        if (q < a.n) {
            long long qb = (long long)a.qblocks[q];
            if (qb > 0) {
                long long parts = qb / per + 2;
                if (a.groupwork) parts = (long long)a.nseg[q] + qb / per + 1;        // sum over its lists of ceil(blocks / segment)
                else if (parts > a.grid) parts = a.grid;
                v = parts * a.keep;
            }
        }
        long long incl = v;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { long long t = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += t; }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            long long w = wsum[lane], wi = w;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) { long long t = __shfl_up_sync(0xffffffffu, wi, off); if (lane >= off) wi += t; }
            wsum[lane] = wi - w;
        }
        __syncthreads();
        long long excl = carry + wsum[warp] + incl - v;
        if (q < a.n) a.cand_off[q] = excl;
        __syncthreads();
        if (tid == 1023) carry = excl + v;
        __syncthreads();
    }
    if (tid == 0) a.cand_off[a.n] = carry;
}

// =================================================================================================
// group plan (pair and quad modes): invert (query -> probed lists) into (list -> probing queries), group the probes of each list
// into work items of gsz queries, and emit the work queue of the grouped scan kernels: units (list, block segment, item), items of
// the same list segment ADJACENT in the queue.  The scan CTAs pull units in queue order, so the items of a list are scanned at the
// same time by different CTAs and all but the first reader of a code block hit L2 instead of HBM.
// =================================================================================================
struct GroupPlanArgs {
    const int* key; long long nq_probes; int nprobe; const int* list_len; long long list_lo, list_hi, nlist; int grid;
    int* cnt; int* fill; int* off; long long* blockpre; unsigned* entries; DphGroupWork* work;
    int* unitpre; unsigned long long* units;
    int gsz;                       // queries per work item: 2 (pair-packed scan) or DPH_QUAD_ITEM_Q (quad-packed scan)
    DphUnit* udesc;                // quad mode (nullable): resolved unit descriptors, parallel to `units`
    const long long* blk_off; const float* cd; const unsigned* gdense; const float2* qparams;
};
__global__ void group_count_kernel(GroupPlanArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.nq_probes) return;
    const int l = a.key[i];
    if (l >= a.list_lo && l < a.list_hi && a.list_len[l] > 0) atomicAdd(&a.cnt[l], 1);
}
__global__ void __launch_bounds__(1024) group_scan_kernel(GroupPlanArgs a) {
    __shared__ long long wsa[32], wsb[32];
    __shared__ long long ca, cb;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { ca = 0; cb = 0; }
    __syncthreads();
    for (long long base = a.list_lo; base < a.list_hi; base += 1024) {
        const long long l = base + tid;
        long long va = 0, vb = 0;
        if (l < a.list_hi) {
            const int c = a.cnt[l];
            va = c;
            vb = (long long)((c + a.gsz - 1) / a.gsz) * (long long)((a.list_len[l] + 31) >> 5);
        }
        long long ia = va, ib = vb;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            long long t1 = __shfl_up_sync(0xffffffffu, ia, off), t2 = __shfl_up_sync(0xffffffffu, ib, off);
            if (lane >= off) { ia += t1; ib += t2; }
        }
        if (lane == 31) { wsa[warp] = ia; wsb[warp] = ib; }
        __syncthreads();
        if (warp == 0) {
            long long w1 = wsa[lane], w2 = wsb[lane], i1 = w1, i2 = w2;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                long long t1 = __shfl_up_sync(0xffffffffu, i1, off), t2 = __shfl_up_sync(0xffffffffu, i2, off);
                if (lane >= off) { i1 += t1; i2 += t2; }
            }
            wsa[lane] = i1 - w1; wsb[lane] = i2 - w2;
        }
        __syncthreads();
        const long long ea = ca + wsa[warp] + ia - va, eb = cb + wsb[warp] + ib - vb;
        if (l < a.list_hi) { a.off[l] = (int)ea; a.blockpre[l] = eb; }
        __syncthreads();
        if (tid == 1023) { ca = ea + va; cb = eb + vb; }
        __syncthreads();
    }
    __shared__ long long segb_s;
    if (tid == 0) {
        a.off[a.list_hi] = (int)ca; a.blockpre[a.list_hi] = cb;
        long long segb = (cb + (long long)a.grid * DPH_GROUP_UNITS_PER_CTA - 1) / ((long long)a.grid * DPH_GROUP_UNITS_PER_CTA);
        if (segb < DPH_GROUP_SEG_MIN) segb = DPH_GROUP_SEG_MIN;
        a.work->total_blocks = cb;
        a.work->per = segb;
        segb_s = segb; ca = 0;
    }
    __syncthreads();
    // second pass: units per list = items x segments -> unitpre (exclusive prefix)
    const long long segb = segb_s;
    for (long long base = a.list_lo; base < a.list_hi; base += 1024) {
        const long long l = base + tid;
        long long va = 0;
        if (l < a.list_hi) {
            const long long nb = (a.list_len[l] + 31) >> 5;
            va = (long long)((a.cnt[l] + a.gsz - 1) / a.gsz) * ((nb + segb - 1) / segb);
        }
        long long ia = va;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { long long t1 = __shfl_up_sync(0xffffffffu, ia, off); if (lane >= off) ia += t1; }
        if (lane == 31) wsa[warp] = ia;
        __syncthreads();
        if (warp == 0) {
            long long w1 = wsa[lane], i1 = w1;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) { long long t1 = __shfl_up_sync(0xffffffffu, i1, off); if (lane >= off) i1 += t1; }
            wsa[lane] = i1 - w1;
        }
        __syncthreads();
        const long long ea = ca + wsa[warp] + ia - va;
        if (l < a.list_hi) a.unitpre[l] = (int)ea;
        __syncthreads();
        if (tid == 1023) ca = ea + va;
        __syncthreads();
    }
    if (tid == 0) { a.work->total_units = (int)ca; a.work->next_unit = 0; }
}
// one thread per list: unit = list | item << 32 | segment << 48, ordered (segment, item) inside the list; quad mode also gets the
// resolved descriptor of every unit (DphUnit)
__global__ void group_units_kernel(GroupPlanArgs a) {
    const long long l = a.list_lo + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= a.list_hi) return;
    const int cnt = a.cnt[l];
    const int items = (cnt + a.gsz - 1) / a.gsz;
    if (items == 0) return;
    const long long segb = a.work->per, nb = (a.list_len[l] + 31) >> 5;
    const int nsegs = (int)((nb + segb - 1) / segb);
    const long long u0 = a.unitpre[l];
    for (int it = 0; it < items; it++) {
        DphUnit d;
        if (a.udesc) {
            d.blk = a.blk_off[l]; d.len = a.list_len[l]; d.list = (int)l; d.pad = 0;
            d.nq = min(a.gsz, cnt - a.gsz * it);
            const int e0 = a.off[l] + a.gsz * it;
#pragma unroll
            for (int i = 0; i < DPH_QUAD_ITEM_Q; i++) {
                const unsigned e = a.entries[e0 + (i < d.nq ? i : 0)];
                const long long q = e >> 10; const int r = (int)(e & 1023u);
                const float2 pp = a.qparams[q];
                d.q[i] = (unsigned)q; d.gs[i] = a.gdense[q * a.nprobe + r];
                d.base[i] = a.cd[q * a.nprobe + r] + pp.y; d.step[i] = pp.x;
            }
        }
        for (int s = 0; s < nsegs; s++) {
            const long long u = u0 + (long long)s * items + it;
            a.units[u] = (unsigned long long)l | ((unsigned long long)it << 32) | ((unsigned long long)s << 48);
            if (a.udesc) {
                d.bi0 = (unsigned)(s * segb);
                d.bend = (unsigned)((nb - (long long)d.bi0 < segb) ? nb : (long long)d.bi0 + segb);
                a.udesc[u] = d;
            }
        }
    }
}
__global__ void group_fill_kernel(GroupPlanArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.nq_probes) return;
    const int l = a.key[i];
    if (l >= a.list_lo && l < a.list_hi && a.list_len[l] > 0) {
        const int pos = a.off[l] + atomicAdd(&a.fill[l], 1);
        a.entries[pos] = (unsigned)((i / a.nprobe) << 10) | (unsigned)(i % a.nprobe);
    }
}

int dph_launch_plan(dph_index* ix, const DphSearchPlan& sp, const DphCodeSrc& src, int64_t n, bool exact, const int32_t* only_flagged,
                    cudaStream_t st) {
    const int group = sp.pass_group(exact);
    const bool grouped = group > 1;
    if (n == 0) return 0;
    PlanArgs a;
    a.key = ix->key.as<int>(); a.cd = ix->cd.as<float>(); a.list_len = ix->list_len; a.blk_off = src.blk_off;
    a.list_lo = src.lo; a.list_hi = src.hi; a.nprobe = ix->nprobe; a.n = n; a.only_flagged = only_flagged;
    a.lutmax = ix->lutmax.as<float>(); a.segs = ix->segs.as<DphSeg>(); a.qblocks = ix->qinfo.as<unsigned>(); a.nseg = ix->nseg.as<int>(); a.eps = ix->eps.as<float>();
    a.gdense = grouped ? ix->gdense.as<unsigned>() : nullptr; a.qparams = grouped ? ix->qparams.as<float2>() : nullptr;
    a.qf = src.qf;
    if (src.qf) plan_segs_kernel<true><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(a);
    else plan_segs_kernel<false><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(a);
    DPH_CUDA(cudaGetLastError());
    if (grouped) {
        GroupPlanArgs p;
        p.key = ix->key.as<int>(); p.nq_probes = n * ix->nprobe; p.nprobe = ix->nprobe; p.list_len = ix->list_len; p.list_lo = src.lo;
        p.list_hi = src.hi; p.nlist = ix->nlist; p.grid = sp.grid; p.cnt = ix->grp_cnt.as<int>(); p.fill = ix->grp_fill.as<int>();
        p.off = ix->grp_off.as<int>(); p.blockpre = ix->grp_blockpre.as<long long>(); p.entries = ix->grp_entries.as<unsigned>();
        p.work = ix->groupwork.as<DphGroupWork>(); p.unitpre = ix->grp_unitpre.as<int>(); p.units = ix->grp_units.as<unsigned long long>();
        p.gsz = sp.item_q;
        p.udesc = group == 4 ? ix->grp_udesc.as<DphUnit>() : nullptr;
        p.blk_off = src.blk_off; p.cd = ix->cd.as<float>(); p.gdense = ix->gdense.as<unsigned>(); p.qparams = ix->qparams.as<float2>();
        DPH_CUDA(cudaMemsetAsync(p.cnt, 0, (size_t)ix->nlist * 4, st));
        DPH_CUDA(cudaMemsetAsync(p.fill, 0, (size_t)ix->nlist * 4, st));
        const unsigned nb = (unsigned)((p.nq_probes + 255) / 256);
        group_count_kernel<<<nb, 256, 0, st>>>(p);
        group_scan_kernel<<<1, 1024, 0, st>>>(p);
        group_fill_kernel<<<nb, 256, 0, st>>>(p);
        if (src.hi > src.lo) group_units_kernel<<<(unsigned)((src.hi - src.lo + 255) / 256), 256, 0, st>>>(p);
        DPH_CUDA(cudaGetLastError());
    }
    PlanScanArgs b;
    b.groupwork = grouped ? ix->groupwork.as<DphGroupWork>() : nullptr; b.nseg = ix->nseg.as<int>();
    b.qblocks = ix->qinfo.as<unsigned>(); b.n = n; b.keep = sp.pass_keep(exact); b.grid = sp.grid; b.qpre = ix->wpre.as<long long>();
    b.cand_off = ix->cand_off.as<long long>(); b.cand_cnt = ix->cand_cnt.as<int>(); b.gthr = ix->gthr.as<unsigned>();
    b.work = ix->work.as<DphWork>();
    plan_scan_kernel<<<1, 1024, 0, st>>>(b);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

// C ABI: out [n,m] = X [n,K] . W [m,K]^T with one sequential fp32 FMA chain per output (the oracle's inner-product definition).
DPH_API int dph_sgemm_nt_seq(const float* X, int64_t n, const float* W, int64_t m, int64_t K, float* out, void* cuda_stream) {
    return dph_launch_sgemm_nt_seq(X, n, W, m, (int)K, out, (cudaStream_t)cuda_stream);
}
