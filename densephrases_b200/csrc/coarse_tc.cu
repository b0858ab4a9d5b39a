// coarse_tc.cu -- coarse quantizer (faiss IndexFlatIP top-nprobe, reference call site densephrases/index.py:200) on the tensor
// cores WITHOUT giving up the bit-exact sequential-FMA definition of the scores (oracle/ivfpq_ref.c):
//   1. approximate scores  S~ = xr . C^T  with the 3xTF32 wgmma GEMM (gemm_tf32.cu), error <= B(q) = c |xr_q| max_l |C_l| plus an
//      absolute term for subnormal operands, products and sums (tiny queries), norms in fp64;
//   2. candidates = top-(nprobe + margin) of S~ per query;
//   3. candidates are re-scored EXACTLY (one sequential fp32 FMA chain each, identical to sgemm_nt_seq / the oracle);
//   4. top-nprobe of the exact scores, (score desc, list asc); the result is provably the global top-nprobe when
//      (smallest candidate S~) + B < (nprobe-th exact score): every non-candidate has exact <= S~ + B < the nprobe-th score;
//   5. otherwise the query is repaired: exact scores for ALL lists of the shard, then the ordinary selection (rare).
// The FLOPs move from ~35 TFLOP/s SIMT FFMA to the tensor pipe; the selected probes and their scores stay bit-identical.
#include "index_internal.cuh"
#include "select.cuh"

int dph_launch_gemm_tf32(int group, const float* const* A, const float* const* W, const float* const* bias, const float* const* residual,
                         float* const* out, int M, int N, int K, int act, cudaStream_t st, const float* const* A_lo, const float* const* W_lo);
int dph_launch_split_tf32(const float* x, float* hi, float* lo, long long n, cudaStream_t st);

// One exact sequential-FMA dot product per thread: the thread streams its own centroid row (16-byte loads, consecutive addresses,
// so every fetched sector is fully used through L1) against the query row in shared memory (broadcast reads).  t ascending, one FFMA
// per element -- the same chain as sgemm_nt_seq and oracle/ivfpq_ref.c:dot_seq.
__device__ __forceinline__ float thread_exact_dot(const float* __restrict__ C, const float* xq, long long li) {
    if (li < 0) return 0.0f;
    const float4* row = reinterpret_cast<const float4*>(C + li * DPH_D);
    float acc = 0.0f;
    // explicit batches of 16 row loads in flight per thread (with one CTA per query and 64 ... 375 busy threads the kernel is L2-latency
    // bound); the FMA chain itself stays t-ascending
#pragma unroll 1
    for (int t0 = 0; t0 < DPH_D / 4; t0 += 16) {
        float4 c[16];
#pragma unroll
        for (int e = 0; e < 16; e++)        // volatile asm: the optimiser otherwise sinks every load next to its use (two in flight)
            asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(c[e].x), "=f"(c[e].y), "=f"(c[e].z), "=f"(c[e].w) : "l"(row + t0 + e));
#pragma unroll
        for (int e = 0; e < 16; e++) {
            const int t4 = t0 + e;
            acc = fmaf(xq[4 * t4 + 0], c[e].x, acc);
            acc = fmaf(xq[4 * t4 + 1], c[e].y, acc);
            acc = fmaf(xq[4 * t4 + 2], c[e].z, acc);
            acc = fmaf(xq[4 * t4 + 3], c[e].w, acc);
        }
    }
    return acc;
}

struct CoarseTcArgs {
    const float* xr; const float* C; const float* Sapprox; long long nl; int ncand; int nprobe; unsigned list_base;
    const unsigned long long* cand_keys;     // [n, ncand] (approx score key << 32 | ~local list), 0 = empty
    const float* cnorm_max;                  // scalar: max_l |C_l| over the shard
    unsigned long long* keys64; int* key; float* cd;    // outputs (either keys64 or key/cd)
    int* flags; float* S_exact;              // repair: flags [n], S_exact [n, nl]
};

// one CTA per query: exact re-score of the candidates, final selection, proof.
__global__ void __launch_bounds__(256, 3) coarse_tc_finish_kernel(CoarseTcArgs a) {     // <= 85 registers: room for 16 row loads in flight
    __shared__ float xq[DPH_D];
    __shared__ unsigned long long sel[DPH_MAX_NPROBE];
    __shared__ double red[8];
    const long long q = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // |xr_q| in fp64: the fp32 squares of a query with |xr| below ~2^-75 underflow (the norm would be 0 and so would the bound), and
    // above ~2^64 they overflow
    double n2 = 0.0;
    for (int t = tid; t < DPH_D; t += 256) { const float v = a.xr[q * DPH_D + t]; xq[t] = v; n2 = fma((double)v, (double)v, n2); }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, off);
    if (lane == 0) red[warp] = n2;
    const int p2 = dph_next_pow2(a.ncand);
    for (int i = tid; i < p2; i += 256) sel[i] = 0ull;
    __syncthreads();
    unsigned amin_key = 0xFFFFFFFFu;          // smallest approximate score among the candidates
    for (int c = tid; c < a.ncand; c += 256) {
        const unsigned long long ck = a.cand_keys[q * a.ncand + c];
        const long long li = ck ? (long long)(0xFFFFFFFFu - (unsigned)ck) : -1;
        const float ex = thread_exact_dot(a.C, xq, li);
        if (ck) {
            sel[c] = ((unsigned long long)dph_fkey(ex) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)li);
            amin_key = min(amin_key, (unsigned)(ck >> 32));
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) amin_key = min(amin_key, __shfl_xor_sync(0xffffffffu, amin_key, off));
    __shared__ unsigned s_amin;
    if (tid == 0) s_amin = 0xFFFFFFFFu;
    __syncthreads();
    if (lane == 0) atomicMin(&s_amin, amin_key);
    __syncthreads();
    block_bitonic_sort_desc(sel, p2);
    const int take = (int)(a.nl < a.nprobe ? a.nl : a.nprobe);
    // proof: the candidate set is complete unless a non-candidate could reach the nprobe-th exact score
    int flag = 0;
    if (a.nl > a.ncand) {
        // relative part: >= 3 K 2^-23 |x||c| (3xTF32 products + fp32 accumulation), K = 768, valid while every split operand,
        // product and partial sum is a normal number.  Absolute part: a subnormal operand, product or partial sum that the tensor
        // cores flush is off by less than 2^-126 (times the other operand): <= 2^-126 (3 sqrt(K) (|x| + |c|) + 4 K), doubled.
        double qn = 0.0;
#pragma unroll
        for (int w = 0; w < 8; w++) qn += red[w];
        qn = sqrt(qn);
        const double cn = *a.cnorm_max;
        const double bound = 3.0e-4 * qn * cn + 0x1p-125 * (3.0 * 27.72 * (qn + cn) + 4.0 * DPH_D);
        const double amin = dph_fkey_inv(s_amin);
        const double te = dph_fkey_inv((unsigned)(sel[take - 1] >> 32));
        if (!(amin + bound < te)) flag = 1;
    }
    if (tid == 0) a.flags[q] = flag;
    if (flag) return;                                            // repaired by coarse_tc_repair_kernel + the exact selection
    for (int r = tid; r < a.nprobe; r += 256) {
        const unsigned long long k = r < take ? sel[r] : 0ull;
        if (a.keys64) a.keys64[q * a.nprobe + r] = k ? ((k & 0xFFFFFFFF00000000ull) | (unsigned long long)(0xFFFFFFFFu - ((0xFFFFFFFFu - (unsigned)k) + a.list_base))) : 0ull;
        else { a.key[q * a.nprobe + r] = k ? (int)(0xFFFFFFFFu - (unsigned)k) : -1; a.cd[q * a.nprobe + r] = k ? dph_fkey_inv((unsigned)(k >> 32)) : DPH_NEUTRAL; }
    }
}

// flagged queries only: exact scores for every list of the shard (same chain as sgemm_nt_seq), written to S_exact[q].
__global__ void __launch_bounds__(256, 3) coarse_tc_repair_kernel(CoarseTcArgs a) {
    const long long q = blockIdx.x;
    if (a.flags[q] == 0) return;
    __shared__ float xq[DPH_D];
    const int tid = threadIdx.x;
    for (int t = tid; t < DPH_D; t += 256) xq[t] = a.xr[q * DPH_D + t];
    __syncthreads();
    for (long long li = tid; li < a.nl; li += 256) a.S_exact[q * a.nl + li] = thread_exact_dot(a.C, xq, li);
}

__global__ void cnorm_max_kernel(const float* C, long long nl, float* out) {
    // max_l |C_l|^2 -> sqrt, in fp64 and rounded up to fp32 (no underflow of tiny centroids); one warp per list, atomicMax on the
    // (non-negative) float bits
    const long long l = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (l >= nl) return;
    double s = 0.0;
    for (int t = lane; t < DPH_D; t += 32) { const double v = C[l * DPH_D + t]; s = fma(v, v, s); }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) atomicMax(reinterpret_cast<unsigned*>(out), __float_as_uint(__double2float_ru(sqrt(s))));
}

// Coarse top-nprobe over lists [lo, lo+nl) of the index.  Writes keys64 (sharded path) or key/cd.  Returns 1 if the tensor-core
// path does not apply to this shape (caller uses the SIMT path).  xr / C: the rotated rows [n, d] and the centroids [nlist, d]
// (nullptr: the index's xr workspace and centroids).  The (hi, lo) centroid split is cached by list range: a caller that passes other
// centroids, or changes them, sets ix->csplit_lo = -1 first.
int dph_coarse_tc(dph_index* ix, int64_t n, int64_t lo, int64_t nl, int nprobe, unsigned long long* keys64, int32_t* key, float* cd, cudaStream_t st,
                  const float* xr, const float* C) {
    const int margin = nprobe / 4 > 32 ? nprobe / 4 : 32;
    const int ncand = (int)std::min<int64_t>(nprobe + margin, nl);
    // pays for small probe counts; at nprobe 256 the exact re-rank of 320 candidates costs about what the tensor cores save, so the
    // SIMT GEMM is kept there.  With many lists per candidate (131 072 lists per shard, 320 candidates) the GEMM dominates again
    // and the tensor cores win.  Compare both paths with tools/bench_shard.py.
    const bool few_candidates = ncand <= 160 && nl > 4 * (int64_t)ncand;
    const bool many_lists = nl >= 32 * (int64_t)ncand;
    if (ncand > DPH_MAX_NPROBE || n < 32 || !(few_candidates || many_lists)) return 1;
    const int64_t nlp = (nl + 127) / 128 * 128;          // GEMM N must be a multiple of the 128-wide tile: zero-padded centroid rows
    if ((size_t)n * nlp * 4 > ix->S.cap) return 1;
    const float* Cl = (C ? C : ix->C) + lo * DPH_D;
    const float* X = xr ? xr : ix->xr.as<float>();
    if (!ix->csplit.p || ix->csplit_lo != lo || ix->csplit_nl != nl) {          // (hi, lo) TF32 split of the shard's centroids + max norm, once
        DPH_TRY(ix->csplit.ensure((size_t)nlp * DPH_D * 8 + 16));
        float* hi = ix->csplit.as<float>();
        DPH_CUDA(cudaMemsetAsync(hi, 0, (size_t)nlp * DPH_D * 8, st));
        DPH_TRY(dph_launch_split_tf32(Cl, hi, hi + nlp * DPH_D, nl * DPH_D, st));
        float* nm = hi + 2 * nlp * DPH_D;
        DPH_CUDA(cudaMemsetAsync(nm, 0, 4, st));
        cnorm_max_kernel<<<(unsigned)((nl + 7) / 8), 256, 0, st>>>(Cl, nl, nm);
        DPH_CUDA(cudaGetLastError());
        ix->csplit_lo = lo; ix->csplit_nl = nl;
    }
    float* chi = ix->csplit.as<float>(); float* clo = chi + nlp * DPH_D; float* cnorm = chi + 2 * nlp * DPH_D;
    DPH_TRY(ix->xsplit.ensure((size_t)n * DPH_D * 8));
    DPH_TRY(ix->candkeys.ensure((size_t)n * ncand * 8));
    DPH_TRY(ix->cflags.ensure((size_t)n * 4));
    float* xhi = ix->xsplit.as<float>(); float* xlo = xhi + n * DPH_D;
    DPH_TRY(dph_launch_split_tf32(X, xhi, xlo, n * DPH_D, st));
    const float* A1[1] = {xhi}; const float* W1[1] = {chi}; const float* A2[1] = {xlo}; const float* W2[1] = {clo}; float* O1[1] = {ix->S.as<float>()};
    DPH_TRY(dph_launch_gemm_tf32(1, A1, W1, nullptr, nullptr, O1, (int)n, (int)nlp, DPH_D, 0, st, A2, W2));
    DPH_TRY(dph_launch_coarse_select(ix->S.as<float>(), n, nl, ncand, nullptr, nullptr, st, ix->candkeys.as<unsigned long long>(), 0u, nullptr, nlp, &ix->selkeys));
    CoarseTcArgs a;
    a.xr = X; a.C = Cl; a.Sapprox = ix->S.as<float>(); a.nl = nl; a.ncand = ncand; a.nprobe = nprobe; a.list_base = (unsigned)lo;
    a.cand_keys = ix->candkeys.as<unsigned long long>(); a.cnorm_max = cnorm; a.keys64 = keys64; a.key = key; a.cd = cd;
    a.flags = ix->cflags.as<int>(); a.S_exact = ix->S.as<float>();       // repaired rows are rewritten with stride nl (the approximate scores are dead by then)
    coarse_tc_finish_kernel<<<(unsigned)n, 256, 0, st>>>(a);
    coarse_tc_repair_kernel<<<(unsigned)n, 256, 0, st>>>(a);
    DPH_CUDA(cudaGetLastError());
    // exact selection for repaired rows only (rows with flag 0 exit immediately and keep the keys written above)
    DPH_TRY(dph_launch_coarse_select(ix->S.as<float>(), n, nl, nprobe, key, cd, st, keys64, (unsigned)lo, ix->cflags.as<int>()));
    return 0;
}
