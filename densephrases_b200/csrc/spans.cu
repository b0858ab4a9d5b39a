// spans.cu -- span decoding of single-passage reading (compute_predictions_logits, reference densephrases/utils/squad_metrics.py:408-684):
// for every example, the first K prelim candidates (feature, start, end) in the reference's order, the counts of valid spans
// before and after the filter test, and the version-2 null choice.
//
// Enumeration (per feature, as the reference's double loop):  start in [0, n_tokens), end in [start, min(n_tokens, start + L - 1));
//   a span is valid when start_ok[start] (in token_to_orig_map and token_is_max_context) and end_ok[end] (in token_to_orig_map);
//   it passes the filter unless double(sft[start]) < thr or double(eft[end]) < thr;
//   its score is double(start[start]) + double(end[end]) (Python float addition).
// Order: score descending, ties in enumeration order (feature, start, end) -- Python's stable sorted(..., reverse=True).
//
// One CTA per example.  Each feature's four logit rows and two masks are staged in shared memory once; a thread owns a start
// index and walks its ends one step per round.  A candidate that beats the current K-th entry is appended to a shared buffer;
// when the buffer can no longer take a full round, it is sorted (bitonic, on (ordered score bits desc, enumeration index asc))
// and cut to K, and the K-th entry becomes the new bar.  No candidate array leaves the SM.
#include "common.cuh"
#include "../../include/dph_b200.h"
#include <vector>

#define RC_THREADS 256
#define RC_MAX_S 512
#define RC_MAX_L 64          // end - start <= L - 2 < 64: six bits of the enumeration index
#define RC_MAX_K 1024

struct SpanArgs {
    const float *st, *en, *sft, *eft;        // [F,S]
    const int* ntok;                         // [F]
    const unsigned *sok, *eok;               // [F,W] bit masks, W = ceil(S / 32)
    const long long* off;                    // [E+1]
    int S, W, L, K, v2, cap;
    double thr;
    int* cand;                               // [E,K,3] (feature within the example, start, end)
    int* ncand;                              // [E]
    long long *total, *vec;                  // [E]
    int* null_feat;                          // [E] feature within the example, -1 when no feature scores below 1e6
    float* null_logit;                       // [E,2]
};

// total order on doubles as unsigned integers (larger = better); -0.0 is folded onto +0.0 first, as Python compares them equal
__device__ __forceinline__ unsigned long long rc_key(double x) {
    if (x == 0.0) x = 0.0;
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ bool rc_better(unsigned long long ka, unsigned ia, unsigned long long kb, unsigned ib) {
    return ka > kb || (ka == kb && ia < ib);
}

// sort buf[0, cap) best first; entries at [n, cap) are padded with the worst key first
__device__ void rc_sort(unsigned long long* key, unsigned* idx, int n, int cap) {
    for (int i = n + threadIdx.x; i < cap; i += blockDim.x) { key[i] = 0ull; idx[i] = 0xffffffffu; }
    __syncthreads();
    for (int k = 2; k <= cap; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < cap; i += blockDim.x) {
                const int p = i ^ j;
                if (p > i) {
                    const bool first_better = rc_better(key[i], idx[i], key[p], idx[p]);
                    if (((i & k) == 0) != first_better) {          // ascending half of the network keeps the better entry first
                        const unsigned long long tk = key[i]; key[i] = key[p]; key[p] = tk;
                        const unsigned ti = idx[i]; idx[i] = idx[p]; idx[p] = ti;
                    }
                }
            }
            __syncthreads();
        }
}

__global__ void __launch_bounds__(RC_THREADS) rc_spans_kernel(SpanArgs a) {
    extern __shared__ __align__(16) unsigned char rc_smem[];
    const int S = a.S, W = a.W, cap = a.cap, tid = threadIdx.x;
    unsigned long long* key = reinterpret_cast<unsigned long long*>(rc_smem);          // [cap]
    unsigned* idx = reinterpret_cast<unsigned*>(key + cap);                              // [cap]
    float* st = reinterpret_cast<float*>(idx + cap);                                     // [S] x 4
    float* en = st + S; float* sf = en + S; float* ef = sf + S;
    unsigned* sok = reinterpret_cast<unsigned*>(ef + S);                                 // [W] x 2
    unsigned* eok = sok + W;
    __shared__ int n_buf;
    __shared__ unsigned long long bar_key;
    __shared__ unsigned bar_idx;
    __shared__ int have_bar;
    __shared__ long long red[2][RC_THREADS / 32];
    const int ex = blockIdx.x;
    const long long f0 = a.off[ex], f1 = a.off[ex + 1];
    if (tid == 0) { n_buf = 0; have_bar = 0; bar_key = 0ull; bar_idx = 0u; }
    long long my_total = 0, my_vec = 0;
    const int steps = a.L - 1;
    for (long long f = f0; f < f1; f++) {
        __syncthreads();                     // previous feature's rows are no longer read
        for (int i = tid; i < S; i += RC_THREADS) {
            st[i] = a.st[f * S + i]; en[i] = a.en[f * S + i]; sf[i] = a.sft[f * S + i]; ef[i] = a.eft[f * S + i];
        }
        for (int i = tid; i < W; i += RC_THREADS) { sok[i] = a.sok[f * W + i]; eok[i] = a.eok[f * W + i]; }
        __syncthreads();
        const int n = a.ntok[f];
        const unsigned fbase = (unsigned)(f - f0) * (unsigned)S;
        for (int s0 = 0; s0 < n; s0 += RC_THREADS) {
            const int s = s0 + tid;
            const bool s_ok = s < n && ((sok[s >> 5] >> (s & 31)) & 1u);
            const double ss = s_ok ? (double)st[s] : 0.0;
            const bool s_pass = s_ok && !((double)sf[s] < a.thr);
            for (int j = 0; j < steps; j++) {
                const int e = s + j;
                if (s_ok && e < n && ((eok[e >> 5] >> (e & 31)) & 1u)) {
                    my_total++;
                    if (s_pass && !((double)ef[e] < a.thr)) {
                        my_vec++;
                        const unsigned long long k = rc_key(ss + (double)en[e]);
                        const unsigned id = ((fbase + (unsigned)s) << 6) | (unsigned)j;
                        if (!have_bar || rc_better(k, id, bar_key, bar_idx)) {
                            const int slot = atomicAdd(&n_buf, 1);
                            key[slot] = k; idx[slot] = id;
                        }
                    }
                }
                __syncthreads();
                if (n_buf > cap - RC_THREADS) {          // the next round might not fit: cut the buffer to the best K
                    rc_sort(key, idx, n_buf, cap);
                    if (tid == 0) {
                        n_buf = min(n_buf, a.K);
                        if (n_buf == a.K) { have_bar = 1; bar_key = key[a.K - 1]; bar_idx = idx[a.K - 1]; }
                    }
                }
                __syncthreads();
            }
        }
    }
    __syncthreads();
    rc_sort(key, idx, n_buf, cap);
    const int nk = min(n_buf, a.K);
    int* out = a.cand + (long long)ex * a.K * 3;
    for (int i = tid; i < nk; i += RC_THREADS) {
        const unsigned id = idx[i];
        const unsigned fs = id >> 6;
        const int s = (int)(fs % (unsigned)S);
        out[3 * i] = (int)(fs / (unsigned)S); out[3 * i + 1] = s; out[3 * i + 2] = s + (int)(id & 63u);
    }
    // counts: warp then block reduction, fixed order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { my_total += __shfl_xor_sync(0xffffffffu, my_total, o); my_vec += __shfl_xor_sync(0xffffffffu, my_vec, o); }
    if ((tid & 31) == 0) { red[0][tid >> 5] = my_total; red[1][tid >> 5] = my_vec; }
    __syncthreads();
    if (tid == 0) {
        long long t = 0, v = 0;
        for (int w = 0; w < RC_THREADS / 32; w++) { t += red[0][w]; v += red[1][w]; }
        a.total[ex] = t; a.vec[ex] = v; a.ncand[ex] = nk;
        // version 2: the feature with the smallest start[0] + end[0] (strict <, from 1e6 like the reference's score_null)
        int nf = -1; float ns = 0.f, ne = 0.f;
        if (a.v2) {
            double best = 1000000.0;
            for (long long f = f0; f < f1; f++) {
                const float s = a.st[f * S], e = a.en[f * S];
                const double sc = (double)s + (double)e;
                if (sc < best) { best = sc; nf = (int)(f - f0); ns = s; ne = e; }
            }
        }
        a.null_feat[ex] = nf; a.null_logit[2 * ex] = ns; a.null_logit[2 * ex + 1] = ne;
    }
}

// scratch for host buffers, grown on demand and kept for the process (the call is synchronous)
struct RcScratch { void* p = nullptr; size_t cap = 0; };
static int rc_grow(RcScratch& s, size_t bytes) {
    if (bytes <= s.cap) return 0;
    if (s.p) { cudaFree(s.p); s.p = nullptr; s.cap = 0; }
    DPH_CUDA(cudaMalloc(&s.p, bytes));
    s.cap = bytes;
    return 0;
}

DPH_API int dph_rc_spans(const float* start, const float* end, const float* sft, const float* eft, int F, int S, const int32_t* n_tokens,
                         const uint32_t* start_ok, const uint32_t* end_ok, const int64_t* ex_off, int E, int max_answer_length,
                         double filter_threshold, int K, int version_2, int32_t* cand, int32_t* n_cand, int64_t* total_count,
                         int64_t* vec_count, int32_t* null_feature, float* null_logits, int mem, void* cuda_stream) {
    DPH_CHECK(start && end && sft && eft && n_tokens && start_ok && end_ok && ex_off && cand && n_cand && total_count && vec_count &&
              null_feature && null_logits, "rc_spans: null buffer");
    DPH_CHECK(F >= 1 && E >= 1 && S >= 1 && S <= RC_MAX_S, "rc_spans: F >= 1 features, E >= 1 examples, 1 <= S <= 512");
    DPH_CHECK(max_answer_length >= 1 && max_answer_length <= RC_MAX_L, "rc_spans: 1 <= max_answer_length <= 64");
    DPH_CHECK(K >= 1 && K <= RC_MAX_K, "rc_spans: 1 <= K <= 1024");
    DPH_CHECK(mem == DPH_MEM_HOST || mem == DPH_MEM_DEVICE, "rc_spans: mem is DPH_MEM_HOST or DPH_MEM_DEVICE");
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const int W = (S + 31) / 32;
    // offsets and token counts are checked on the host: every example has >= 1 feature, in order, covering [0, F)
    std::string err;
    {
        std::vector<int64_t> off_h;
        std::vector<int32_t> nt_h;
        const int64_t* off = ex_off;
        const int32_t* nt = n_tokens;
        if (mem == DPH_MEM_DEVICE) {
            off_h.resize((size_t)E + 1); nt_h.resize((size_t)F);
            DPH_CUDA(cudaMemcpyAsync(off_h.data(), ex_off, (size_t)(E + 1) * 8, cudaMemcpyDeviceToHost, st));
            DPH_CUDA(cudaMemcpyAsync(nt_h.data(), n_tokens, (size_t)F * 4, cudaMemcpyDeviceToHost, st));
            DPH_CUDA(cudaStreamSynchronize(st));
            off = off_h.data(); nt = nt_h.data();
        }
        if (off[0] != 0 || off[E] != F) err = "rc_spans: example offsets must start at 0 and end at F";
        for (int x = 0; err.empty() && x < E; x++) {
            const int64_t nf = off[x + 1] - off[x];
            if (nf < 1) err = "rc_spans: every example needs at least one feature (offsets strictly increasing)";
            else if (nf * S * 64 > 0xffffffffll) err = "rc_spans: too many features in one example (features * S * 64 must fit 32 bits)";
        }
        for (int f = 0; err.empty() && f < F; f++)
            if (nt[f] < 0 || nt[f] > S) err = "rc_spans: n_tokens must lie in [0, S]";
    }
    DPH_CHECK(err.empty(), err);
    int cap = 512;
    while (cap < K + RC_THREADS) cap <<= 1;
    const size_t smem = (size_t)cap * 12 + (size_t)S * 16 + (size_t)W * 8;
    static DphPerDeviceOnce once;
    if (once.first()) DPH_CUDA(cudaFuncSetAttribute(rc_spans_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    SpanArgs a{};
    a.S = S; a.W = W; a.L = max_answer_length; a.K = K; a.v2 = version_2 ? 1 : 0; a.cap = cap; a.thr = filter_threshold;
    const size_t in_f = (size_t)F * S * 4, in_m = (size_t)F * W * 4;
    const size_t out_c = (size_t)E * K * 3 * 4;
    if (mem == DPH_MEM_DEVICE) {
        a.st = start; a.en = end; a.sft = sft; a.eft = eft; a.ntok = n_tokens; a.sok = start_ok; a.eok = end_ok; a.off = (const long long*)ex_off;
        a.cand = cand; a.ncand = n_cand; a.total = (long long*)total_count; a.vec = (long long*)vec_count; a.null_feat = null_feature;
        a.null_logit = null_logits;
    } else {
        static RcScratch scratch[64];
        int dev = 0;
        DPH_CUDA(cudaGetDevice(&dev));
        RcScratch& sc = scratch[dev & 63];
        const size_t sizes[] = {in_f, in_f, in_f, in_f, (size_t)F * 4, in_m, in_m, (size_t)(E + 1) * 8, out_c, (size_t)E * 4, (size_t)E * 8,
                                (size_t)E * 8, (size_t)E * 4, (size_t)E * 8};
        size_t offs[14], tot = 0;
        for (int i = 0; i < 14; i++) { offs[i] = tot; tot += (sizes[i] + 255) & ~(size_t)255; }
        DPH_TRY(rc_grow(sc, tot));
        char* base = (char*)sc.p;
        const void* src[8] = {start, end, sft, eft, n_tokens, start_ok, end_ok, ex_off};
        for (int i = 0; i < 8; i++) DPH_CUDA(cudaMemcpyAsync(base + offs[i], src[i], sizes[i], cudaMemcpyHostToDevice, st));
        a.st = (const float*)(base + offs[0]); a.en = (const float*)(base + offs[1]); a.sft = (const float*)(base + offs[2]);
        a.eft = (const float*)(base + offs[3]); a.ntok = (const int*)(base + offs[4]); a.sok = (const unsigned*)(base + offs[5]);
        a.eok = (const unsigned*)(base + offs[6]); a.off = (const long long*)(base + offs[7]);
        a.cand = (int*)(base + offs[8]); a.ncand = (int*)(base + offs[9]); a.total = (long long*)(base + offs[10]);
        a.vec = (long long*)(base + offs[11]); a.null_feat = (int*)(base + offs[12]); a.null_logit = (float*)(base + offs[13]);
    }
    rc_spans_kernel<<<(unsigned)E, RC_THREADS, smem, st>>>(a);
    DPH_CUDA(cudaGetLastError());
    if (mem == DPH_MEM_HOST) {
        void* dst[6] = {cand, n_cand, total_count, vec_count, null_feature, null_logits};
        const void* from[6] = {a.cand, a.ncand, a.total, a.vec, a.null_feat, a.null_logit};
        const size_t nb[6] = {out_c, (size_t)E * 4, (size_t)E * 8, (size_t)E * 8, (size_t)E * 4, (size_t)E * 8};
        for (int i = 0; i < 6; i++) DPH_CUDA(cudaMemcpyAsync(dst[i], from[i], nb[i], cudaMemcpyDeviceToHost, st));
    }
    DPH_CUDA(cudaStreamSynchronize(st));
    return 0;
}
