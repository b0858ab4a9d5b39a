// train.cu -- training a resident index: the spherical k-means coarse quantizer and the PQ codebooks of faiss
// IndexPreTransform(OPQ) -> IndexIVFPQ(IndexFlatIP) (Clustering with cp.spherical, ProductQuantizer::train, faiss 1.6.x) [3P],
// reference build_phrase_index.py:96-142, bit-identical to oracle/train_ref.c (DESIGN.md 3.3 "Training the index").
// Per k-means iteration:
//   assign   the encoding's own kernels: dph_coarse_top1 (coarse, smallest list on a tie) or pq_encode_kernel (PQ, lowest codeword)
//   sort     stable sort of (cluster, row) so every cluster's members are contiguous and ascending
//   update   one thread per (centroid, dimension) adds its members' values in ascending row order, times 1 / count
//   split    the host plans faiss' split_clusters from the counts; one kernel applies the splits in order
//   renorm   (coarse) every centroid to unit L2 norm
// Only the rotated sample is resident; host input is gathered, uploaded and rotated chunk by chunk.  Every buffer of a call is
// allocated before the first iteration and the result replaces the index's tables only at the end: a refused or failed call leaves
// the index as it was.
#include "index_internal.cuh"
#include <algorithm>
#include <numeric>
#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/sequence.h>
#include <thrust/sort.h>

enum { TR_STREAM_SAMPLE = 4, TR_STREAM_INIT = 5, TR_STREAM_SPLIT = 6 };
#define TR_SPLIT_EPS (1.0f / 1024.0f)
#define TR_UPDATE_THREADS 256

// Positions [0, n) ranked by (key(p), p) ascending: the first `take` of them, in rank order.
template <class K> static std::vector<int64_t> rank_first(int64_t n, int64_t take, K key) {
    std::vector<std::pair<uint64_t, int64_t>> v((size_t)n);
    for (int64_t p = 0; p < n; p++) v[p] = {key(p), p};
    if (take < n) std::nth_element(v.begin(), v.begin() + take, v.end());
    std::sort(v.begin(), v.begin() + take);
    std::vector<int64_t> out((size_t)take);
    for (int64_t r = 0; r < take; r++) out[r] = v[r].second;
    return out;
}

// The training sample: every row, or the first cap rows of the ranking by rnd64(seed, SAMPLE, i, which), in ascending row order.
static std::vector<int64_t> train_sample(int64_t n, int64_t cap, uint64_t seed, uint64_t which) {
    if (n <= cap) { std::vector<int64_t> all((size_t)n); std::iota(all.begin(), all.end(), 0); return all; }
    std::vector<int64_t> idx = rank_first(n, cap, [&](int64_t i) { return dph_rnd64(seed, TR_STREAM_SAMPLE, (uint64_t)i, which); });
    std::sort(idx.begin(), idx.end());
    return idx;
}

// faiss split_clusters with the repo's draws (oracle/train_ref.c:ref_split_clusters): appends (empty c, donor cj) in order.
static int64_t plan_splits(std::vector<float>& h, int64_t ns, uint64_t seed, uint64_t s, uint64_t it, int64_t row0,
                           std::vector<int2>& out) {
    const int64_t k = (int64_t)h.size();
    int64_t nsplit = 0;
    uint64_t draw = 0;
    for (int64_t ci = 0; ci < k; ci++) {
        if (h[ci] != 0.0f) continue;
        int64_t cj = 0;
        for (;; cj = (cj + 1) % k) {
            const float p = (h[cj] - 1.0f) / (float)(ns - k);
            const float u = (float)(dph_rnd64(seed, TR_STREAM_SPLIT, (s << 32) | it, draw++) >> 40) * 0x1p-24f;
            if (u < p) break;
        }
        out.push_back(make_int2((int)(row0 + ci), (int)(row0 + cj)));
        h[ci] = h[cj] / 2.0f;
        h[cj] -= h[ci];
        nsplit++;
    }
    return nsplit;
}

// rows of x (device, [*, d]) listed in idx -> out [m, d]
__global__ void gather_rows_kernel(const float* __restrict__ x, const long long* __restrict__ idx, long long m, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m * (DPH_D / 4)) return;
    const long long r = i / (DPH_D / 4), c = i - r * (DPH_D / 4);
    reinterpret_cast<float4*>(out)[r * (DPH_D / 4) + c] = reinterpret_cast<const float4*>(x)[idx[r] * (DPH_D / 4) + c];
}

// cent[c] = sample row first[c] restricted to columns [col0 + g * dd, + dd) of group g = c / k  (init)
__global__ void init_rows_kernel(const float* __restrict__ xs, const int* __restrict__ first, long long G, int k, int dd, float* __restrict__ cent) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= G * k * dd) return;
    const long long gc = i / dd; const int t = (int)(i - gc * dd); const long long g = gc / k;
    cent[i] = xs[(long long)first[gc] * DPH_D + g * dd + t];
}

// xs[i] = xs[i] - C[list[i]] (fp32, in place): the residual pq_encode_kernel forms when it encodes row i
__global__ void residual_kernel(float* __restrict__ xs, const float* __restrict__ C, const int* __restrict__ list, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * DPH_D) return;
    const long long r = i / DPH_D;
    xs[i] = __fsub_rn(xs[i], C[(long long)list[r] * DPH_D + (i - r * DPH_D)]);
}

__global__ void count_kernel(const int* __restrict__ key, long long n, int* __restrict__ cnt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(&cnt[key[i]], 1);
}

// PQ: one sort key per (row, sub-quantizer) pair q = i * 96 + m: key m * 256 + code, value i
__global__ void pq_pairs_kernel(const uint8_t* __restrict__ codes, long long n, int* __restrict__ key, int* __restrict__ row) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n * DPH_M) return;
    const int m = (int)(q % DPH_M);
    key[q] = m * DPH_KSUB + codes[q];
    row[q] = (int)(q / DPH_M);
}

// One thread per (group g, centroid c, dimension t) -- group = sub-quantizer (dd = 8) or the whole coarse row (G = 1, dd = 768):
// s = +0.0f; s = s + xs[row][g * dd + t] over the cluster's members in ascending row order (plain fp32 adds); centroid = s * (1 / count).
// A warp covers 32 consecutive dimensions, so for the coarse quantizer every member row is read as one coalesced 128 B segment.  The
// member numbers and values are loaded 8 ahead of the dependent add chain.  Empty clusters keep their row (the split rewrites it).
__global__ void __launch_bounds__(TR_UPDATE_THREADS) km_update_kernel(const float* __restrict__ xs, const int* __restrict__ members,
                                                                      const int* __restrict__ off, long long G, int k, int dd, float* __restrict__ cent) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= G * k * dd) return;
    const long long gc = i / dd; const int t = (int)(i - gc * dd); const long long g = gc / k;
    const int p0 = off[gc], p1 = off[gc + 1];
    if (p0 == p1) return;
    const float* col = xs + g * dd + t;
    float s = 0.0f;
    int p = p0;
    for (; p + 8 <= p1; p += 8) {
        int r[8]; float v[8];
#pragma unroll
        for (int e = 0; e < 8; e++) r[e] = __ldg(members + p + e);
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = __ldg(col + (long long)r[e] * DPH_D);
#pragma unroll
        for (int e = 0; e < 8; e++) s = __fadd_rn(s, v[e]);
    }
    for (; p < p1; p++) s = __fadd_rn(s, __ldg(col + (long long)__ldg(members + p) * DPH_D));
    cent[i] = __fmul_rn(s, __fdiv_rn(1.0f, __int2float_rn(p1 - p0)));
}

// The planned splits, in order (a donor may be split twice): thread (group g, dimension t) walks its group's splits.
__global__ void km_split_kernel(const int2* __restrict__ splits, const int* __restrict__ soff, long long G, int dd, float* __restrict__ cent) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= G * dd) return;
    const long long g = i / dd; const int t = (int)(i - g * dd);
    const float up = 1.0f + TR_SPLIT_EPS, dn = 1.0f - TR_SPLIT_EPS;
    for (int e = soff[g]; e < soff[g + 1]; e++) {
        const int2 sp = splits[e];
        const float v = cent[(long long)sp.y * dd + t];
        cent[(long long)sp.x * dd + t] = __fmul_rn(v, (t % 2 == 0) ? up : dn);
        cent[(long long)sp.y * dd + t] = __fmul_rn(v, (t % 2 == 0) ? dn : up);
    }
}

// Spherical k-means: nr = fmaf chain over t ascending; nr > 0 -> every component times 1 / sqrt(nr).  One thread per centroid.
__global__ void km_renorm_kernel(float* __restrict__ cent, long long k) {
    const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= k) return;
    float4* row = reinterpret_cast<float4*>(cent + c * DPH_D);
    float nr = 0.0f;
    for (int t = 0; t < DPH_D / 4; t++) {
        const float4 v = row[t];
        nr = fmaf(v.x, v.x, nr); nr = fmaf(v.y, v.y, nr); nr = fmaf(v.z, v.z, nr); nr = fmaf(v.w, v.w, nr);
    }
    if (!(nr > 0.0f)) return;
    const float inv = __fdiv_rn(1.0f, __fsqrt_rn(nr));
    for (int t = 0; t < DPH_D / 4; t++) {
        float4 v = row[t];
        v.x = __fmul_rn(v.x, inv); v.y = __fmul_rn(v.y, inv); v.z = __fmul_rn(v.z, inv); v.w = __fmul_rn(v.w, inv);
        row[t] = v;
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// One k-means run over G groups of k centroids of dd dimensions each (coarse: G = 1, k = nlist, dd = 768; PQ: G = 96, k = 256,
// dd = 8), on the resident rotated sample xs [ns, 768].
struct KMeans {
    dph_index* ix;
    const float* xs; int64_t ns;
    int64_t G; int k, dd;
    float* cent;                          // [G * k * dd] working centroids
    int *key, *members, *cnt, *off, *soff; int2* splits;
    float* cd; int32_t* zero_key; float* zero_row; int64_t* list_scratch; uint8_t* codes;
    uint64_t seed;
};

static int km_alloc(KMeans& km, DevTmp& tmp, const char* oom) {
    const int64_t pairs = km.G == 1 ? km.ns : km.ns * DPH_M;
    const int64_t K = km.G * km.k;
    DPH_TRY(tmp.alloc(&km.cent, (size_t)K * km.dd, oom));
    DPH_TRY(tmp.alloc(&km.key, pairs, oom)); DPH_TRY(tmp.alloc(&km.members, pairs, oom));
    DPH_TRY(tmp.alloc(&km.cnt, K, oom)); DPH_TRY(tmp.alloc(&km.off, K + 1, oom));
    DPH_TRY(tmp.alloc(&km.splits, K, oom)); DPH_TRY(tmp.alloc(&km.soff, km.G + 1, oom));
    if (km.G == 1) DPH_TRY(tmp.alloc(&km.cd, km.ns, oom));
    else {
        DPH_TRY(tmp.alloc(&km.zero_key, km.ns, oom)); DPH_TRY(tmp.alloc(&km.zero_row, DPH_D, oom));
        DPH_TRY(tmp.alloc(&km.list_scratch, km.ns, oom)); DPH_TRY(tmp.alloc(&km.codes, (size_t)km.ns * DPH_M, oom));
        DPH_CUDA(cudaMemsetAsync(km.zero_key, 0, (size_t)km.ns * 4, km.ix->stream));
        DPH_CUDA(cudaMemsetAsync(km.zero_row, 0, DPH_D * 4, km.ix->stream));
    }
    return 0;
}

// Coarse top-1 of every sample row, in chunks whose score matrix fits the search workspace (<= 1 GiB).
static int coarse_assign_all(dph_index* ix, const float* xs, const float* Cw, int64_t ns, int32_t* key, float* cd) {
    const int64_t cs = std::min(dph_encode_chunk(ix), ns), nlp = (ix->nlist + 127) / 128 * 128;
    DPH_TRY(ix->S.ensure((size_t)cs * nlp * 4));
    ix->csplit_lo = -1;                                    // the tensor-core path caches a split of the centroids: they changed
    for (int64_t o = 0; o < ns; o += cs)
        DPH_TRY(dph_coarse_top1(ix, xs + o * DPH_D, Cw, std::min(cs, ns - o), key + o, cd + o, ix->stream));
    return 0;
}

static int km_init(KMeans& km) {
    std::vector<int> first((size_t)(km.G * km.k));
    for (int64_t g = 0; g < km.G; g++) {
        const uint64_t s = km.G == 1 ? 0 : 1 + (uint64_t)g;
        const std::vector<int64_t> r = rank_first(km.ns, km.k, [&](int64_t p) { return dph_rnd64(km.seed, TR_STREAM_INIT, s, (uint64_t)p); });
        for (int c = 0; c < km.k; c++) first[g * km.k + c] = (int)r[c];
    }
    DevTmp tmp;
    int* d_first;
    DPH_TRY(tmp.alloc(&d_first, first.size(), "train: init rows"));
    DPH_CUDA(cudaMemcpyAsync(d_first, first.data(), first.size() * 4, cudaMemcpyHostToDevice, km.ix->stream));
    const long long tot = km.G * km.k * km.dd;
    init_rows_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, km.ix->stream>>>(km.xs, d_first, km.G, km.k, km.dd, km.cent);
    DPH_CUDA(cudaGetLastError());
    if (km.G == 1) { km_renorm_kernel<<<(unsigned)((km.k + 127) / 128), 128, 0, km.ix->stream>>>(km.cent, km.k); DPH_CUDA(cudaGetLastError()); }
    DPH_CUDA(cudaStreamSynchronize(km.ix->stream));        // d_first is freed on return
    return 0;
}

// One iteration; obj (coarse, may be null): the sum of the assigned scores in fp64, ascending row.  -> the number of splits.
static int km_iterate(KMeans& km, uint64_t it, double* obj, int64_t* nsplit_out) {
    dph_index* ix = km.ix;
    cudaStream_t st = ix->stream;
    const bool prof = ix->profile && ix->aev[0];
    const int64_t K = km.G * km.k, pairs = km.G == 1 ? km.ns : km.ns * DPH_M;
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[0], st));
    // 1. assign
    if (km.G == 1) DPH_TRY(coarse_assign_all(ix, km.xs, km.cent, km.ns, km.key, km.cd));
    else {
        DPH_TRY(dph_pq_assign(ix, km.xs, km.zero_row, km.zero_key, km.cent, km.ns, km.list_scratch, km.codes, st));
        pq_pairs_kernel<<<(unsigned)((pairs + 255) / 256), 256, 0, st>>>(km.codes, km.ns, km.key, km.members);
        DPH_CUDA(cudaGetLastError());
    }
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[1], st));
    // 2. counts, member order, update
    DPH_CUDA(cudaMemsetAsync(km.cnt, 0, (size_t)K * 4, st));
    count_kernel<<<(unsigned)((pairs + 255) / 256), 256, 0, st>>>(km.key, pairs, km.cnt);
    DPH_CUDA(cudaGetLastError());
    try {
        thrust::device_ptr<int> kp(km.key), mp(km.members);
        if (km.G == 1) thrust::sequence(thrust::cuda::par.on(st), mp, mp + pairs);
        thrust::stable_sort_by_key(thrust::cuda::par.on(st), kp, kp + pairs, mp);
    } catch (const std::exception& e) {
        cudaGetLastError();
        dph_set_error(std::string("train: device sort failed; the index is unchanged: ") + e.what());
        return 1;
    }
    std::vector<int> cnt((size_t)K), off((size_t)K + 1, 0);
    std::vector<float> cdh(obj ? (size_t)km.ns : 0);
    DPH_CUDA(cudaMemcpyAsync(cnt.data(), km.cnt, (size_t)K * 4, cudaMemcpyDeviceToHost, st));
    if (obj) DPH_CUDA(cudaMemcpyAsync(cdh.data(), km.cd, (size_t)km.ns * 4, cudaMemcpyDeviceToHost, st));
    DPH_CUDA(cudaStreamSynchronize(st));
    for (int64_t c = 0; c < K; c++) off[c + 1] = off[c] + cnt[c];
    DPH_CUDA(cudaMemcpyAsync(km.off, off.data(), off.size() * 4, cudaMemcpyHostToDevice, st));
    const long long tot = K * km.dd;
    km_update_kernel<<<(unsigned)((tot + TR_UPDATE_THREADS - 1) / TR_UPDATE_THREADS), TR_UPDATE_THREADS, 0, st>>>(km.xs, km.members, km.off,
                                                                                                                  km.G, km.k, km.dd, km.cent);
    DPH_CUDA(cudaGetLastError());
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[2], st));
    if (obj) { double o = 0.0; for (float v : cdh) o += (double)v; *obj = o; }
    // 3. splits (planned on the host from the counts), renorm
    std::vector<int2> splits;
    std::vector<int> soff((size_t)km.G + 1, 0);
    int64_t nsplit = 0;
    for (int64_t g = 0; g < km.G; g++) {
        std::vector<float> h(cnt.begin() + g * km.k, cnt.begin() + (g + 1) * km.k);
        nsplit += plan_splits(h, km.ns, km.seed, km.G == 1 ? 0 : 1 + (uint64_t)g, it, g * km.k, splits);
        soff[g + 1] = (int)splits.size();
    }
    if (!splits.empty()) {
        DPH_CUDA(cudaMemcpyAsync(km.splits, splits.data(), splits.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
        DPH_CUDA(cudaMemcpyAsync(km.soff, soff.data(), soff.size() * 4, cudaMemcpyHostToDevice, st));
        km_split_kernel<<<(unsigned)((km.G * km.dd + 127) / 128), 128, 0, st>>>(km.splits, km.soff, km.G, km.dd, km.cent);
        DPH_CUDA(cudaGetLastError());
    }
    if (km.G == 1) { km_renorm_kernel<<<(unsigned)((km.k + 127) / 128), 128, 0, st>>>(km.cent, km.k); DPH_CUDA(cudaGetLastError()); }
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[3], st));
    DPH_CUDA(cudaStreamSynchronize(st));                   // the host vectors above are the copies' sources
    if (prof)
        for (int s = 0; s < 3; s++) { float ms = 0.f; DPH_CUDA(cudaEventElapsedTime(&ms, ix->aev[s], ix->aev[s + 1])); ix->train_ms[s] += ms; }
    if (nsplit_out) *nsplit_out = nsplit;
    return 0;
}

// The sample rows of x (host or device), rotated by the OPQ matrix, into xs [idx.size(), 768]; *bad |= 1 on a non-finite value.
static int load_sample(dph_index* ix, const float* x, int mem, const std::vector<int64_t>& idx, float* xs, int* bad, DevTmp& tmp) {
    cudaStream_t st = ix->stream;
    const int64_t ns = (int64_t)idx.size(), cs = std::min(dph_encode_chunk(ix), ns);
    const char* oom = "train: not enough device memory for the staging buffers; the index is unchanged";
    float* stage; long long* d_idx;
    DPH_TRY(tmp.alloc(&stage, (size_t)cs * DPH_D, oom));
    DPH_TRY(tmp.alloc(&d_idx, (size_t)cs, oom));
    std::vector<float> h_stage(mem == DPH_MEM_HOST ? (size_t)cs * DPH_D : 0);
    for (int64_t o = 0; o < ns; o += cs) {
        const int64_t m = std::min(cs, ns - o);
        if (mem == DPH_MEM_HOST) {
            for (int64_t r = 0; r < m; r++) memcpy(&h_stage[(size_t)r * DPH_D], x + idx[o + r] * DPH_D, DPH_D * 4);
            DPH_CUDA(cudaMemcpyAsync(stage, h_stage.data(), (size_t)m * DPH_D * 4, cudaMemcpyHostToDevice, st));
        } else {
            DPH_CUDA(cudaMemcpyAsync(d_idx, idx.data() + o, (size_t)m * 8, cudaMemcpyHostToDevice, st));
            gather_rows_kernel<<<(unsigned)((m * (DPH_D / 4) + 255) / 256), 256, 0, st>>>(x, d_idx, m, stage);
            DPH_CUDA(cudaGetLastError());
        }
        nonfinite_kernel<<<(unsigned)std::min<int64_t>((m * DPH_D + 255) / 256, 4 * ix->num_sms), 256, 0, st>>>(stage, m * DPH_D, bad);
        DPH_CUDA(cudaGetLastError());
        DPH_TRY(dph_launch_sgemm_nt_seq(stage, m, ix->A, DPH_D, DPH_D, xs + o * DPH_D, st));
        DPH_CUDA(cudaStreamSynchronize(st));               // the host staging buffer is refilled by the next chunk
    }
    return 0;
}

static int train_checks(dph_index* ix, const float* x, int64_t n, int niter, int64_t mppc, int mem, int64_t k, const char* what) {
    DPH_CHECK(ix != nullptr && (x != nullptr || n == 0) && niter >= 0 && mppc >= 1 && (mem == DPH_MEM_HOST || mem == DPH_MEM_DEVICE),
              std::string(what) + ": bad arguments");
    DPH_CHECK(ix->ntotal == 0, std::string(what) + ": the index holds vectors (faiss trains an empty index); the index is unchanged");
    DPH_CHECK(ix->A != nullptr, std::string(what) + ": the OPQ matrix is not set; the index is unchanged");
    DPH_CHECK(n >= k, std::string(what) + ": fewer training vectors than centroids; the index is unchanged");
    DPH_CHECK(n < (1ll << 31) / DPH_M, std::string(what) + ": more than 2^31 / 96 training vectors; the index is unchanged");
    return 0;
}

// Replace *dst (the index's table, may be null) by the trained `src` of `count` floats.
static int commit_table(dph_index* ix, float** dst, float* src, size_t count, DevTmp& tmp) {
    if (*dst) {
        DPH_CUDA(cudaMemcpyAsync(*dst, src, count * 4, cudaMemcpyDeviceToDevice, ix->stream));
        DPH_CUDA(cudaStreamSynchronize(ix->stream));
    } else {
        *dst = src; tmp.release(src);
    }
    return 0;
}

DPH_API int dph_index_train_coarse(dph_index* ix, const float* x, int64_t n, int niter, uint64_t seed, int64_t max_points_per_centroid,
                                   int hot_start, int mem, double* obj_out, int64_t* nsplit_out) {
    DPH_TRY(train_checks(ix, x, n, niter, max_points_per_centroid, mem, ix ? ix->nlist : 0, "train_coarse"));
    DPH_CHECK(!hot_start || ix->C != nullptr, "train_coarse: hot start needs centroids; the index is unchanged");
    DPH_CUDA(cudaSetDevice(ix->device));
    for (float& a : ix->train_ms) a = 0.f;
    const std::vector<int64_t> idx = train_sample(n, max_points_per_centroid * ix->nlist, seed, 0);
    KMeans km{};
    km.ix = ix; km.ns = (int64_t)idx.size(); km.G = 1; km.k = (int)ix->nlist; km.dd = DPH_D; km.seed = seed;
    DevTmp tmp;
    const char* oom = "train_coarse: not enough device memory for the rotated sample and the workspace; the index is unchanged";
    float* xs; int* bad;
    DPH_TRY(tmp.alloc(&xs, (size_t)km.ns * DPH_D, oom)); DPH_TRY(tmp.alloc(&bad, 1, oom));
    km.xs = xs;
    DPH_TRY(km_alloc(km, tmp, oom));
    DPH_CUDA(cudaMemsetAsync(bad, 0, 4, ix->stream));
    DPH_TRY(load_sample(ix, x, mem, idx, xs, bad, tmp));
    int h_bad = 0;
    DPH_CUDA(cudaMemcpy(&h_bad, bad, 4, cudaMemcpyDeviceToHost));
    DPH_CHECK(!h_bad, "train_coarse: a training vector holds a non-finite value; the index is unchanged");
    if (hot_start) DPH_CUDA(cudaMemcpyAsync(km.cent, ix->C, (size_t)km.k * DPH_D * 4, cudaMemcpyDeviceToDevice, ix->stream));
    else DPH_TRY(km_init(km));
    int rc = 0;
    for (int it = 0; it < niter && !rc; it++) rc = km_iterate(km, (uint64_t)it, obj_out ? obj_out + it : nullptr, nsplit_out ? nsplit_out + it : nullptr);
    ix->csplit_lo = -1;                                    // the cached split is of the working centroids, or of the old ones
    DPH_TRY(rc);
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    return commit_table(ix, &ix->C, km.cent, (size_t)km.k * DPH_D, tmp);
}

DPH_API int dph_index_train_pq(dph_index* ix, const float* x, int64_t n, int niter, uint64_t seed, int64_t max_points_per_centroid,
                               int hot_start, int residual, int mem) {
    DPH_TRY(train_checks(ix, x, n, niter, max_points_per_centroid, mem, DPH_KSUB, "train_pq"));
    DPH_CHECK(!residual || ix->C != nullptr, "train_pq: training on residuals needs the coarse centroids; the index is unchanged");
    DPH_CHECK(!hot_start || ix->pq != nullptr, "train_pq: hot start needs PQ codebooks; the index is unchanged");
    DPH_CUDA(cudaSetDevice(ix->device));
    for (float& a : ix->train_ms) a = 0.f;
    const std::vector<int64_t> idx = train_sample(n, max_points_per_centroid * DPH_KSUB, seed, 1);
    KMeans km{};
    km.ix = ix; km.ns = (int64_t)idx.size(); km.G = DPH_M; km.k = DPH_KSUB; km.dd = DPH_DSUB; km.seed = seed;
    cudaStream_t st = ix->stream;
    DevTmp tmp;
    const char* oom = "train_pq: not enough device memory for the rotated sample and the workspace; the index is unchanged";
    float* xs; int* bad;
    DPH_TRY(tmp.alloc(&xs, (size_t)km.ns * DPH_D, oom)); DPH_TRY(tmp.alloc(&bad, 1, oom));
    km.xs = xs;
    DPH_TRY(km_alloc(km, tmp, oom));
    int32_t* list = nullptr; float* cd = nullptr;
    if (residual) { DPH_TRY(tmp.alloc(&list, km.ns, oom)); DPH_TRY(tmp.alloc(&cd, km.ns, oom)); }
    DPH_CUDA(cudaMemsetAsync(bad, 0, 4, st));
    DPH_TRY(load_sample(ix, x, mem, idx, xs, bad, tmp));
    int h_bad = 0;
    DPH_CUDA(cudaMemcpy(&h_bad, bad, 4, cudaMemcpyDeviceToHost));
    DPH_CHECK(!h_bad, "train_pq: a training vector holds a non-finite value; the index is unchanged");
    if (residual) {
        // r = xr - C[top-1 list]: pq_encode_kernel's own fp32 subtraction, done once in place (the iterations use a zero centroid)
        DPH_TRY(coarse_assign_all(ix, xs, ix->C, km.ns, list, cd));
        residual_kernel<<<(unsigned)((km.ns * DPH_D + 255) / 256), 256, 0, st>>>(xs, ix->C, list, km.ns);
        DPH_CUDA(cudaGetLastError());
    }
    if (hot_start) DPH_CUDA(cudaMemcpyAsync(km.cent, ix->pq, (size_t)DPH_M * DPH_KSUB * DPH_DSUB * 4, cudaMemcpyDeviceToDevice, st));
    else DPH_TRY(km_init(km));
    for (int it = 0; it < niter; it++) DPH_TRY(km_iterate(km, (uint64_t)it, nullptr, nullptr));
    DPH_CUDA(cudaStreamSynchronize(st));
    ix->csplit_lo = -1;
    return commit_table(ix, &ix->pq, km.cent, (size_t)DPH_M * DPH_KSUB * DPH_DSUB, tmp);
}

// PQ codes of x A^T without a coarse residual (IndexPQ-style, what OPQ's training encodes): rotation, then pq_encode_kernel against
// a zero centroid row.
DPH_API int dph_index_encode_pq(dph_index* ix, const float* x, int64_t n, uint8_t* codes_out, int mem) {
    DPH_CHECK(ix != nullptr && n >= 0, "encode_pq: bad arguments");
    DPH_CHECK(ix->A && ix->pq, "encode_pq: OPQ matrix and PQ codebooks must be set");
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n == 0) return 0;
    cudaStream_t st = ix->stream;
    const int64_t cs = std::min(dph_encode_chunk(ix), n);
    DevTmp tmp;
    const char* oom = "encode_pq: not enough device memory for the staging buffers";
    int32_t* zkey; float* zrow; int64_t* lscr; uint8_t* cstage = nullptr;
    DPH_TRY(tmp.alloc(&zkey, cs, oom)); DPH_TRY(tmp.alloc(&zrow, DPH_D, oom)); DPH_TRY(tmp.alloc(&lscr, cs, oom));
    if (mem == DPH_MEM_HOST) DPH_TRY(tmp.alloc(&cstage, (size_t)cs * DPH_M, oom));
    DPH_CUDA(cudaMemsetAsync(zkey, 0, (size_t)cs * 4, st));
    DPH_CUDA(cudaMemsetAsync(zrow, 0, DPH_D * 4, st));
    DPH_TRY(ix->xr.ensure((size_t)cs * DPH_D * 4));
    if (mem == DPH_MEM_HOST) DPH_TRY(ix->xdev.ensure((size_t)cs * DPH_D * 4));
    for (int64_t o = 0; o < n; o += cs) {
        const int64_t m = std::min(cs, n - o);
        const float* src = x + o * DPH_D;
        if (mem == DPH_MEM_HOST) {
            DPH_CUDA(cudaMemcpyAsync(ix->xdev.p, src, (size_t)m * DPH_D * 4, cudaMemcpyHostToDevice, st));
            src = ix->xdev.as<float>();
        }
        DPH_TRY(dph_launch_sgemm_nt_seq(src, m, ix->A, DPH_D, DPH_D, ix->xr.as<float>(), st));
        uint8_t* dst = mem == DPH_MEM_HOST ? cstage : codes_out + o * DPH_M;
        DPH_TRY(dph_pq_assign(ix, ix->xr.as<float>(), zrow, zkey, ix->pq, m, lscr, dst, st));
        if (mem == DPH_MEM_HOST) {
            DPH_CUDA(cudaMemcpyAsync(codes_out + o * DPH_M, cstage, (size_t)m * DPH_M, cudaMemcpyDeviceToHost, st));
            DPH_CUDA(cudaStreamSynchronize(st));
        }
    }
    if (mem == DPH_MEM_HOST) DPH_CUDA(cudaStreamSynchronize(st));
    return 0;
}

DPH_API int dph_index_get_centroids(const dph_index* ix, float* C_out, int mem) {
    DPH_CHECK(ix && ix->C != nullptr, "centroids not set");
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_CUDA(cudaMemcpy(C_out, ix->C, (size_t)ix->nlist * ix->d * 4, mem == DPH_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice));
    return 0;
}

DPH_API int dph_index_get_pq(const dph_index* ix, float* pq_out, int mem) {
    DPH_CHECK(ix && ix->pq != nullptr, "PQ codebooks not set");
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_CUDA(cudaMemcpy(pq_out, ix->pq, (size_t)DPH_M * DPH_KSUB * DPH_DSUB * 4, mem == DPH_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice));
    return 0;
}

DPH_API int dph_index_last_train_ms(const dph_index* ix, float* ms_out) {
    DPH_CHECK(ix->aev[0] != nullptr, "profiling was never enabled");
    std::copy(ix->train_ms, ix->train_ms + 3, ms_out);
    return 0;
}
