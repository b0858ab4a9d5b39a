/*
 * oracle/train_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the training that reference build_phrase_index.py:96-142 asks faiss 1.6.x to do for
 *   IndexPreTransform(OPQMatrix(768, 96), IndexIVFPQ(IndexFlatIP(768), 768, nlist, 96, 8, IP))
 * -- the spherical k-means of the coarse quantizer (Clustering with cp.spherical, IndexIVF::train_q1) and the 96 L2 k-means of the
 * PQ on residuals (ProductQuantizer::train) [3P] -- with the fixed floating-point order and the repo's own random draws of
 * DESIGN.md 3.3.  ivfpq_ref.c is compiled into this library, so the rotation, the coarse top-1 (ref_coarse, nprobe 1) and rnd64 are
 * the search oracle's own code; the PQ assignment is the encoding argmin of encode_ref.c:ref_encode, restated in the same words.
 * The loops are literal: sums in ascending row order, one plain fp32 add per member, the split rule of faiss' split_clusters.
 * What pins it: tests/test_train_cpu.py (numpy restatement bit for bit, a split checked by hand, unit-norm centroids, falling PQ
 * distortion, the sample and the init as functions of (seed, n)).
 *
 * Only tests/, __graft_entry__.smoke() and tools/bench_train.py may load this library.
 */
#include "ivfpq_ref.c"

enum { STREAM_SAMPLE = 4, STREAM_INIT = 5, STREAM_SPLIT = 6 };
#define SPLIT_EPS (1.0f / 1024.0f)

typedef struct { uint64_t key; int64_t i; } rank_kv;
static int rank_cmp(const void* a, const void* b) {
    const rank_kv *x = (const rank_kv*)a, *y = (const rank_kv*)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->i < y->i ? -1 : (x->i > y->i);
}
static int i64_cmp(const void* a, const void* b) {
    const int64_t x = *(const int64_t*)a, y = *(const int64_t*)b;
    return x < y ? -1 : (x > y);
}

/* The training sample: when n > cap, the first cap rows of the ranking by (rnd64(seed, STREAM_SAMPLE, i, which), i) ascending, in
 * ascending row order; else every row.  which: 0 coarse quantizer, 1 PQ.  idx [min(n, cap)] -> the sample size. */
REF_API int64_t ref_train_sample(int64_t n, int64_t cap, uint64_t seed, uint64_t which, int64_t* idx) {
    if (n <= cap) { for (int64_t i = 0; i < n; i++) idx[i] = i; return n; }
    rank_kv* v = (rank_kv*)malloc(sizeof(rank_kv) * (size_t)n);
    for (int64_t i = 0; i < n; i++) { v[i].key = rnd64(seed, STREAM_SAMPLE, (uint64_t)i, which); v[i].i = i; }
    qsort(v, (size_t)n, sizeof(rank_kv), rank_cmp);
    for (int64_t r = 0; r < cap; r++) idx[r] = v[r].i;
    qsort(idx, (size_t)cap, sizeof(int64_t), i64_cmp);
    free(v);
    return cap;
}

/* Init of k-means run s (0: coarse, 1 + m: sub-quantizer m): centroid c is the sample row of rank c under
 * (rnd64(seed, STREAM_INIT, s, p), p) ascending, p = position in the sample.  first [k]. */
REF_API void ref_train_init_rows(int64_t ns, int64_t k, uint64_t seed, uint64_t s, int64_t* first) {
    rank_kv* v = (rank_kv*)malloc(sizeof(rank_kv) * (size_t)ns);
    for (int64_t p = 0; p < ns; p++) { v[p].key = rnd64(seed, STREAM_INIT, s, (uint64_t)p); v[p].i = p; }
    qsort(v, (size_t)ns, sizeof(rank_kv), rank_cmp);
    for (int64_t c = 0; c < k; c++) first[c] = v[c].i;
    free(v);
}

/* faiss split_clusters [3P] with the repo's draws: for every empty c in ascending order, cycle cj = 0, 1, ... and take the first
 * cj whose draw u < (h[cj] - 1) / (float)(ns - k); copy C[cj] to C[c], scale by 1 -/+ 2^-10 by parity of t, halve the count.
 * u = (rnd64(seed, STREAM_SPLIT, s << 32 | it, draw) >> 40) * 2^-24, draw counting every draw of this iteration.  -> splits. */
REF_API int64_t ref_split_clusters(float* Cc, int64_t k, int dd, float* h, int64_t ns, uint64_t seed, uint64_t s, uint64_t it) {
    int64_t nsplit = 0;
    uint64_t draw = 0;
    for (int64_t ci = 0; ci < k; ci++) {
        if (h[ci] != 0.0f) continue;
        int64_t cj = 0;
        for (;; cj = (cj + 1) % k) {
            const float p = (h[cj] - 1.0f) / (float)(ns - k);
            const float u = (float)(rnd64(seed, STREAM_SPLIT, (s << 32) | it, draw++) >> 40) * 0x1p-24f;
            if (u < p) break;
        }
        memcpy(Cc + ci * dd, Cc + cj * dd, sizeof(float) * (size_t)dd);
        for (int t = 0; t < dd; t++) {
            if (t % 2 == 0) { Cc[ci * dd + t] *= 1.0f + SPLIT_EPS; Cc[cj * dd + t] *= 1.0f - SPLIT_EPS; }
            else { Cc[ci * dd + t] *= 1.0f - SPLIT_EPS; Cc[cj * dd + t] *= 1.0f + SPLIT_EPS; }
        }
        h[ci] = h[cj] / 2.0f;
        h[cj] -= h[ci];
        nsplit++;
    }
    return nsplit;
}

/* Update of one k-means: column block [col0, col0 + dd) of the sample rows xs [ns, ld]; C[c][t] = (sum in ascending row order,
 * plain fp32 adds from +0.0f) * (1.0f / (float)count[c]); empty clusters keep their centroid (the split overwrites it).  h = counts. */
static void km_update(const float* xs, int64_t ns, int ld, int col0, int dd, const int64_t* assign, int64_t k, float* Cc, float* h) {
    float* sum = (float*)calloc((size_t)k * dd, sizeof(float));
    int64_t* cnt = (int64_t*)calloc((size_t)k, sizeof(int64_t));
    for (int64_t i = 0; i < ns; i++) {
        const int64_t c = assign[i];
        cnt[c]++;
        for (int t = 0; t < dd; t++) sum[c * dd + t] = sum[c * dd + t] + xs[i * ld + col0 + t];
    }
    for (int64_t c = 0; c < k; c++) {
        h[c] = (float)cnt[c];
        if (cnt[c] == 0) continue;
        const float inv = 1.0f / (float)cnt[c];
        for (int t = 0; t < dd; t++) Cc[c * dd + t] = sum[c * dd + t] * inv;
    }
    free(sum); free(cnt);
}

/* Spherical: nr = fmaf chain of C[c][t]^2, t ascending; nr > 0 -> C[c][t] *= 1.0f / sqrtf(nr). */
static void km_renorm(float* Cc, int64_t k, int d) {
    for (int64_t c = 0; c < k; c++) {
        float nr = 0.0f;
        for (int t = 0; t < d; t++) nr = fmaf(Cc[c * d + t], Cc[c * d + t], nr);
        if (nr > 0.0f) {
            const float inv = 1.0f / sqrtf(nr);
            for (int t = 0; t < d; t++) Cc[c * d + t] *= inv;
        }
    }
}

static float* rotated_sample(const float* x, int64_t n, int d, const float* A, int64_t cap, uint64_t seed, uint64_t which, int64_t* ns_out) {
    int64_t* idx = (int64_t*)malloc(sizeof(int64_t) * (size_t)(n < cap ? n : cap));
    const int64_t ns = ref_train_sample(n, cap, seed, which, idx);
    float* g = (float*)malloc(sizeof(float) * (size_t)ns * d);
    for (int64_t r = 0; r < ns; r++) memcpy(g + r * d, x + idx[r] * d, sizeof(float) * (size_t)d);
    float* xs = (float*)malloc(sizeof(float) * (size_t)ns * d);
    ref_rotate(g, ns, d, A, xs);
    free(g); free(idx);
    *ns_out = ns;
    return xs;
}

static void coarse_top1(const float* xs, int64_t ns, int d, const float* Cc, int64_t k, int64_t* assign, float* cd) {
    const int64_t chunk = 4096;                 /* bounds the score matrix of ref_coarse */
    for (int64_t o = 0; o < ns; o += chunk) ref_coarse(xs + o * d, ns - o < chunk ? ns - o : chunk, d, Cc, k, 1, cd + o, assign + o);
}

/* Coarse quantizer (DESIGN.md 3.3): x [n, d] is rotated by A; C [k, d] in/out (read when hot_start); obj [niter] = sum of the
 * assigned scores in fp64, ascending row; nsplit [niter].  Either may be NULL.  -> 0, or -1 when n < k. */
REF_API int ref_train_coarse(const float* x, int64_t n, int d, const float* A, int64_t k, int niter, uint64_t seed, int64_t mppc,
                             int hot_start, float* Cc, double* obj, int64_t* nsplit) {
    if (n < k) return -1;
    int64_t ns;
    float* xs = rotated_sample(x, n, d, A, mppc * k, seed, 0, &ns);
    if (!hot_start) {
        int64_t* first = (int64_t*)malloc(sizeof(int64_t) * (size_t)k);
        ref_train_init_rows(ns, k, seed, 0, first);
        for (int64_t c = 0; c < k; c++) memcpy(Cc + c * d, xs + first[c] * d, sizeof(float) * (size_t)d);
        free(first);
        km_renorm(Cc, k, d);
    }
    int64_t* assign = (int64_t*)malloc(sizeof(int64_t) * (size_t)ns);
    float* cd = (float*)malloc(sizeof(float) * (size_t)ns);
    float* h = (float*)malloc(sizeof(float) * (size_t)k);
    for (int it = 0; it < niter; it++) {
        coarse_top1(xs, ns, d, Cc, k, assign, cd);
        double o = 0.0;
        for (int64_t i = 0; i < ns; i++) o += (double)cd[i];
        if (obj) obj[it] = o;
        km_update(xs, ns, d, 0, d, assign, k, Cc, h);
        const int64_t s = ref_split_clusters(Cc, k, d, h, ns, seed, 0, (uint64_t)it);
        if (nsplit) nsplit[it] = s;
        km_renorm(Cc, k, d);
    }
    free(assign); free(cd); free(h); free(xs);
    return 0;
}

/* PQ codebooks pq [M, ksub, dsub] in/out (read when hot_start): x [n, d] rotated by A; with C (coarse centroids [nlist, d]) the
 * sample is replaced by its residual xr - C[top-1 list] (the fp32 subtraction of the encoding), without C (OPQ) it is used as is.
 * Then M independent L2 k-means, run s = 1 + m; assignment = the encoding argmin (fmaf chain of squared differences, lowest j on a
 * tie).  -> 0, or -1 when n < ksub. */
REF_API int ref_train_pq(const float* x, int64_t n, int d, const float* A, const float* Cc, int64_t nlist, int M, int ksub, int dsub,
                         int niter, uint64_t seed, int64_t mppc, int hot_start, float* pq) {
    if (n < ksub) return -1;
    int64_t ns;
    float* xs = rotated_sample(x, n, d, A, mppc * ksub, seed, 1, &ns);
    if (Cc) {
        int64_t* list = (int64_t*)malloc(sizeof(int64_t) * (size_t)ns);
        float* cd = (float*)malloc(sizeof(float) * (size_t)ns);
        coarse_top1(xs, ns, d, Cc, nlist, list, cd);
        for (int64_t i = 0; i < ns; i++)
            for (int t = 0; t < d; t++) xs[i * d + t] = xs[i * d + t] - Cc[list[i] * d + t];
        free(list); free(cd);
    }
#pragma omp parallel for schedule(dynamic, 1)
    for (int m = 0; m < M; m++) {
        float* cb = pq + (size_t)m * ksub * dsub;
        const uint64_t s = 1 + (uint64_t)m;
        if (!hot_start) {
            int64_t* first = (int64_t*)malloc(sizeof(int64_t) * (size_t)ksub);
            ref_train_init_rows(ns, ksub, seed, s, first);
            for (int c = 0; c < ksub; c++) memcpy(cb + c * dsub, xs + first[c] * d + m * dsub, sizeof(float) * (size_t)dsub);
            free(first);
        }
        int64_t* assign = (int64_t*)malloc(sizeof(int64_t) * (size_t)ns);
        float* h = (float*)malloc(sizeof(float) * (size_t)ksub);
        for (int it = 0; it < niter; it++) {
            for (int64_t i = 0; i < ns; i++) {
                const float* r = xs + i * d + m * dsub;
                float best = INFINITY; int bj = 0;
                for (int j = 0; j < ksub; j++) {
                    const float* cw = cb + j * dsub;
                    float acc = 0.0f;
                    for (int t = 0; t < dsub; t++) { const float df = r[t] - cw[t]; acc = fmaf(df, df, acc); }
                    if (acc < best) { best = acc; bj = j; }
                }
                assign[i] = bj;
            }
            km_update(xs, ns, d, m * dsub, dsub, assign, ksub, cb, h);
            ref_split_clusters(cb, ksub, dsub, h, ns, seed, s, (uint64_t)it);
        }
        free(assign); free(h);
    }
    free(xs);
    return 0;
}
