/*
 * oracle/ivfpq_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the search arithmetic DensePhrases delegates to FAISS:
 *   faiss.IndexPreTransform(OPQMatrix(768,96), IndexIVFPQ(IndexFlatIP(768), 768, nlist, 96, 8, IP))
 * built at reference build_phrase_index.py:113-116, searched at
 * reference densephrases/index.py:200 (self.index.search) and reconstructed from at
 * reference densephrases/index.py:31,286,296 (reconst_fn).
 *
 * The algorithm lives in the un-vendored third-party dependency faiss-gpu==1.6.5
 * (reference requirements.txt:2); it is restated here from its published algorithm
 * (IndexPreTransform::search -> LinearTransform::apply -> IndexIVF::search ->
 *  IndexFlatIP coarse top-nprobe -> IVFPQScanner<IP, CMin, PQDecoder8>::scan_codes with
 *  precompute_mode 2 -> heap_pop/heap_push/heap_reorder), see SURVEY.md Appendix A.
 *
 * PARITY UNPINNED at the FAISS boundary: the reference repo holds no golden vectors for this path
 * (SURVEY.md 8c) and faiss itself is not installable here. What pins this restatement instead:
 *   tests/test_oracle.py: (1) numpy restatement == this C restatement bit-for-bit,
 *   (2) both == exhaustive fp64 scoring of decoded vectors over the probed lists,
 *   (3) search score == <xr, reconstruct(id)> identity.
 *
 * Floating-point definition (the one degree of freedom FAISS leaves to BLAS/SIMD): every inner
 * product (OPQ rotation, coarse scores, dis0, LUT entries) is ONE sequential fp32 FMA chain,
 * t ascending, starting from +0.0f:   acc = fmaf(a[t], b[t], acc).
 * That is exactly what a k-ascending FFMA GEMM computes on the GPU, so the CUDA path can be
 * held to bit-identical scores.  The ADC sum is FAISS's own: dis = dis0; for m asc: dis += LUT[m][c[m]].
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define REF_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * Counter-based generator shared (bit-for-bit) by oracle, numpy helper and the CUDA generator.
 * ---------------------------------------------------------------------------------------- */
static inline uint64_t mix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
static inline uint64_t rnd64(uint64_t seed, uint64_t stream, uint64_t a, uint64_t b) {
    return mix64(mix64(mix64(seed ^ (stream * 0xA24BAED4963EE407ull)) + a) + b);
}
/* Irwin-Hall(4) of 16-bit fields: integer arithmetic + one exact int->float + one multiply. */
static inline float approx_normal(uint64_t u, float sigma_over_std) {
    int32_t s = (int32_t)(u & 0xFFFF) + (int32_t)((u >> 16) & 0xFFFF) + (int32_t)((u >> 32) & 0xFFFF) +
                (int32_t)(u >> 48) - 131070;
    return (float)s * sigma_over_std;
}
#define IH4_STD 37837.227f /* 65536/sqrt(3) */

enum { STREAM_CODES = 1, STREAM_CENTROIDS = 2, STREAM_PQ = 3 };

REF_API uint64_t ref_rnd64(uint64_t seed, uint64_t stream, uint64_t a, uint64_t b) { return rnd64(seed, stream, a, b); }

/* codes of list `list_no`, rows j0 .. j0+n-1, row-major [n][code_size] (code_size multiple of 8) */
REF_API void ref_gen_codes(uint64_t seed, int64_t list_no, int64_t j0, int64_t n, int code_size, uint8_t* out) {
    int words = code_size / 8;
    for (int64_t j = 0; j < n; j++)
        for (int w = 0; w < words; w++) {
            uint64_t u = rnd64(seed, STREAM_CODES, (uint64_t)list_no, (uint64_t)((j0 + j) * words + w));
            memcpy(out + j * code_size + 8 * w, &u, 8); /* little endian */
        }
}
/* codes of several whole lists, list i written at row offs[i] of out (OpenMP over lists) */
REF_API void ref_gen_codes_lists(uint64_t seed, const int64_t* lists, int64_t nl, const int64_t* lens, const int64_t* offs,
                                 int code_size, uint8_t* out) {
#pragma omp parallel for schedule(dynamic, 1)
    for (int64_t i = 0; i < nl; i++) ref_gen_codes(seed, lists[i], 0, lens[i], code_size, out + (size_t)offs[i] * code_size);
}
REF_API void ref_gen_centroids(uint64_t seed, int64_t l0, int64_t n, int d, float sigma, float* out) {
    float sc = sigma / IH4_STD;
    for (int64_t l = 0; l < n; l++)
        for (int t = 0; t < d; t++) out[l * d + t] = approx_normal(rnd64(seed, STREAM_CENTROIDS, (uint64_t)(l0 + l), (uint64_t)t), sc);
}
REF_API void ref_gen_pq(uint64_t seed, int M, int ksub, int dsub, float sigma, float* out) {
    float sc = sigma / IH4_STD;
    for (int64_t e = 0; e < (int64_t)M * ksub; e++)
        for (int t = 0; t < dsub; t++) out[e * dsub + t] = approx_normal(rnd64(seed, STREAM_PQ, (uint64_t)e, (uint64_t)t), sc);
}

/* ------------------------------------------------------------------------------------------
 * Sequential-FMA inner product (the fp definition above).
 * ---------------------------------------------------------------------------------------- */
static inline float dot_seq(const float* a, const float* b, int d) {
    float acc = 0.0f;
    for (int t = 0; t < d; t++) acc = fmaf(a[t], b[t], acc);
    return acc;
}
/* out[i][o] = dot_seq(x[i], W[o])  (x [n,d], W [m,d], out [n,m]); 8 independent chains for ILP. */
static void matmul_nt_seq(const float* x, int64_t n, const float* W, int64_t m, int d, float* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        const float* xi = x + i * d;
        int64_t o = 0;
        for (; o + 8 <= m; o += 8) {
            float a0 = 0, a1 = 0, a2 = 0, a3 = 0, a4 = 0, a5 = 0, a6 = 0, a7 = 0;
            const float* w = W + o * d;
            for (int t = 0; t < d; t++) {
                float xv = xi[t];
                a0 = fmaf(xv, w[t], a0);
                a1 = fmaf(xv, w[d + t], a1);
                a2 = fmaf(xv, w[2 * d + t], a2);
                a3 = fmaf(xv, w[3 * d + t], a3);
                a4 = fmaf(xv, w[4 * d + t], a4);
                a5 = fmaf(xv, w[5 * d + t], a5);
                a6 = fmaf(xv, w[6 * d + t], a6);
                a7 = fmaf(xv, w[7 * d + t], a7);
            }
            float* r = out + i * m + o;
            r[0] = a0; r[1] = a1; r[2] = a2; r[3] = a3; r[4] = a4; r[5] = a5; r[6] = a6; r[7] = a7;
        }
        for (; o < m; o++) out[i * m + o] = dot_seq(xi, W + o * d, d);
    }
}

/* IndexPreTransform::apply_chain -> LinearTransform::apply_noalloc (OPQ, no bias): xr = x A^T.
 * A is [d_out, d_in] row-major (index.py:32 reshapes it to [d, d]). */
REF_API void ref_rotate(const float* x, int64_t n, int d, const float* A, float* xr) { matmul_nt_seq(x, n, A, d, d, xr); }

/* ------------------------------------------------------------------------------------------
 * FAISS Heap.h, CMin<float, int64>: root = current minimum of the kept k; textbook 1-based
 * sift-down / sift-up comparing VALUES ONLY (no id tie-break in 1.6.x).
 * ---------------------------------------------------------------------------------------- */
#define NEUTRAL (-FLT_MAX)
static inline void heap_pop(size_t k, float* bh_val, int64_t* bh_ids) {
    bh_val--; bh_ids--; /* 1-based */
    float val = bh_val[k];
    size_t i = 1, i1, i2;
    while (1) {
        i1 = i << 1; i2 = i1 + 1;
        if (i1 > k) break;
        if (i2 == k + 1 || bh_val[i1] < bh_val[i2]) {
            if (val < bh_val[i1]) break;
            bh_val[i] = bh_val[i1]; bh_ids[i] = bh_ids[i1]; i = i1;
        } else {
            if (val < bh_val[i2]) break;
            bh_val[i] = bh_val[i2]; bh_ids[i] = bh_ids[i2]; i = i2;
        }
    }
    bh_val[i] = bh_val[k]; bh_ids[i] = bh_ids[k];
}
static inline void heap_push(size_t k, float* bh_val, int64_t* bh_ids, float val, int64_t id) {
    bh_val--; bh_ids--;
    size_t i = k, i_father;
    while (i > 1) {
        i_father = i >> 1;
        if (!(val < bh_val[i_father])) break;
        bh_val[i] = bh_val[i_father]; bh_ids[i] = bh_ids[i_father]; i = i_father;
    }
    bh_val[i] = val; bh_ids[i] = id;
}
static inline void heap_heapify(size_t k, float* v, int64_t* ids) {
    for (size_t i = 0; i < k; i++) { v[i] = NEUTRAL; ids[i] = -1; }
}
static void heap_reorder(size_t k, float* bh_val, int64_t* bh_ids) {
    size_t i, ii;
    for (i = 0, ii = 0; i < k; i++) {
        float val = bh_val[0]; int64_t id = bh_ids[0];
        heap_pop(k - i, bh_val, bh_ids);
        bh_val[k - ii - 1] = val; bh_ids[k - ii - 1] = id;
        if (id != -1) ii++;
    }
    memmove(bh_val, bh_val + k - ii, ii * sizeof(*bh_val));
    memmove(bh_ids, bh_ids + k - ii, ii * sizeof(*bh_ids));
    for (; ii < k; ii++) { bh_val[ii] = NEUTRAL; bh_ids[ii] = -1; }
}

/* IndexFlatIP::search as coarse quantizer: top-nprobe of S[i,:] = xr[i] . C^T, descending.
 * Slots beyond nlist get key -1 (nlist < nprobe; C1: IVF1 with nprobe 256). cd may be NULL. */
REF_API void ref_coarse(const float* xr, int64_t n, int d, const float* C, int64_t nlist, int nprobe,
                        float* cd, int64_t* key) {
    float* S = (float*)malloc(sizeof(float) * (size_t)n * (size_t)nlist);
    matmul_nt_seq(xr, n, C, nlist, d, S);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        float* hv = (float*)malloc(sizeof(float) * nprobe);
        int64_t* hi = key + i * nprobe;
        heap_heapify(nprobe, hv, hi);
        for (int64_t j = 0; j < nlist; j++) {
            float ip = S[i * nlist + j];
            if (hv[0] < ip) { heap_pop(nprobe, hv, hi); heap_push(nprobe, hv, hi, ip, j); }
        }
        heap_reorder(nprobe, hv, hi);
        if (cd) memcpy(cd + i * nprobe, hv, sizeof(float) * nprobe);
        free(hv);
    }
    free(S);
}

/* ProductQuantizer::compute_inner_prod_table for one query: LUT[m][j] = <xr[m*dsub..], pq[m][j]> */
REF_API void ref_lut(const float* xr_row, const float* pq, int M, int ksub, int dsub, float* lut) {
    for (int m = 0; m < M; m++)
        for (int j = 0; j < ksub; j++) lut[m * ksub + j] = dot_seq(xr_row + m * dsub, pq + ((size_t)m * ksub + j) * dsub, dsub);
}

/* ------------------------------------------------------------------------------------------
 * Inverted lists: explicit (arrays) or synthetic (regenerated per probed list from the seed).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int d, M, ksub, dsub, code_size;
    int64_t nlist;
    const float* A;          /* [d,d]  OPQ */
    const float* C;          /* [nlist,d] centroids, or NULL when synthetic_centroids */
    const float* pq;         /* [M,ksub,dsub] */
    const int64_t* list_len; /* [nlist] */
    const int64_t* list_off; /* [nlist] exclusive prefix of list_len (row offset into codes/ids) */
    const uint8_t* codes;    /* [ntotal, code_size] list-major, or NULL when synthetic */
    const int64_t* ids;      /* [ntotal] list-major, or NULL -> id = list_off[l] + j */
    uint64_t seed;           /* synthetic seed */
    float centroid_sigma;    /* synthetic centroids when C == NULL */
    const int64_t* code_off; /* optional: row offset of each list inside `codes` when only some lists are resident
                                (bench cpu_baseline keeps just the probed lists in RAM); NULL -> list_off */
} ref_index;

static const uint8_t* list_codes(const ref_index* ix, int64_t l, uint8_t** scratch, size_t* cap) {
    int64_t len = ix->list_len[l];
    if (ix->codes) return ix->codes + (size_t)(ix->code_off ? ix->code_off[l] : ix->list_off[l]) * ix->code_size;
    size_t need = (size_t)len * ix->code_size;
    if (need > *cap) { free(*scratch); *scratch = (uint8_t*)malloc(need ? need : 1); *cap = need; }
    ref_gen_codes(ix->seed, l, 0, len, ix->code_size, *scratch);
    return *scratch;
}
static inline int64_t list_id(const ref_index* ix, int64_t l, int64_t j) {
    return ix->ids ? ix->ids[ix->list_off[l] + j] : ix->list_off[l] + j;
}
static void centroid_row(const ref_index* ix, int64_t l, float* out) {
    if (ix->C) memcpy(out, ix->C + (size_t)l * ix->d, sizeof(float) * ix->d);
    else ref_gen_centroids(ix->seed, l, 1, ix->d, ix->centroid_sigma, out);
}

/* IndexIVF::search_preassigned + IVFPQScanner (IP, by_residual, precompute_mode 2), parallel_mode 0
 * (OpenMP over queries).  key [n,nprobe] from ref_coarse (or any preassignment).  */
REF_API void ref_search_preassigned(const ref_index* ix, const float* xr, int64_t n, const int64_t* key, int nprobe,
                                    int k, float* D, int64_t* I, int64_t* ncodes_scanned) {
    int64_t total = 0;
#pragma omp parallel reduction(+ : total)
    {
        float* lut = (float*)malloc(sizeof(float) * ix->M * ix->ksub);
        float* cen = (float*)malloc(sizeof(float) * ix->d);
        uint8_t* scratch = NULL; size_t cap = 0;
#pragma omp for schedule(dynamic, 1)
        for (int64_t i = 0; i < n; i++) {
            const float* q = xr + i * ix->d;
            float* simi = D + i * k; int64_t* idxi = I + i * k;
            ref_lut(q, ix->pq, ix->M, ix->ksub, ix->dsub, lut);           /* init_query_IP */
            heap_heapify(k, simi, idxi);
            for (int r = 0; r < nprobe; r++) {
                int64_t l = key[i * nprobe + r];
                if (l < 0) continue;
                int64_t len = ix->list_len[l];
                if (len == 0) continue;
                centroid_row(ix, l, cen);
                float dis0 = dot_seq(q, cen, ix->d);                       /* set_list: fvec_inner_product(qi, centroid) */
                const uint8_t* codes = list_codes(ix, l, &scratch, &cap);
                /* scan_list_with_table.  Four code rows are summed side by side (four independent chains, each still
                 * dis = dis0; for m asc: dis += LUT[m][c[m]] -- the values are those of the one-row loop bit for bit) so that
                 * the 96-long dependent add chain of one row overlaps the next rows' on any core; the heap sees the rows in
                 * storage order. */
                const int64_t cs = ix->code_size; const int M = ix->M, ksub = ix->ksub;
                int64_t j = 0;
                for (; j + 4 <= len; j += 4) {
                    const uint8_t* c0 = codes + j * cs; const uint8_t* c1 = c0 + cs; const uint8_t* c2 = c1 + cs; const uint8_t* c3 = c2 + cs;
                    const float* tab = lut;
                    float d0 = dis0, d1 = dis0, d2 = dis0, d3 = dis0;
                    for (int m = 0; m < M; m++) { d0 += tab[c0[m]]; d1 += tab[c1[m]]; d2 += tab[c2[m]]; d3 += tab[c3[m]]; tab += ksub; }
                    if (simi[0] < d0) { heap_pop(k, simi, idxi); heap_push(k, simi, idxi, d0, list_id(ix, l, j)); }
                    if (simi[0] < d1) { heap_pop(k, simi, idxi); heap_push(k, simi, idxi, d1, list_id(ix, l, j + 1)); }
                    if (simi[0] < d2) { heap_pop(k, simi, idxi); heap_push(k, simi, idxi, d2, list_id(ix, l, j + 2)); }
                    if (simi[0] < d3) { heap_pop(k, simi, idxi); heap_push(k, simi, idxi, d3, list_id(ix, l, j + 3)); }
                }
                for (; j < len; j++) {
                    const uint8_t* c = codes + j * cs;
                    const float* tab = lut;
                    float dis = dis0;
                    for (int m = 0; m < M; m++) { dis += tab[c[m]]; tab += ksub; }
                    if (simi[0] < dis) { heap_pop(k, simi, idxi); heap_push(k, simi, idxi, dis, list_id(ix, l, j)); }
                }
                total += len;
            }
            heap_reorder(k, simi, idxi);
        }
        free(lut); free(cen); free(scratch);
    }
    if (ncodes_scanned) *ncodes_scanned = total;
}

/* faiss.Index.search for the whole chain (index.py:200): rotate, coarse, scan. */
REF_API void ref_search(const ref_index* ix, const float* x, int64_t n, int k, int nprobe, float* D, int64_t* I,
                        int64_t* key_out /* [n,nprobe] or NULL */, int64_t* ncodes_scanned) {
    float* xr = (float*)malloc(sizeof(float) * (size_t)n * ix->d);
    int64_t* key = key_out ? key_out : (int64_t*)malloc(sizeof(int64_t) * (size_t)n * nprobe);
    ref_rotate(x, n, ix->d, ix->A, xr);
    if (ix->C) ref_coarse(xr, n, ix->d, ix->C, ix->nlist, nprobe, NULL, key);
    else {
        float* C = (float*)malloc(sizeof(float) * (size_t)ix->nlist * ix->d);
        ref_gen_centroids(ix->seed, 0, ix->nlist, ix->d, ix->centroid_sigma, C);
        ref_coarse(xr, n, ix->d, C, ix->nlist, nprobe, NULL, key);
        free(C);
    }
    ref_search_preassigned(ix, xr, n, key, nprobe, k, D, I, ncodes_scanned);
    if (!key_out) free(key);
    free(xr);
}

/* IndexIVFPQ::reconstruct_from_offset: v = centroid[l] + pq.decode(code) -- ROTATED space
 * (index.py:282-300; the caller un-rotates with R, index.py:340,365). found[i]=0 -> zeros. */
REF_API void ref_reconstruct_at(const ref_index* ix, const int64_t* list_no, const int64_t* offset, int64_t m,
                                float* out, uint8_t* found) {
    uint8_t* row = (uint8_t*)malloc(ix->code_size);
    for (int64_t i = 0; i < m; i++) {
        float* v = out + i * ix->d;
        int64_t l = list_no[i], j = offset[i];
        if (l < 0 || l >= ix->nlist || j < 0 || j >= ix->list_len[l]) {
            memset(v, 0, sizeof(float) * ix->d); if (found) found[i] = 0; continue;
        }
        if (ix->codes) memcpy(row, ix->codes + (size_t)((ix->code_off ? ix->code_off[l] : ix->list_off[l]) + j) * ix->code_size, ix->code_size);
        else ref_gen_codes(ix->seed, l, j, 1, ix->code_size, row);
        centroid_row(ix, l, v);
        for (int mm = 0; mm < ix->M; mm++) {
            const float* cb = ix->pq + ((size_t)mm * ix->ksub + row[mm]) * ix->dsub;
            for (int t = 0; t < ix->dsub; t++) v[mm * ix->dsub + t] = cb[t] + v[mm * ix->dsub + t]; /* decode then += centroid */
        }
        if (found) found[i] = 1;
    }
    free(row);
}

REF_API int ref_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
REF_API void ref_set_num_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}
REF_API int ref_sizeof_index(void) { return (int)sizeof(ref_index); }
