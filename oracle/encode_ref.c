/*
 * oracle/encode_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the encoding that faiss.IndexPreTransform(OPQ) -> IndexIVFPQ::add_with_ids (faiss 1.6.x, by_residual) [3P]
 * performs when reference build_phrase_index.py:145-150,156-279 fills a phrase index, with a fixed floating-point order
 * (DESIGN.md 3.1).  It extends the search restatement: ivfpq_ref.c is compiled into this library, so the rotation and the coarse
 * quantizer are literally the same code as the search oracle's.
 *   xr   = x A^T                         ref_rotate (sequential FMA chains)
 *   list = top-1 of ref_coarse           same scores and tie rule as nprobe = 1: on an exact tie the smallest list id wins
 *                                        (faiss' k = 1 heap keeps the first maximum it sees: strict <)
 *   r    = xr - C[list]                  element-wise fp32
 *   dist[m][j] = fmaf chain over t of d_t * d_t, acc from +0.0f, d_t = r[8m+t] - pq[m][j][t]
 *   code[m] = argmin_j dist[m][j], strict <: the lowest j wins a tie (ProductQuantizer::compute_code, dsub < 16)
 * What pins it: tests/test_add_cpu.py (numpy restatement bit for bit, lists == ref_coarse top-1, codes == the fp64 argmin outside
 * rounding gaps, planted ties).
 *
 * Only tests/, __graft_entry__.smoke() and tools/bench_add.py's host baseline may load this library.
 */
#include "ivfpq_ref.c"

/* list_no [n] int64, codes [n, M] (m ascending).  A row whose best score does not beat the heap's neutral value (-FLT_MAX) gets
 * list -1 and zero codes; the callers reject it. */
REF_API void ref_encode(const float* x, int64_t n, int d, const float* A, const float* C, int64_t nlist, const float* pq, int M,
                        int ksub, int dsub, int64_t* list_no, uint8_t* codes) {
    const int64_t chunk = 4096;                 /* bounds the coarse score matrix of ref_coarse */
    float* xr = (float*)malloc(sizeof(float) * (size_t)(n < chunk ? n : chunk) * d + 4);
    for (int64_t o = 0; o < n; o += chunk) {
        const int64_t m = n - o < chunk ? n - o : chunk;
        ref_rotate(x + o * d, m, d, A, xr);
        ref_coarse(xr, m, d, C, nlist, 1, NULL, list_no + o);
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < m; i++) {
            uint8_t* code = codes + (size_t)(o + i) * M;
            const int64_t l = list_no[o + i];
            if (l < 0) { memset(code, 0, M); continue; }
            float r[dsub];
            for (int mm = 0; mm < M; mm++) {
                for (int t = 0; t < dsub; t++) r[t] = xr[i * d + mm * dsub + t] - C[(size_t)l * d + mm * dsub + t];
                float best = INFINITY; int bj = 0;
                for (int j = 0; j < ksub; j++) {
                    const float* cw = pq + ((size_t)mm * ksub + j) * dsub;
                    float acc = 0.0f;
                    for (int t = 0; t < dsub; t++) { const float df = r[t] - cw[t]; acc = fmaf(df, df, acc); }
                    if (acc < best) { best = acc; bj = j; }
                }
                code[mm] = (uint8_t)bj;
            }
        }
    }
    free(xr);
}
