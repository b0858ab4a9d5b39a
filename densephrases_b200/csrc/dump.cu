// dump.cu -- the phrase dump's device step (generate_phrase_vecs.py --do_dump; embed_utils.py get_metadata -> filter_metadata ->
// compress_metadata, :40-191): from the phrase tower's fp32 outputs of one forward batch, select the rows a document keeps,
// re-index their ends, quantise them to int8 and compact them into one page-locked host buffer.
//
// Rows: feature f contributes its valid rows [row_lo, row_hi) (the reference's [to+1, len(tokens)-1)), in batch order; a document
// is a run of consecutive features, and may continue from the previous batch (its kept count so far comes in as doc_base).
// Keep rule: float(filter_start) > float(thr) or float(filter_end) > float(thr) -- numpy compares a float32 array with a Python
//   float in float32, so the threshold is rounded to fp32 first.
// Short index of a kept row: doc_base + the number of kept rows of its document before it in this batch.
// start2end[k] of a kept row at position p of its feature: the short index of row p + k when p + k < row_hi and that row passes the
//   filter_end test, else -1.
// Quantisation: rint(clip((x - offset) * scale, -128, 127)) as separate fp32 operations (no FMA), rounded half to even.
// Empty documents (filter_metadata's fallback): for each document that has kept no row so far (neither before this batch nor in
//   it) and whose caller still needs a fallback, the first row of this batch with filter_start > -999999 is quantised into its
//   own slot.
//
// Two kernels: one CTA computes the flags, the kept-row scan and each document's counts; then one CTA per kept row (and per fallback
// slot) quantises the row and writes its f2o index and start2end straight into the caller's pinned buffer through its device
// mapping, so the only device-to-host traffic is the kept rows.
#include "common.cuh"
#include "../../include/dph_b200.h"
#include <vector>

#define DUMP_SCAN_THREADS 1024
#define DUMP_ROW_THREADS 192           // 768 / 4: one float4 per thread
#define DUMP_MAX_L 64
#define DUMP_MAX_S 512

struct DumpArgs {
    const float* start;                // [B,S,768]
    const float* filt;                 // [B,S,2]
    const int* feat;                   // [B,4] row_lo, row_hi, doc slot, document-level index of row_lo
    const int* rowoff;                 // [B+1] first batch row of each feature
    const int* docoff;                 // [n_doc+1] first batch row of each document
    const int* doc;                    // [n_doc,2] kept rows before this batch, needs a fallback row (0/1)
    unsigned char* flags;              // [R] bit 0: filter_start test, bit 1: filter_end test
    int* scan;                         // [R] exclusive count of kept rows before each row
    int* kept_row;                     // [R] batch row of each kept row
    int* fb_row;                       // [n_doc] fallback batch row, -1 when none
    int* total;                        // kept rows of the batch (device copy of n_kept)
    // outputs (device view of the pinned buffer)
    long long* n_kept;
    int* doc_kept;                     // [n_doc]
    long long* fb_f2o;                 // [n_doc]
    signed char* rows;                 // [R,768]
    long long* f2o;                    // [R]
    int* s2e;                          // [R,L]
    signed char* fb_rows;              // [n_doc,768]
    int B, S, R, n_doc, L;
    float thr, offset, scale;
};

__device__ __forceinline__ int dump_feature(const int* rowoff, int B, int r) {     // last f with rowoff[f] <= r
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (rowoff[mid] <= r) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(DUMP_SCAN_THREADS) dump_select_kernel(DumpArgs a) {
    __shared__ int warp_sum[DUMP_SCAN_THREADS / 32];
    __shared__ int carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < a.R; base += DUMP_SCAN_THREADS) {
        const int r = base + tid;
        int keep = 0;
        if (r < a.R) {
            const int f = dump_feature(a.rowoff, a.B, r);
            const int p = a.feat[4 * f] + (r - a.rowoff[f]);
            const float2 lg = reinterpret_cast<const float2*>(a.filt)[(size_t)f * a.S + p];
            const int s = lg.x > a.thr, e = lg.y > a.thr;
            a.flags[r] = (unsigned char)(s | (e << 1));
            keep = s | e;
        }
        int incl = keep;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int w = warp_sum[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += v;
            }
            warp_sum[lane] = wi - w;
        }
        __syncthreads();
        const int ex = carry + warp_sum[warp] + incl - keep;
        if (r < a.R) {
            a.scan[r] = ex;
            if (keep) a.kept_row[ex] = r;
        }
        __syncthreads();
        if (tid == DUMP_SCAN_THREADS - 1) carry = ex + keep;
        __syncthreads();
    }
    const int total = carry;
    if (tid == 0) { *a.n_kept = total; *a.total = total; }
    for (int d = tid; d < a.n_doc; d += DUMP_SCAN_THREADS) {
        const int lo = a.docoff[d], hi = a.docoff[d + 1];
        const int kept = (hi < a.R ? a.scan[hi] : total) - (lo < a.R ? a.scan[lo] : total);
        a.doc_kept[d] = kept;
        int fb = -1;
        long long fo = -1;
        if (a.doc[2 * d + 1] && kept == 0) {            // only a document with nothing kept so far needs the fallback row
            for (int r = lo; r < hi; r++) {
                const int f = dump_feature(a.rowoff, a.B, r);
                const int p = a.feat[4 * f] + (r - a.rowoff[f]);
                if (a.filt[((size_t)f * a.S + p) * 2] > -999999.0f) {
                    fb = r;
                    fo = (long long)a.feat[4 * f + 3] + (r - a.rowoff[f]);
                    break;
                }
            }
        }
        a.fb_row[d] = fb;
        a.fb_f2o[d] = fo;
    }
}

__device__ __forceinline__ signed char dump_q(float x, float offset, float scale) {
    const float y = fminf(fmaxf(__fmul_rn(__fsub_rn(x, offset), scale), -128.0f), 127.0f);
    return (signed char)__float2int_rn(y);
}

__global__ void __launch_bounds__(DUMP_ROW_THREADS) dump_rows_kernel(DumpArgs a) {
    const int b = blockIdx.x, t = threadIdx.x;
    int r;
    signed char* dst;
    if (b < a.R) {
        if (b >= *a.total) return;
        r = a.kept_row[b];
        dst = a.rows + (size_t)b * DPH_D;
    } else {
        r = a.fb_row[b - a.R];
        if (r < 0) return;
        dst = a.fb_rows + (size_t)(b - a.R) * DPH_D;
    }
    const int f = dump_feature(a.rowoff, a.B, r);
    const int lo = a.feat[4 * f], p = lo + (r - a.rowoff[f]);
    const float4 v = reinterpret_cast<const float4*>(a.start + ((size_t)f * a.S + p) * DPH_D)[t];
    char4 q;
    q.x = dump_q(v.x, a.offset, a.scale); q.y = dump_q(v.y, a.offset, a.scale);
    q.z = dump_q(v.z, a.offset, a.scale); q.w = dump_q(v.w, a.offset, a.scale);
    reinterpret_cast<char4*>(dst)[t] = q;
    if (b >= a.R) return;
    if (t == 0) a.f2o[b] = (long long)a.feat[4 * f + 3] + (p - lo);
    if (t < a.L) {
        const int hi = a.feat[4 * f + 1], d = a.feat[4 * f + 2];
        int v2 = -1;
        if (p + t < hi && (a.flags[r + t] & 2)) v2 = a.doc[2 * d] + a.scan[r + t] - a.scan[a.docoff[d]];
        a.s2e[(size_t)b * a.L + t] = v2;
    }
}

static inline int64_t dump_align(int64_t x) { return (x + 255) & ~(int64_t)255; }

DPH_API int64_t dph_dump_layout(int64_t R, int n_doc, int L, int64_t* offsets) {
    if (R < 0 || n_doc < 0 || L < 1) return -1;
    const int64_t sizes[7] = {8, 4 * (int64_t)n_doc, 8 * (int64_t)n_doc, R * DPH_D, 8 * R, 4 * R * L, (int64_t)n_doc * DPH_D};
    int64_t at = 0;
    for (int i = 0; i < 7; i++) { offsets[i] = at; at = dump_align(at + sizes[i]); }
    return at;
}

struct DumpScratch { void* p = nullptr; size_t cap = 0; };
static int dump_grow(DumpScratch& s, size_t bytes) {
    if (bytes <= s.cap) return 0;
    if (s.p) { cudaFree(s.p); s.p = nullptr; s.cap = 0; }
    DPH_CUDA(cudaMalloc(&s.p, bytes));
    s.cap = bytes;
    return 0;
}

DPH_API int dph_dump_select(const float* start, const float* filt, int B, int S, const int32_t* feat, int n_doc, const int32_t* doc,
                            int max_answer_length, double filter_threshold, double dense_offset, double dense_scale, void* out,
                            int64_t out_bytes, void* cuda_stream) {
    DPH_CHECK(start && filt && feat && doc && out, "dump_select: null buffer");
    DPH_CHECK(((uintptr_t)start & 15) == 0 && ((uintptr_t)filt & 7) == 0, "dump_select: start must be 16-byte and filt 8-byte aligned");
    DPH_CHECK(((uintptr_t)out & 7) == 0, "dump_select: out must be 8-byte aligned");
    DPH_CHECK(B >= 1 && S >= 1 && S <= DUMP_MAX_S, "dump_select: B >= 1 and 1 <= S <= 512");
    DPH_CHECK(n_doc >= 1, "dump_select: n_doc >= 1");
    DPH_CHECK(max_answer_length >= 1 && max_answer_length <= DUMP_MAX_L, "dump_select: 1 <= max_answer_length <= 64");
    cudaStream_t st = (cudaStream_t)cuda_stream;
    // feature table: rows in range, documents in order and contiguous, every document used
    std::vector<int32_t> host((size_t)B + 1 + (size_t)n_doc + 1);
    int32_t* rowoff = host.data();
    int32_t* docoff = rowoff + B + 1;
    int64_t R = 0;
    int prev = -1;
    for (int f = 0; f < B; f++) {
        const int lo = feat[4 * f], hi = feat[4 * f + 1], d = feat[4 * f + 2];
        DPH_CHECK(lo >= 0 && lo <= hi && hi <= S, "dump_select: feature rows must satisfy 0 <= row_lo <= row_hi <= S");
        DPH_CHECK(feat[4 * f + 3] >= 0, "dump_select: document-level row index must be >= 0");
        DPH_CHECK(d == prev || d == prev + 1, "dump_select: document slots must run 0, 1, ... over consecutive features");
        if (d != prev) docoff[d] = (int32_t)R;
        prev = d;
        rowoff[f] = (int32_t)R;
        R += hi - lo;
    }
    DPH_CHECK(prev == n_doc - 1, "dump_select: n_doc must equal the number of document slots the features use");
    rowoff[B] = docoff[n_doc] = (int32_t)R;
    for (int d = 0; d < n_doc; d++) DPH_CHECK(doc[2 * d] >= 0, "dump_select: kept count before the batch must be >= 0");
    int64_t offs[7];
    const int64_t need = dph_dump_layout(R, n_doc, max_answer_length, offs);
    DPH_CHECK(out_bytes >= need, "dump_select: output buffer smaller than dph_dump_layout");
    char* dout = nullptr;
    DPH_CUDA(cudaHostGetDevicePointer((void**)&dout, out, 0));

    static DumpScratch scratch[64];
    int dev = 0;
    DPH_CUDA(cudaGetDevice(&dev));
    DumpScratch& sc = scratch[dev & 63];
    const size_t in_feat = (size_t)B * 16, in_tab = host.size() * 4, in_doc = (size_t)n_doc * 8;
    const size_t sizes[8] = {in_feat, in_tab, in_doc, (size_t)R, (size_t)R * 4, (size_t)R * 4, (size_t)n_doc * 4, 4};
    size_t so[8], tot = 0;
    for (int i = 0; i < 8; i++) { so[i] = tot; tot += (sizes[i] + 255) & ~(size_t)255; }
    DPH_TRY(dump_grow(sc, tot));
    char* base = (char*)sc.p;
    DPH_CUDA(cudaMemcpyAsync(base + so[0], feat, in_feat, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemcpyAsync(base + so[1], host.data(), in_tab, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemcpyAsync(base + so[2], doc, in_doc, cudaMemcpyHostToDevice, st));
    DumpArgs a{};
    a.start = start; a.filt = filt;
    a.feat = (const int*)(base + so[0]); a.rowoff = (const int*)(base + so[1]); a.docoff = a.rowoff + B + 1;
    a.doc = (const int*)(base + so[2]);
    a.flags = (unsigned char*)(base + so[3]); a.scan = (int*)(base + so[4]); a.kept_row = (int*)(base + so[5]); a.fb_row = (int*)(base + so[6]);
    a.total = (int*)(base + so[7]);
    a.n_kept = (long long*)(dout + offs[0]); a.doc_kept = (int*)(dout + offs[1]); a.fb_f2o = (long long*)(dout + offs[2]);
    a.rows = (signed char*)(dout + offs[3]); a.f2o = (long long*)(dout + offs[4]); a.s2e = (int*)(dout + offs[5]);
    a.fb_rows = (signed char*)(dout + offs[6]);
    a.B = B; a.S = S; a.R = (int)R; a.n_doc = n_doc; a.L = max_answer_length;
    a.thr = (float)filter_threshold; a.offset = (float)dense_offset; a.scale = (float)dense_scale;
    dump_select_kernel<<<1, DUMP_SCAN_THREADS, 0, st>>>(a);
    DPH_CUDA(cudaGetLastError());
    dump_rows_kernel<<<(unsigned)(R + n_doc), DUMP_ROW_THREADS, 0, st>>>(a);
    DPH_CUDA(cudaGetLastError());
    DPH_CUDA(cudaStreamSynchronize(st));
    return 0;
}
