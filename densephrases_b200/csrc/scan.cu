// scan.cu -- the PQ asymmetric-distance scan over the probed inverted lists and the top-k merge.
//
// Replaces faiss IVFPQScanner::scan_codes + the result heap behind self.index.search(...) at
// reference densephrases/index.py:200 (SURVEY.md 8a-10(iv), Appendix A).
//
// Work decomposition: the plan kernel linearises all in-shard (query, probe, 32-vector block) triples in
// canonical scan order; scan CTA c of G takes the contiguous range [T c/G, T (c+1)/G).  One persistent CTA
// per SM (the per-query LUT fills shared memory); inside a CTA each warp owns one 32-vector block per round,
// lane l <-> vector l.
//
// FAST (one query per gather, fp32 LUT).  Shared-memory gathers, not HBM, co-limit this scan (one 4-byte LUT gather per code
// byte).  The code blocks are stored lane-rotated (common.cuh: dph_blk_addr) and the LUT is stored as three [256][64] tables
// (32 sub-quantizers + 31 wrap copies per row), so that at step t lane l reads word (l + t%32) of row `code byte` of table t/32:
// the 32 lanes always hit 32 different banks -> every LDS is one conflict-free wavefront regardless of the code values.  One
// PRMT builds the address (code<<8 | lane*4), so a lookup is PRMT + LDS + FADD.  The rotated summation order differs from faiss'
// m-ascending order by at most eps (plan kernel), so the scores are used as a FILTER: each CTA keeps its best k+slack by filter
// score, the merge kernel re-scores the survivors in canonical order (bit-exact with the oracle) and PROVES that nothing that was
// dropped could have been in the top-k (T_k - max drop threshold > 2 eps); otherwise the query is flagged and re-run through
// EXACT mode.
//
// GROUPED (further down): QUAD (scan_quad_kernel, four queries per gather, 8-bit LUTs) is the default whenever long lists are shared
// by the batch (the reference's nprobe = 256); PAIR (scan_pair_kernel, two per gather, u16 LUTs) serves the k whose keep does not fit
// the quad kernel's candidate buffers.  search.cu (search_plan) picks the mode per batch.
//
// EXACT: canonical m-ascending fp32 sum for every code (bank conflicts and all) -- fallback/cross-check.
#include "index_internal.cuh"
#include "select.cuh"

struct ScanArgs {
    const uint8_t* codes; const long long* qpre; const DphSeg* segs; const int* nseg; const DphWork* work;
    const float* lut_canon;
    unsigned* gthr; unsigned long long* cand; const long long* cand_off; int* cand_cnt;
    long long n; int nprobe; int keep;
    const unsigned* mask; const long long* mask_off;     // filtered variants: the row mask, and the shard's first block of each list
    const DphQfView* qf;                                 // per-query filtered variant: the chunk's selectors (device memory, DESIGN.md 3.7)
};

#define NT DPH_SCAN_THREADS
#define NW DPH_SCAN_WARPS
#define SMEM_LUT_FAST (DPH_LUT_SCAN_FLOATS * 4)                 // 196608
#define SMEM_LUT_EXACT (DPH_LUT_CANON_FLOATS * 4 + NW * DPH_BLK_BYTES)   // 98304 + 49152

struct ScanShared {   // tail of the dynamic shared memory
    unsigned long long cbuf[DPH_CAND_CAP];
    DphSeg segtab[DPH_SEG_SMEM];
    SelectScratch sc;
    int cnt; unsigned thr; int base; int ndone; int ndone_snap; int pad[3];
};
static_assert(DPH_MAX_K + DPH_KEEP_SLACK <= DPH_CAND_CAP - NT, "one-query latch margin: the largest keep fits below the latch (scan_kernel)");

__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
// TMA-engine bulk prefetch of one contiguous code block into L2 (no register / shared-memory cost).
__device__ __forceinline__ void l2_prefetch_block(const void* p) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(p), "n"(DPH_BLK_BYTES) : "memory");
}
// The same two with an L2 eviction-priority policy (createpolicy): per-instruction hints only, no device-wide L2 set-aside.
__device__ __forceinline__ uint4 ldg_stream(const uint4* p, unsigned long long pol) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ void l2_prefetch_block(const void* p, unsigned long long pol) {
    asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;" :: "l"(p), "n"(DPH_BLK_BYTES), "l"(pol) : "memory");
}
__device__ __forceinline__ uint4 ldg_policy(const uint4* p, unsigned long long pol) {
    uint4 r;
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

extern __shared__ __align__(1024) unsigned char dph_smem[];
// The dynamic shared memory window of a kernel without static shared memory starts at this shared-space address on
// sm_90 (1 KB is reserved by the system); probed once at library init (dph_scan_setup_attrs), a mismatch is fatal.
#define DPH_DYN_SMEM_BASE 0x400

// One FAST lookup: PRMT builds (cta window bits | code << 8 | lane*4); the table base, the step offset and the window
// base are folded into the LDS immediate -> PRMT + LDS + FADD per code byte.
template <int IMM> __device__ __forceinline__ float lds_imm(unsigned addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(IMM));
    return v;
}
// The four running sums live in two float2 registers (dph_fadd2: two independent IEEE fp32 adds) -- the same per-component
// summation order as four scalar accumulators.
template <int T0> __device__ __forceinline__ void fast_word(unsigned wv, unsigned y, float2& a01, float2& a23) {
    constexpr int TB = DPH_DYN_SMEM_BASE + (T0 >> 5) * 65536 + (T0 & 31) * 4;   // T0 % 4 == 0: the 4 bytes share a table
    const float v0 = lds_imm<TB + 0>(__byte_perm(wv, y, 0x7504));
    const float v1 = lds_imm<TB + 4>(__byte_perm(wv, y, 0x7514));
    const float v2 = lds_imm<TB + 8>(__byte_perm(wv, y, 0x7524));
    const float v3 = lds_imm<TB + 12>(__byte_perm(wv, y, 0x7534));
    a01 = dph_fadd2(a01, make_float2(v0, v1));
    a23 = dph_fadd2(a23, make_float2(v2, v3));
}
template <int C> __device__ __forceinline__ void fast_chunk(const uint4& v, unsigned y, float2& a01, float2& a23) {
    fast_word<C * 16 + 0>(v.x, y, a01, a23);
    fast_word<C * 16 + 4>(v.y, y, a01, a23);
    fast_word<C * 16 + 8>(v.z, y, a01, a23);
    fast_word<C * 16 + 12>(v.w, y, a01, a23);
}

// Segment cursor: blocks are visited in increasing order, so a forward-only cursor finds the segment of work block b
// (relative to the query's first block).  The segment fields are cached in registers and re-read only when a
// segment boundary is crossed (every ~48 rounds at C2 sizes), all lanes reading the same table entry (broadcast).
struct SegCursor {
    int seg; unsigned wrel, wend; const uint4* base; int len; unsigned gstart; float dis0;
    __device__ __forceinline__ void init() { seg = -1; wrel = 0; wend = 0; base = nullptr; len = 0; gstart = 0; dis0 = 0.f; }
    __device__ __forceinline__ void seek(const DphSeg* __restrict__ tab, unsigned b, const uint8_t* codes) {
        if (b < wend) return;
        do { seg++; } while (b >= tab[seg].wend);
        const uint4 u0 = *reinterpret_cast<const uint4*>(tab + seg);
        const uint4 u1 = *(reinterpret_cast<const uint4*>(tab + seg) + 1);
        base = reinterpret_cast<const uint4*>(codes + (long long)(((unsigned long long)u0.y << 32) | u0.x) * DPH_BLK_BYTES);
        len = (int)u0.z; gstart = u0.w; dis0 = __uint_as_float(u1.x); wrel = u1.y; wend = u1.z;
    }
    __device__ __forceinline__ const uint4* ptr(unsigned b) const { return base + (size_t)(b - wrel) * (DPH_BLK_BYTES / 16); }
    __device__ __forceinline__ unsigned j0(unsigned b) const { return (b - wrel) * 32u; }       // the list row of lane 0 of work block b
};
// The filtered scan's cursor: also the segment's row of the mask, mrow[b] = the mask word of work block b (the list's block b - wrel,
// in the shard's block numbering).  The unfiltered scan keeps the plain SegCursor, so its code is what it was.
struct SegCursorF : SegCursor {
    const unsigned* mrow;
    __device__ __forceinline__ void seek(const DphSeg* __restrict__ tab, unsigned b, const uint8_t* codes, const ScanArgs& a) {
        if (b < wend) return;
        SegCursor::seek(tab, b, codes);
        mrow = a.mask + (a.mask_off[tab[seg].list] - (long long)wrel);
    }
};
// The per-query filtered scan's cursor (DESIGN.md 3.7).  A query with a selector (f >= 0) has as many work blocks in a segment as its
// selector has blocks in the segment's list: work block b is the list's block qblk[b] with the mask word qword[b] (the selector's CSR
// entries of the list, shifted by wrel).  A query without one (f = -1) walks every block of the list with the word ~0u.  The code
// address and the row numbers come from the list's block, so the scan positions are those of the unfiltered scan.
struct SegCursorQ : SegCursor {
    const unsigned* qblk; const unsigned* qword; int f;
    __device__ __forceinline__ void seek(const DphSeg* __restrict__ tab, unsigned b, const uint8_t* codes, const ScanArgs& a) {
        if (b < wend) return;
        SegCursor::seek(tab, b, codes);
        if (f >= 0) {
            const DphQfView& v = *a.qf;
            const long long e = v.base[f] + (long long)v.off[(long long)f * v.stride + (tab[seg].list - v.lo)] - (long long)wrel;
            qblk = v.blk + e; qword = v.word + e;
        }
    }
    __device__ __forceinline__ unsigned blk(unsigned b) const { return f >= 0 ? __ldg(qblk + b) : b - wrel; }
    __device__ __forceinline__ const uint4* ptr(unsigned b) const { return base + (size_t)blk(b) * (DPH_BLK_BYTES / 16); }
    __device__ __forceinline__ unsigned j0(unsigned b) const { return blk(b) * 32u; }
};
// The scan kernel's row filter: none, the batch-wide row mask (3.6) or per-query selectors (3.7).
enum { DPH_FILT_NONE = 0, DPH_FILT_MASK = 1, DPH_FILT_QUERY = 2 };
template <int FK> struct ScanCursor { using T = SegCursor; };
template <> struct ScanCursor<DPH_FILT_MASK> { using T = SegCursorF; };
template <> struct ScanCursor<DPH_FILT_QUERY> { using T = SegCursorQ; };
__device__ __forceinline__ void cursor_seek(SegCursor& c, const DphSeg* tab, unsigned b, const uint8_t* codes, const ScanArgs&) { c.seek(tab, b, codes); }
__device__ __forceinline__ void cursor_seek(SegCursorF& c, const DphSeg* tab, unsigned b, const uint8_t* codes, const ScanArgs& a) { c.seek(tab, b, codes, a); }
__device__ __forceinline__ void cursor_seek(SegCursorQ& c, const DphSeg* tab, unsigned b, const uint8_t* codes, const ScanArgs& a) { c.seek(tab, b, codes, a); }
__device__ __forceinline__ unsigned cursor_mask(const SegCursor&, unsigned) { return ~0u; }
__device__ __forceinline__ unsigned cursor_mask(const SegCursorF& c, unsigned b) { return c.mrow[b]; }
__device__ __forceinline__ unsigned cursor_mask(const SegCursorQ& c, unsigned b) { return c.f >= 0 ? __ldg(c.qword + b) : ~0u; }
// Start of query q's range: only the per-query cursor depends on the query (its selector).
__device__ __forceinline__ void cursor_query(SegCursor&, const ScanArgs&, long long) {}
__device__ __forceinline__ void cursor_query(SegCursorQ& c, const ScanArgs& a, long long q) { c.f = a.qf->assign[q]; }

__device__ __forceinline__ void block_compact(ScanShared* sh, int keep, unsigned* gthr_q) {
    const int tid = threadIdx.x;
    const int n = sh->cnt;
    unsigned long long* cb = sh->cbuf;
    unsigned long long pivot = block_radix_select([&](int i) { return cb[i]; }, n, keep, &sh->sc);
    unsigned long long mine[DPH_CAND_CAP / NT];
#pragma unroll
    for (int e = 0; e < DPH_CAND_CAP / NT; e++) { int i = tid + e * NT; mine[e] = (i < n) ? cb[i] : 0ull; }
    __syncthreads();
    if (tid == 0) sh->cnt = 0;
    __syncthreads();
#pragma unroll
    for (int e = 0; e < DPH_CAND_CAP / NT; e++)
        if (mine[e] >= pivot && mine[e] != 0ull) { int p = atomicAdd(&sh->cnt, 1); cb[p] = mine[e]; }
    if (tid == 0) {
        unsigned t = (unsigned)(pivot >> 32);
        unsigned old = atomicMax(gthr_q, t);
        sh->thr = t > old ? t : old;
        sh->ndone_snap = sh->ndone;
    }
    __syncthreads();
}

// FK (DPH_FILT_*): with a filter, a row passes only when its mask bit is set; a block whose mask word is 0 is not prefetched, loaded
// or scored.  The per-query filter's work blocks are only the selected blocks, so its mask words are never 0.
template <int MODE, int FK>
__global__ void __launch_bounds__(NT, 1) scan_kernel(ScanArgs a) {
    constexpr bool FILT = FK != DPH_FILT_NONE;
    unsigned char* const smem = dph_smem;
    constexpr int LUT_BYTES = (MODE == DPH_SCAN_FAST) ? SMEM_LUT_FAST : SMEM_LUT_EXACT;
    ScanShared* sh = reinterpret_cast<ScanShared*>(smem + LUT_BYTES);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long T = a.work->total_blocks;
    const long long G = gridDim.x, c = blockIdx.x;
    const long long g0 = T * c / G, g1 = T * (c + 1) / G;
    if (g0 >= g1) return;
    long long lo = 0, hi = a.n;
    while (hi - lo > 1) { long long mid = (lo + hi) >> 1; if (a.qpre[mid] <= g0) lo = mid; else hi = mid; }
    long long q = lo, g = g0;
    const unsigned ywin = (((unsigned)__cvta_generic_to_shared(dph_smem)) & 0xFF000000u) | ((unsigned)lane * 4u);

    while (g < g1) {
        while (a.qpre[q + 1] <= g) q++;
        const long long qstart = a.qpre[q];
        const long long gend = (a.qpre[q + 1] < g1) ? a.qpre[q + 1] : g1;
        const unsigned b0 = (unsigned)(g - qstart), b1 = (unsigned)(gend - qstart);
        __syncthreads();
        {
            const int nsg0 = a.nseg[q];
            if (nsg0 <= DPH_SEG_SMEM) {
                const uint4* src = reinterpret_cast<const uint4*>(a.segs + q * a.nprobe);
                uint4* dst = reinterpret_cast<uint4*>(sh->segtab);
                for (int i = tid; i < nsg0 * 2; i += NT) dst[i] = __ldg(src + i);
            }
        }
        if (tid == 0) { sh->cnt = 0; sh->ndone = 0; sh->ndone_snap = 0; sh->thr = *((volatile unsigned*)(a.gthr + q)); }
        __syncthreads();

        // segment table of this query: shared memory when it fits (always for nprobe <= 256), else global
        const DphSeg* tab = (a.nseg[q] <= DPH_SEG_SMEM) ? sh->segtab : (a.segs + q * a.nprobe);
        typename ScanCursor<FK>::T cc, pc;                // consume / L2-prefetch cursors
        cc.init(); pc.init();
        cursor_query(cc, a, q); cursor_query(pc, a, q);
        unsigned b = b0 + warp;                           // next block this warp consumes
        unsigned bp = b0 + warp;                          // next block this warp prefetches into L2
        uint4 nxt[6];
        int n_len = 0; unsigned n_gstart = 0, n_j0 = 0; float n_dis0 = 0.f;
        // the first code blocks are requested BEFORE the LUT is staged: their HBM latency overlaps the staging
#pragma unroll 1
        for (int r = 0; r < DPH_L2_PREFETCH_ROUNDS && bp < b1; r++, bp += NW) {
            cursor_seek(pc, tab, bp, a.codes, a);
            if (lane == 0 && (!FILT || cursor_mask(pc, bp))) l2_prefetch_block(pc.ptr(bp));
        }
        bool more = b < b1;
        unsigned n_mask = ~0u;                            // FILT: the mask word of the block in nxt
        if (more) {
            cursor_seek(cc, tab, b, a.codes, a);
            if (FILT) n_mask = cursor_mask(cc, b);
            if (!FILT || n_mask) {
                const uint4* p = cc.ptr(b) + lane;
#pragma unroll
                for (int c6 = 0; c6 < 6; c6++) nxt[c6] = ldg_stream(p + c6 * 32);
            }
            n_len = cc.len; n_gstart = cc.gstart; n_dis0 = cc.dis0; n_j0 = cc.j0(b);
        }
        // ---- stage this query's LUT into shared memory (twelve 16-byte loads in flight per thread) ----
        {
            const float4* src = reinterpret_cast<const float4*>(a.lut_canon + (size_t)q * DPH_LUT_CANON_FLOATS);
            constexpr int PER_T = DPH_LUT_CANON_FLOATS / 4 / NT;      // 12
            constexpr int LB = 12;
            static_assert(PER_T % LB == 0, "LUT staging batches");
            if (MODE == DPH_SCAN_FAST) {
                // canonical rows [seg][code][32] -> scan rows [seg][code][64]: words 0..31 = the row, words 32..62 = its first 31
                // entries again (the wrap copies that let lane l read word l + t without a modulo), word 63 unused.  One thread
                // moves one float4; a quarter-warp writes 128 contiguous bytes of one row -> conflict-free.
                float* dstf = reinterpret_cast<float*>(smem);
#pragma unroll 1
                for (int i0 = tid; i0 < DPH_LUT_CANON_FLOATS / 4; i0 += NT * LB) {
                    float4 v[LB];
#pragma unroll
                    for (int e = 0; e < LB; e++) v[e] = __ldg(src + i0 + e * NT);
#pragma unroll
                    for (int e = 0; e < LB; e++) {
                        const int i = i0 + e * NT;
                        const int row = i >> 3, w = (i & 7) * 4;              // row = seg * 256 + code
                        float* r = dstf + row * 64;
                        *reinterpret_cast<float4*>(r + w) = v[e];
                        if (w < 28) *reinterpret_cast<float4*>(r + 32 + w) = v[e];
                        else { r[60] = v[e].x; r[61] = v[e].y; r[62] = v[e].z; r[63] = 0.0f; }
                    }
                }
            } else {
                float4* dst = reinterpret_cast<float4*>(smem);
#pragma unroll 8
                for (int i = tid; i < DPH_LUT_CANON_FLOATS / 4; i += NT) dst[i] = __ldg(src + i);
            }
        }
        __syncthreads();
        bool counted = false;
        while (true) {      // epochs: run until the candidate buffer may overflow or this warp is out of blocks, then meet
            while (more) {
                if (*((volatile int*)&sh->cnt) > DPH_CAND_CAP - NT) break;     // every warp adds <= 32 per round after this check
                uint4 cur[6];
#pragma unroll
                for (int c6 = 0; c6 < 6; c6++) cur[c6] = nxt[c6];
                const int c_len = n_len; const unsigned c_gstart = n_gstart, c_j0 = n_j0; const float c_dis0 = n_dis0;
                const unsigned c_mask = n_mask;
                if (bp < b1) {
                    cursor_seek(pc, tab, bp, a.codes, a);
                    if (lane == 0 && (!FILT || cursor_mask(pc, bp))) l2_prefetch_block(pc.ptr(bp));
                    bp += NW;
                }
                b += NW;
                more = b < b1;
                if (more) {
                    cursor_seek(cc, tab, b, a.codes, a);
                    if (FILT) n_mask = cursor_mask(cc, b);
                    if (!FILT || n_mask) {
                        const uint4* p = cc.ptr(b) + lane;
#pragma unroll
                        for (int c6 = 0; c6 < 6; c6++) nxt[c6] = ldg_stream(p + c6 * 32);
                    }
                    n_len = cc.len; n_gstart = cc.gstart; n_dis0 = cc.dis0; n_j0 = cc.j0(b);
                }
                if (FILT && c_mask == 0) continue;                 // warp-uniform: no row of the block is selected
                float score;
                if (MODE == DPH_SCAN_FAST) {
                    float2 a01 = make_float2(c_dis0, 0.f), a23 = make_float2(0.f, 0.f);
                    fast_chunk<0>(cur[0], ywin, a01, a23);
                    fast_chunk<1>(cur[1], ywin, a01, a23);
                    fast_chunk<2>(cur[2], ywin, a01, a23);
                    fast_chunk<3>(cur[3], ywin, a01, a23);
                    fast_chunk<4>(cur[4], ywin, a01, a23);
                    fast_chunk<5>(cur[5], ywin, a01, a23);
                    score = (a01.x + a01.y) + (a23.x + a23.y);
                } else {
                    unsigned char* stage = smem + DPH_LUT_CANON_FLOATS * 4 + warp * DPH_BLK_BYTES;
                    const float* lutc = reinterpret_cast<const float*>(smem);
#pragma unroll
                    for (int c6 = 0; c6 < 6; c6++) *reinterpret_cast<uint4*>(stage + c6 * 512 + lane * 16) = cur[c6];
                    __syncwarp();
                    float dis = c_dis0;
#pragma unroll 8
                    for (int m = 0; m < DPH_M; m++) dis += lutc[DPH_LUTC_IDX(m, (int)stage[dph_blk_addr(lane, m)])];
                    score = dis;
                    __syncwarp();
                }
                const unsigned j = c_j0 + lane;
                const unsigned sk = dph_fkey(score);
                const bool pass = ((int)j < c_len) && (!FILT || ((c_mask >> lane) & 1u)) && (sk >= *((volatile unsigned*)&sh->thr));
                const unsigned pm = __ballot_sync(0xffffffffu, pass);
                if (pm) {
                    int basep = 0;
                    if (lane == 0) basep = atomicAdd(&sh->cnt, __popc(pm));
                    basep = __shfl_sync(0xffffffffu, basep, 0);
                    if (pass) {
                        int p = basep + __popc(pm & ((1u << lane) - 1u));
                        if (p < DPH_CAND_CAP) sh->cbuf[p] = ((unsigned long long)sk << 32) | (unsigned long long)(0xFFFFFFFFu - (c_gstart + j));
                    }
                }
            }
            if (!more && !counted) { counted = true; if (lane == 0) atomicAdd(&sh->ndone, 1); }
            __syncthreads();
            if (sh->cnt > a.keep) block_compact(sh, a.keep, a.gthr + q);
            else {
                if (tid == 0) {
                    unsigned gt = *((volatile unsigned*)(a.gthr + q));
                    if (gt > sh->thr) sh->thr = gt;
                    sh->ndone_snap = sh->ndone;
                }
                __syncthreads();
            }
            if (sh->ndone_snap == NW) break;
        }
        // ---- publish this CTA's candidates for query q ----
        __syncthreads();
        const int cnt = sh->cnt;
        if (tid == 0) sh->base = atomicAdd(a.cand_cnt + q, cnt);
        __syncthreads();
        {
            const long long off = a.cand_off[q], cap = a.cand_off[q + 1] - off;
            const int basep = sh->base;
            for (int i = tid; i < cnt; i += NT)
                if (basep + i < cap) a.cand[off + basep + i] = sh->cbuf[i];
        }
        g = gend;
        q++;
    }
}

// =================================================================================================
// PAIR mode: when a list is probed by several queries of the batch (C2: 64 x 256 probes over 4096 lists = 4 per list),
// two of them share every gather: their LUTs are quantised to 10-bit integers (plan: lutq_kernel) and packed into one
// 32-bit word (query a in the low half, query b in the high half), so ONE PRMT + LDS + IADD advances both running sums
// (96 x 682 < 2^16: the halves cannot carry into each other).  Per (query, byte) that halves the code bytes read from HBM,
// the shared-memory gathers and the instructions.  The integer sums are exact; the only error is the quantisation
// (<= 0.5 step per entry), which the plan folds into eps, so the same proof + exact canonical re-scoring applies.
// Work: the plan inverts probes into per-list query groups and pairs them; an item = (list, query pair), linearised by
// blocks; a CTA takes a contiguous block range, rebuilding the packed LUT (192 KB, from L2) at every item boundary.
// =================================================================================================
struct GroupScanArgs {     // both grouped kernels (scan_pair_kernel, scan_quad_kernel)
    const uint8_t* codes; const long long* blk_off; const int* list_len;
    const int* grp_cnt; const int* grp_off; const unsigned long long* units; const unsigned* entries; const DphGroupWork* work; int* next_unit;
    const unsigned short* lutq; const float2* qparams; const float* cd; const unsigned* gdense;
    unsigned* gthr; unsigned long long* cand; const long long* cand_off; int* cand_cnt;
    long long list_lo, list_hi; int nprobe; int keep;
    const DphUnit* udesc;          // quad mode: resolved unit records (plan)
    unsigned one;                  // the constant 1, as a run-time value (imad_add)
    const unsigned* mask; const long long* mask_off;     // filtered variants: the row mask, and the shard's first block of each list
};
#define PCAP 1536                  // PCAP - NT = DPH_PAIR_KEEP_MAX (each warp adds <= 32 per buffer after the latch is polled)
static_assert(PCAP - NT == DPH_PAIR_KEEP_MAX, "pair latch margin");
struct PairShared {
    unsigned long long cbuf[2][PCAP];
    SelectScratch sc;
    int cnt[2]; unsigned thr[2]; int base[2]; int ndone; int ndone_snap; int unit;
};
template <int IMM> __device__ __forceinline__ unsigned lds_imm_u32(unsigned addr) {
    unsigned v;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(IMM));
    return v;
}
template <int T0> __device__ __forceinline__ void pair_word(unsigned wv, unsigned y, unsigned& a0, unsigned& a1, unsigned& a2, unsigned& a3) {
    constexpr int TB = DPH_DYN_SMEM_BASE + (T0 >> 5) * 65536 + (T0 & 31) * 4;
    a0 += lds_imm_u32<TB + 0>(__byte_perm(wv, y, 0x7504));
    a1 += lds_imm_u32<TB + 4>(__byte_perm(wv, y, 0x7514));
    a2 += lds_imm_u32<TB + 8>(__byte_perm(wv, y, 0x7524));
    a3 += lds_imm_u32<TB + 12>(__byte_perm(wv, y, 0x7534));
}
template <int C> __device__ __forceinline__ void pair_chunk(const uint4& v, unsigned y, unsigned& a0, unsigned& a1, unsigned& a2, unsigned& a3) {
    pair_word<C * 16 + 0>(v.x, y, a0, a1, a2, a3);
    pair_word<C * 16 + 4>(v.y, y, a0, a1, a2, a3);
    pair_word<C * 16 + 8>(v.z, y, a0, a1, a2, a3);
    pair_word<C * 16 + 12>(v.w, y, a0, a1, a2, a3);
}
template <int CAP, int NTH>     // NTH: the block's thread count
__device__ __forceinline__ void compact_buffer(unsigned long long* cb, int* cnt, unsigned* thr, int keep, unsigned* gthr_q, SelectScratch* sc) {
    const int tid = threadIdx.x;
    const int n = *cnt;
    unsigned long long pivot = block_radix_select([&](int i) { return cb[i]; }, n, keep, sc);
    constexpr int PER = (CAP + NTH - 1) / NTH;
    unsigned long long mine[PER];
#pragma unroll
    for (int e = 0; e < PER; e++) { int i = tid + e * NTH; mine[e] = (i < n) ? cb[i] : 0ull; }
    __syncthreads();
    if (tid == 0) *cnt = 0;
    __syncthreads();
#pragma unroll
    for (int e = 0; e < PER; e++)
        if (mine[e] >= pivot && mine[e] != 0ull) { int p = atomicAdd(cnt, 1); cb[p] = mine[e]; }
    if (tid == 0) {
        unsigned t = (unsigned)(pivot >> 32);
        unsigned old = atomicMax(gthr_q, t);
        *thr = t > old ? t : old;
    }
    __syncthreads();
}
__device__ __forceinline__ void warp_append(bool pass, unsigned long long key, unsigned long long* cb, int* cnt, int cap, int lane) {
    const unsigned pm = __ballot_sync(0xffffffffu, pass);
    if (pm) {
        int basep = 0;
        if (lane == 0) basep = atomicAdd(cnt, __popc(pm));
        basep = __shfl_sync(0xffffffffu, basep, 0);
        if (pass) { int p = basep + __popc(pm & ((1u << lane) - 1u)); if (p < cap) cb[p] = key; }
    }
}

template <bool FILT>
__global__ void __launch_bounds__(NT, 1) scan_pair_kernel(GroupScanArgs a) {
    unsigned char* const smem = dph_smem;
    PairShared* sh = reinterpret_cast<PairShared*>(smem + SMEM_LUT_FAST);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int total_units = a.work->total_units;
    const unsigned segb = (unsigned)a.work->per;
    const unsigned ywin = (((unsigned)__cvta_generic_to_shared(dph_smem)) & 0xFF000000u) | ((unsigned)lane * 4u);

    while (true) {
        // pull the next unit of the queue: consecutive units are the items of one list segment, so they run at the same time on
        // different CTAs and share the segment's code blocks through L2
        if (tid == 0) sh->unit = atomicAdd(a.next_unit, 1);
        __syncthreads();
        const int u = sh->unit;
        if (u >= total_units) break;
        const unsigned long long ud = a.units[u];
        const long long l = (long long)(ud & 0xFFFFFFFFull);
        const int it = (int)((ud >> 32) & 0xFFFFull);
        const int len = a.list_len[l];
        const unsigned nb = (unsigned)((len + 31) >> 5);
        const unsigned bi0 = (unsigned)(ud >> 48) * segb;
        const unsigned bend = (nb - bi0 < segb) ? nb : bi0 + segb;
        const int e0 = a.grp_off[l] + 2 * it;
        const bool has_b = (2 * it + 1) < a.grp_cnt[l];
        const unsigned ea = a.entries[e0], eb = has_b ? a.entries[e0 + 1] : ea;
        const long long qa = ea >> 10, qb = eb >> 10;
        const int ra = (int)(ea & 1023u), rb = (int)(eb & 1023u);
        __syncthreads();
        {   // ---- packed LUT: word = qa entry | qb entry << 16, same [3][256][64] scan layout ----
            const uint4* A4 = reinterpret_cast<const uint4*>(a.lutq + (size_t)qa * DPH_LUT_SCAN_FLOATS);
            const uint4* B4 = reinterpret_cast<const uint4*>(a.lutq + (size_t)qb * DPH_LUT_SCAN_FLOATS);
            uint4* dst = reinterpret_cast<uint4*>(smem);
            for (int i = tid; i < DPH_LUT_SCAN_FLOATS / 8; i += NT) {
                const uint4 va = __ldg(A4 + i);
                uint4 vb = make_uint4(0u, 0u, 0u, 0u);
                if (has_b) vb = __ldg(B4 + i);
                uint4 o0, o1;
                o0.x = (va.x & 0xFFFFu) | (vb.x << 16); o0.y = (va.x >> 16) | (vb.x & 0xFFFF0000u);
                o0.z = (va.y & 0xFFFFu) | (vb.y << 16); o0.w = (va.y >> 16) | (vb.y & 0xFFFF0000u);
                o1.x = (va.z & 0xFFFFu) | (vb.z << 16); o1.y = (va.z >> 16) | (vb.z & 0xFFFF0000u);
                o1.z = (va.w & 0xFFFFu) | (vb.w << 16); o1.w = (va.w >> 16) | (vb.w & 0xFFFF0000u);
                dst[2 * i] = o0; dst[2 * i + 1] = o1;
            }
        }
        if (tid == 0) {
            sh->cnt[0] = 0; sh->cnt[1] = 0; sh->ndone = 0; sh->ndone_snap = 0;
            sh->thr[0] = *((volatile unsigned*)(a.gthr + qa));
            sh->thr[1] = has_b ? *((volatile unsigned*)(a.gthr + qb)) : 0xFFFFFFFFu;
        }
        __syncthreads();
        const float2 pa = a.qparams[qa], pb = a.qparams[qb];
        const float base_a = a.cd[qa * a.nprobe + ra] + pa.y, base_b = a.cd[qb * a.nprobe + rb] + pb.y;
        const unsigned gs_a = a.gdense[qa * a.nprobe + ra], gs_b = a.gdense[qb * a.nprobe + rb];
        const uint4* lbase = reinterpret_cast<const uint4*>(a.codes + a.blk_off[l] * DPH_BLK_BYTES);
        const unsigned* mrow = FILT ? a.mask + a.mask_off[l] : nullptr;      // FILT: mask word of the list's block b = mrow[b]

        unsigned b = bi0 + warp, bp = bi0 + warp;
        uint4 nxt[6];
#pragma unroll 1
        for (int r = 0; r < DPH_L2_PREFETCH_ROUNDS && bp < bend; r++, bp += NW)
            if (lane == 0 && (!FILT || mrow[bp])) l2_prefetch_block(lbase + (size_t)bp * (DPH_BLK_BYTES / 16));
        bool more = b < bend;
        unsigned n_mask = ~0u;
        if (more) {
            if (FILT) n_mask = mrow[b];
            if (!FILT || n_mask) {
                const uint4* p = lbase + (size_t)b * (DPH_BLK_BYTES / 16) + lane;
#pragma unroll
                for (int c6 = 0; c6 < 6; c6++) nxt[c6] = ldg_stream(p + c6 * 32);
            }
        }
        bool counted = false;
        while (true) {
            while (more) {
                if (*((volatile int*)&sh->cnt[0]) > PCAP - NT || *((volatile int*)&sh->cnt[1]) > PCAP - NT) break;
                uint4 cur[6];
#pragma unroll
                for (int c6 = 0; c6 < 6; c6++) cur[c6] = nxt[c6];
                const unsigned bcur = b, c_mask = n_mask;
                if (bp < bend) { if (lane == 0 && (!FILT || mrow[bp])) l2_prefetch_block(lbase + (size_t)bp * (DPH_BLK_BYTES / 16)); bp += NW; }
                b += NW;
                more = b < bend;
                if (more) {
                    if (FILT) n_mask = mrow[b];
                    if (!FILT || n_mask) {
                        const uint4* p = lbase + (size_t)b * (DPH_BLK_BYTES / 16) + lane;
#pragma unroll
                        for (int c6 = 0; c6 < 6; c6++) nxt[c6] = ldg_stream(p + c6 * 32);
                    }
                }
                if (FILT && c_mask == 0) continue;                 // warp-uniform: no row of the block is selected
                unsigned s0 = 0, s1 = 0, s2 = 0, s3 = 0;
                pair_chunk<0>(cur[0], ywin, s0, s1, s2, s3);
                pair_chunk<1>(cur[1], ywin, s0, s1, s2, s3);
                pair_chunk<2>(cur[2], ywin, s0, s1, s2, s3);
                pair_chunk<3>(cur[3], ywin, s0, s1, s2, s3);
                pair_chunk<4>(cur[4], ywin, s0, s1, s2, s3);
                pair_chunk<5>(cur[5], ywin, s0, s1, s2, s3);
                const unsigned tot = (s0 + s1) + (s2 + s3);
                const float sc_a = fmaf(pa.x, (float)(tot & 0xFFFFu), base_a);
                const float sc_b = fmaf(pb.x, (float)(tot >> 16), base_b);
                const unsigned j = bcur * 32u + lane;
                const bool valid = (int)j < len && (!FILT || ((c_mask >> lane) & 1u));
                const unsigned ka = dph_fkey(sc_a), kb = dph_fkey(sc_b);
                warp_append(valid && ka >= *((volatile unsigned*)&sh->thr[0]), ((unsigned long long)ka << 32) | (unsigned long long)(0xFFFFFFFFu - (gs_a + j)),
                            sh->cbuf[0], &sh->cnt[0], PCAP, lane);
                warp_append(valid && kb >= *((volatile unsigned*)&sh->thr[1]), ((unsigned long long)kb << 32) | (unsigned long long)(0xFFFFFFFFu - (gs_b + j)),
                            sh->cbuf[1], &sh->cnt[1], PCAP, lane);
            }
            if (!more && !counted) { counted = true; if (lane == 0) atomicAdd(&sh->ndone, 1); }
            __syncthreads();
            if (sh->cnt[0] > a.keep) compact_buffer<PCAP, NT>(sh->cbuf[0], &sh->cnt[0], &sh->thr[0], a.keep, a.gthr + qa, &sh->sc);
            if (sh->cnt[1] > a.keep) compact_buffer<PCAP, NT>(sh->cbuf[1], &sh->cnt[1], &sh->thr[1], a.keep, a.gthr + qb, &sh->sc);
            if (tid == 0) {
                unsigned ga = *((volatile unsigned*)(a.gthr + qa));
                if (ga > sh->thr[0]) sh->thr[0] = ga;
                if (has_b) { unsigned gb = *((volatile unsigned*)(a.gthr + qb)); if (gb > sh->thr[1]) sh->thr[1] = gb; }
                sh->ndone_snap = sh->ndone;
            }
            __syncthreads();
            if (sh->ndone_snap == NW) break;
        }
        // ---- publish both candidate sets ----
        for (int s2i = 0; s2i < (has_b ? 2 : 1); s2i++) {
            const long long q = s2i ? qb : qa;
            const int cnt = sh->cnt[s2i];
            if (tid == 0) sh->base[s2i] = atomicAdd(a.cand_cnt + q, cnt);
            __syncthreads();
            const long long off = a.cand_off[q], cap = a.cand_off[q + 1] - off;
            const int basep = sh->base[s2i];
            for (int i = tid; i < cnt; i += NT)
                if (basep + i < cap) a.cand[off + basep + i] = sh->cbuf[s2i][i];
        }
    }
}


// =================================================================================================
// QUAD mode: FOUR queries that probe the same list share every gather.  Their LUTs are quantised to 8-bit integers
// (plan: lutq_kernel<unsigned char, 255>) and packed into one 32-bit word (query i in byte i), so one PRMT + LDS serves
// four (query, code byte) lookups -- the shared-memory gather pipe, which bounds the pair kernel, does half the work per
// lookup.  The byte lanes would overflow after two additions, so the running sums are kept as TWO 32-bit registers:
//     sraw  = sum of the gathered words, plain 32-bit wrap-around arithmetic
//           = S0 + 2^8 S1 + 2^16 S2 + 2^24 S3   (mod 2^32),        S_i = sum of query i's entries  (<= 96 * 255 < 2^15)
//     accb  = sum of PRMT(word -> [b1, 0, b3, 0]) = S1 + 2^16 S3     (exact: both lanes stay below 2^16)
// and decoded once per vector:  sraw - (accb << 8) = S0 + 2^16 S2 (exact, < 2^32).
// The integer sums are exact; the only error is the quantisation (<= 0.5 step per entry), which the plan folds into eps, so the
// same proof + exact canonical re-scoring applies (merge_kernel).
//
// Work items are (list segment, group of <= 8 probing queries): every code block is read from HBM once into registers and run
// through one packed table (queries 0-3) or two (queries 4-7 as well), so a list probed by up to 8 queries of the batch is read
// once, by one CTA.  Two tables fit in shared memory because the table is WRAP-FREE: a row holds only the 32 real words, and the
// lane rotation lives in the address instead -- at step t lane l reads word (l + t) & 31, whose byte offset comes from per-lane
// registers (11 registers of three offsets and a zero byte; the dynamic window's top address byte is 0, checked at setup).  One
// PRMT still builds the address (rotated offset | code << 8) and serves both tables; the table, segment and half-row go in the
// LDS immediate.  Rows stay 256 bytes: three 64 KB regions, region r row c = two 128-byte halves:
//     region 0: [table 0 segment 0 | table 0 segment 1]   region 1: [table 1 segment 0 | table 1 segment 1]
//     region 2: [table 0 segment 2 | table 1 segment 2]
// A lane's bank is still (l + t) mod 32, so the gathers stay conflict-free.
// =================================================================================================
#define QNT 256                    // quad kernel threads: eight candidate buffers must fit next to the two 96 KB tables
#define QNW (QNT / 32)
#define QCAP 512                   // QCAP - QNT = DPH_QUAD_KEEP_MAX (each warp adds <= 32 per buffer after the latch is polled)
#define SMEM_QUAD_TABLES (3 * 65536)
static_assert(QCAP - QNT == DPH_QUAD_KEEP_MAX, "quad latch margin");
static_assert(offsetof(DphUnit, bend) < 32, "the run-out prefetch reads the block range from the record's first 32 bytes");
struct QuadShared {
    unsigned long long cbuf[DPH_QUAD_ITEM_Q][QCAP];
    SelectScratch sc;
    DphUnit desc[2];                 // current item / next item (fetched with cp.async while the current one is scanned)
    uint4 head[QNW][2];              // per warp: the first 32 bytes of the next item's record (its block range), for the run-out prefetch
    int cnt[DPH_QUAD_ITEM_Q]; unsigned thr[DPH_QUAD_ITEM_Q]; int base[DPH_QUAD_ITEM_Q]; int ndone; int ndone_snap; int unit; int full;
    long long qs[DPH_QUAD_ITEM_Q];   // the group's queries (shared copy: indexed by thread id in the publish step)
};
// 32-bit add on the FMA pipe: d = a * one + c with `one` a kernel parameter holding 1 (opaque to ptxas, so the multiply-add is not
// folded back into an IADD3).  The quad scan's gathers are bound by the ALU pipe (PRMT + IADD3, one warp instruction per two cycles
// per sub-partition); IMAD issues on the otherwise idle FMA pipe at the same rate.
__device__ __forceinline__ unsigned imad_add(unsigned x, unsigned one, unsigned c) {
    unsigned d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(x), "r"(one), "r"(c));
    return d;
}
// Four gathers of one table (code bytes T0..T0+3 of a segment, addresses built by quad_word) into that table's sums.
// The raw sums are added on the FMA pipe (imad_add), the odd-byte sums by IADD3.  Moving the odd-byte sums to the FMA pipe as well
// (half or all of them) makes the issue slots the limit instead (DESIGN.md 4.1).
template <int T0, int TAB> __device__ __forceinline__ void quad_gather(const unsigned (&ad)[4], unsigned one, unsigned (&sr)[4], unsigned (&ab)[4]) {
    constexpr int S = T0 >> 5;
    constexpr int TB = DPH_DYN_SMEM_BASE + (S < 2 ? TAB : 2) * 65536 + (S < 2 ? S : TAB) * 128;
    constexpr int A = (T0 >> 2) & 1;                  // two accumulator sets, alternating per code word
    const unsigned w0 = lds_imm_u32<TB>(ad[0]);
    const unsigned w1 = lds_imm_u32<TB>(ad[1]);
    const unsigned w2 = lds_imm_u32<TB>(ad[2]);
    const unsigned w3 = lds_imm_u32<TB>(ad[3]);
    // 8-bit entries: the odd bytes are widened per gather (a lane-wise add of two words could carry).  A 7-bit variant that widens
    // once per TWO gathers is faster but doubles eps, and then the exactness proof fails for ~10 % of the queries at C2 (measured
    // on B200); the exact fallback costs far more than it saves.
    sr[2 * A] = imad_add(w1, one, imad_add(w0, one, sr[2 * A]));
    sr[2 * A + 1] = imad_add(w3, one, imad_add(w2, one, sr[2 * A + 1]));
    const unsigned e0 = __byte_perm(w0, 0u, 0x4341), e1 = __byte_perm(w1, 0u, 0x4341);
    const unsigned e2 = __byte_perm(w2, 0u, 0x4341), e3 = __byte_perm(w3, 0u, 0x4341);
    ab[2 * A] += e0 + e1;
    ab[2 * A + 1] += e2 + e3;
}
// Byte b of rot[r] = ((lane + 3r + b) & 31) * 4, the rotated word offset of step t = 3r + b of a segment; byte 3 is zero.
// Selector of code byte i at step t: [rotated offset of t, code byte i, 0, 0].
template <int T> struct RotSel { static constexpr int reg = (T & 31) / 3, sel = 0x7700 | (4 + (T & 31) % 3); };
template <int T0, int NTAB> __device__ __forceinline__ void quad_word(unsigned wv, const unsigned (&rot)[11], unsigned one,
                                                                        unsigned (&sr)[2][4], unsigned (&ab)[2][4]) {
    const unsigned ad[4] = {__byte_perm(wv, rot[RotSel<T0>::reg], RotSel<T0>::sel | 0x00),
                            __byte_perm(wv, rot[RotSel<T0 + 1>::reg], RotSel<T0 + 1>::sel | 0x10),
                            __byte_perm(wv, rot[RotSel<T0 + 2>::reg], RotSel<T0 + 2>::sel | 0x20),
                            __byte_perm(wv, rot[RotSel<T0 + 3>::reg], RotSel<T0 + 3>::sel | 0x30)};
    quad_gather<T0, 0>(ad, one, sr[0], ab[0]);
    if (NTAB == 2) quad_gather<T0, 1>(ad, one, sr[1], ab[1]);
}
template <int C, int NTAB> __device__ __forceinline__ void quad_chunk(const uint4& v, const unsigned (&rot)[11], unsigned one,
                                                                         unsigned (&sr)[2][4], unsigned (&ab)[2][4]) {
    quad_word<C * 16 + 0, NTAB>(v.x, rot, one, sr, ab);
    quad_word<C * 16 + 4, NTAB>(v.y, rot, one, sr, ab);
    quad_word<C * 16 + 8, NTAB>(v.z, rot, one, sr, ab);
    quad_word<C * 16 + 12, NTAB>(v.w, rot, one, sr, ab);
}
// append with an overflow latch: the round loop polls ONE flag instead of every buffer's counter
__device__ __forceinline__ void warp_append_latch(bool pass, unsigned long long key, unsigned long long* cb, int* cnt, int* full, int lane) {
    const unsigned pm = __ballot_sync(0xffffffffu, pass);
    if (pm) {
        int basep = 0;
        const int np = __popc(pm);
        if (lane == 0) { basep = atomicAdd(cnt, np); if (basep + np > QCAP - QNT) *((volatile int*)full) = 1; }
        basep = __shfl_sync(0xffffffffu, basep, 0);
        if (pass) { int p = basep + __popc(pm & ((1u << lane) - 1u)); if (p < QCAP) cb[p] = key; }
    }
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
// float image of a threshold (0xFFFFFFFF = "never passes" for the empty slots of a short group -> +inf)
__device__ __forceinline__ float quad_thr_f(unsigned t) {
    return t == 0xFFFFFFFFu ? __int_as_float(0x7f800000) : (t == 0u ? -__int_as_float(0x7f800000) : dph_fkey_inv(t));
}

#ifdef DPH_SCAN_PHASES
// Per-CTA %globaltimer phase totals of thread 0 (build -DDPH_SCAN_PHASES): packed-table build, scan rounds (to the epoch barrier),
// compaction barriers, candidate publish; summed over the CTAs of a launch and printed by the last CTA to finish.
__device__ unsigned long long g_quad_phase_ns[4];
__device__ unsigned g_quad_phase_ctas;
__device__ __forceinline__ unsigned long long globaltimer_ns() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define QPH_MARK(i) do { if (threadIdx.x == 0) { const unsigned long long t_ = globaltimer_ns(); ph[i] += t_ - ph_t; ph_t = t_; } } while (0)
#else
#define QPH_MARK(i) do { } while (0)
#endif

// A warp that runs out of blocks starts the next item's stream: it waits for its copy of the next record's head (requested with
// cp.async after this item's table build; warp 0 also waits for the whole record here) and issues the L2 prefetch of its first
// DPH_L2_PREFETCH_ROUNDS blocks of the next item, so HBM keeps streaming while the other warps finish, compact and publish.
template <bool FILT>
__device__ __forceinline__ void quad_prefetch_next(const GroupScanArgs& a, const QuadShared* sh, int total_units, unsigned long long pol) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    asm volatile("cp.async.wait_all;" ::: "memory");
    if (lane == 0 && sh->unit < total_units) {
        const DphUnit* nd = reinterpret_cast<const DphUnit*>(sh->head[warp]);
        const uint4* lb = reinterpret_cast<const uint4*>(a.codes + nd->blk * DPH_BLK_BYTES);
        const unsigned bend = nd->bend;
        const unsigned* mrow = FILT ? a.mask + a.mask_off[nd->list] : nullptr;
        unsigned bp = nd->bi0 + warp;
#pragma unroll 1
        for (int r = 0; r < DPH_L2_PREFETCH_ROUNDS && bp < bend; r++, bp += QNW)
            if (!FILT || mrow[bp]) l2_prefetch_block(lb + (size_t)bp * (DPH_BLK_BYTES / 16), pol);
    }
}

// The scan of one item over its block range with NTAB packed tables: rounds until a candidate buffer may overflow or the warp is out
// of blocks, then a barrier, the compaction of the buffers over keep and the refresh of the thresholds; until every warp is done.
// The code stream is loaded with the evict_first policy `pol`: each block is read once per batch.
// FILT: nmask is the mask word of the block in nxt (in and out), mrow[b] the mask word of the item's list's block b.
template <int NTAB, bool FILT>
__device__ __forceinline__ void quad_item_rounds(const GroupScanArgs& a, QuadShared* sh, const DphUnit* dsc, const uint4* lbase, unsigned b,
                                                 unsigned bp, uint4 (&nxt)[6], const unsigned (&rot)[11], unsigned one, int total_units,
                                                 unsigned long long pol, unsigned long long* ph, unsigned long long& ph_t, unsigned& nmask,
                                                 const unsigned* mrow) {
    (void)ph; (void)ph_t;
    const int lane = threadIdx.x & 31;
    const int len = dsc->len, nq = dsc->nq;
    const unsigned bend = dsc->bend;
    constexpr int NS = 4 * NTAB;
    unsigned gsv[NS]; float stepv[NS], basev[NS], tf[NS]; unsigned thr[NS];
#pragma unroll
    for (int i = 0; i < NS; i++) { gsv[i] = dsc->gs[i]; basev[i] = dsc->base[i]; stepv[i] = dsc->step[i]; thr[i] = sh->thr[i]; tf[i] = quad_thr_f(thr[i]); }
    bool more = b < bend, counted = false;
    while (true) {
        while (more) {
            if (*((volatile int*)&sh->full)) break;
            uint4 cur6[6];
#pragma unroll
            for (int c6 = 0; c6 < 6; c6++) cur6[c6] = nxt[c6];
            const unsigned bcur = b, cmask = nmask;
            if (bp < bend) { if (lane == 0 && (!FILT || mrow[bp])) l2_prefetch_block(lbase + (size_t)bp * (DPH_BLK_BYTES / 16), pol); bp += QNW; }
            b += QNW;
            more = b < bend;
            if (more) {
                if (FILT) nmask = mrow[b];
                if (!FILT || nmask) {
                    const uint4* p = lbase + (size_t)b * (DPH_BLK_BYTES / 16) + lane;
#pragma unroll
                    for (int c6 = 0; c6 < 6; c6++) nxt[c6] = ldg_stream(p + c6 * 32, pol);
                }
            }
            if (FILT && cmask == 0) continue;                      // warp-uniform: no row of the block is selected
            unsigned sr[2][4] = {}, ab[2][4] = {};
            quad_chunk<0, NTAB>(cur6[0], rot, one, sr, ab);
            quad_chunk<1, NTAB>(cur6[1], rot, one, sr, ab);
            quad_chunk<2, NTAB>(cur6[2], rot, one, sr, ab);
            quad_chunk<3, NTAB>(cur6[3], rot, one, sr, ab);
            quad_chunk<4, NTAB>(cur6[4], rot, one, sr, ab);
            quad_chunk<5, NTAB>(cur6[5], rot, one, sr, ab);
            const unsigned j = bcur * 32u + lane;
            const bool valid = (int)j < len && (!FILT || ((cmask >> lane) & 1u));
            // thresholds are compared in the float domain (one FSETP per query); the order-preserving integer key is built only for
            // the rare vector that passes.  (float)(unsigned short) converts a 16-bit half of the register without a mask / shift.
            float f[NS]; bool p[NS]; bool any = false;
#pragma unroll
            for (int tb = 0; tb < NTAB; tb++) {
                const unsigned SR = (sr[tb][0] + sr[tb][1]) + (sr[tb][2] + sr[tb][3]);
                const unsigned AB = (ab[tb][0] + ab[tb][1]) + (ab[tb][2] + ab[tb][3]);      // S1 | S3 << 16
                const unsigned AE = SR - (AB << 8);                                         // S0 | S2 << 16
                f[4 * tb + 0] = fmaf(stepv[4 * tb + 0], (float)(unsigned short)(AE), basev[4 * tb + 0]);
                f[4 * tb + 1] = fmaf(stepv[4 * tb + 1], (float)(unsigned short)(AB), basev[4 * tb + 1]);
                f[4 * tb + 2] = fmaf(stepv[4 * tb + 2], (float)(unsigned short)(AE >> 16), basev[4 * tb + 2]);
                f[4 * tb + 3] = fmaf(stepv[4 * tb + 3], (float)(unsigned short)(AB >> 16), basev[4 * tb + 3]);
            }
#pragma unroll
            for (int i = 0; i < NS; i++) { p[i] = valid && f[i] >= tf[i]; any = any || p[i]; }
            if (__any_sync(0xffffffffu, any)) {
#pragma unroll
                for (int i = 0; i < NS; i++) {
                    const unsigned k = dph_fkey(f[i]);
                    warp_append_latch(p[i] && k >= thr[i], ((unsigned long long)k << 32) | (unsigned long long)(0xFFFFFFFFu - (gsv[i] + j)),
                                      sh->cbuf[i], &sh->cnt[i], &sh->full, lane);
                }
            }
        }
        if (!more && !counted) {
            counted = true;
            quad_prefetch_next<FILT>(a, sh, total_units, pol);
            if (lane == 0) atomicAdd(&sh->ndone, 1);
        }
        __syncthreads();
        QPH_MARK(1);
#pragma unroll 1
        for (int i = 0; i < nq; i++)
            if (sh->cnt[i] > a.keep) compact_buffer<QCAP, QNT>(sh->cbuf[i], &sh->cnt[i], &sh->thr[i], a.keep, a.gthr + sh->qs[i], &sh->sc);
        if (threadIdx.x == 0) {
            for (int i = 0; i < nq; i++) { unsigned g = *((volatile unsigned*)(a.gthr + sh->qs[i])); if (g > sh->thr[i]) sh->thr[i] = g; }
            sh->ndone_snap = sh->ndone;
            sh->full = 0;
        }
        __syncthreads();
        QPH_MARK(2);
#pragma unroll
        for (int i = 0; i < NS; i++) { thr[i] = sh->thr[i]; tf[i] = quad_thr_f(thr[i]); }
        if (sh->ndone_snap == QNW) break;
    }
}

// 4 x 4 byte transpose: word j of the result = byte j of a, b, c, d (query 0..3 of a packed table).
__device__ __forceinline__ uint4 quad_pack(unsigned a, unsigned b, unsigned c, unsigned d) {
    const unsigned t0 = __byte_perm(a, b, 0x5140), t1 = __byte_perm(a, b, 0x7362);     // [a0 b0 a1 b1], [a2 b2 a3 b3]
    const unsigned u0 = __byte_perm(c, d, 0x5140), u1 = __byte_perm(c, d, 0x7362);
    return make_uint4(__byte_perm(t0, u0, 0x5410), __byte_perm(t0, u0, 0x7632), __byte_perm(t1, u1, 0x5410), __byte_perm(t1, u1, 0x7632));
}
// This warp's first code block of an item into registers (FILT: with its mask word in nmask; not loaded when that is 0).
template <bool FILT>
__device__ __forceinline__ void quad_first_block(const GroupScanArgs& a, const DphUnit* d, uint4 (&nxt)[6], unsigned long long pol,
                                                 unsigned& nmask) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned b = d->bi0 + warp;
    if (b < d->bend) {
        if (FILT) nmask = a.mask[a.mask_off[d->list] + b];
        if (!FILT || nmask) {
            const uint4* p = reinterpret_cast<const uint4*>(a.codes + d->blk * DPH_BLK_BYTES) + (size_t)b * (DPH_BLK_BYTES / 16) + lane;
#pragma unroll
            for (int c6 = 0; c6 < 6; c6++) nxt[c6] = ldg_stream(p + c6 * 32, pol);
        }
    }
}

// Item start-up is kept off the critical path, so that HBM streams across item boundaries: the plan resolves every unit into one
// DphUnit record; the record of the NEXT unit is fetched into shared memory with cp.async while the current one is scanned (its queue
// index is requested at the start of the current item, so that the fetch can be issued right after the table build); a warp that runs
// out of blocks prefetches its first blocks of the next item into L2 (quad_prefetch_next), and every warp loads its first block of the
// next item into registers before the candidates are published, so those are in flight during the publish and the next table build.
// The table sources (a few MB per batch, re-read at every item) are loaded evict_last, the code stream evict_first.
template <bool FILT>
__global__ void __launch_bounds__(QNT, 1) scan_quad_kernel(GroupScanArgs a) {
    unsigned char* const smem = dph_smem;
    QuadShared* sh = reinterpret_cast<QuadShared*>(smem + SMEM_QUAD_TABLES);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int total_units = a.work->total_units;
    const unsigned char* lut8 = reinterpret_cast<const unsigned char*>(a.lutq);
    const unsigned one = a.one;
    const unsigned long long pol_stream = l2_policy_evict_first(), pol_table = l2_policy_evict_last();
    unsigned rot[11];
#pragma unroll
    for (int r = 0; r < 11; r++) {
        unsigned v = 0;
#pragma unroll
        for (int bb = 0; bb < 3; bb++)
            if (3 * r + bb < 32) v |= (unsigned)(((lane + 3 * r + bb) & 31) * 4) << (8 * bb);
        rot[r] = v;
    }
    unsigned long long ph[4] = {0ull, 0ull, 0ull, 0ull}, ph_t = 0ull;
#ifdef DPH_SCAN_PHASES
    if (tid == 0) ph_t = globaltimer_ns();
#endif

    if (tid == 0) sh->unit = atomicAdd(a.next_unit, 1);
    __syncthreads();
    int cur = 0;
    bool any_unit = sh->unit < total_units;
    if (any_unit && tid < (int)(sizeof(DphUnit) / 16))
        reinterpret_cast<uint4*>(&sh->desc[0])[tid] = __ldg(reinterpret_cast<const uint4*>(a.udesc + sh->unit) + tid);
    __syncthreads();
    uint4 nxt[6];
    unsigned nmask = ~0u;
    if (any_unit) {      // the first item's first blocks; later items get theirs at the end of the previous item
        const DphUnit* d = &sh->desc[0];
        const uint4* lb = reinterpret_cast<const uint4*>(a.codes + d->blk * DPH_BLK_BYTES);
        const unsigned* mrow = FILT ? a.mask + a.mask_off[d->list] : nullptr;
        unsigned bp = d->bi0 + warp;
#pragma unroll 1
        for (int r = 0; r < DPH_L2_PREFETCH_ROUNDS && bp < d->bend; r++, bp += QNW)
            if (lane == 0 && (!FILT || mrow[bp])) l2_prefetch_block(lb + (size_t)bp * (DPH_BLK_BYTES / 16), pol_stream);
        quad_first_block<FILT>(a, d, nxt, pol_stream, nmask);
    }
    while (any_unit) {
        int next_u = 0;
        if (tid == 0) next_u = atomicAdd(a.next_unit, 1);          // consumed after the table build (fetch of the next record)
        const DphUnit* dsc = &sh->desc[cur];
        const int nq = dsc->nq;
        const int ntab = nq > 4 ? 2 : 1;
        const unsigned bi0 = dsc->bi0;
        const uint4* lbase = reinterpret_cast<const uint4*>(a.codes + dsc->blk * DPH_BLK_BYTES);
        // this warp's first block is in registers and its first DPH_L2_PREFETCH_ROUNDS blocks are requested into L2
        const unsigned b = bi0 + warp, bp = bi0 + warp + DPH_L2_PREFETCH_ROUNDS * QNW;
        unsigned gq = 0xFFFFFFFFu;
        if (tid < DPH_QUAD_ITEM_Q && tid < nq) gq = *((volatile unsigned*)(a.gthr + dsc->q[tid]));
        {   // ---- packed tables: byte j of a word of table t = query 4t + j's 8-bit entry, wrap-free layout (see above) ----
            // A unit = one 16-byte chunk (four words) of one source row of the table's four queries: four 16-byte loads, a 4 x 4 byte
            // transpose per word, four 16-byte stores.  All 24 loads of a thread (96 KB per CTA) are issued before any store.  The
            // source swizzle (prep.cu: word group g of row `code` at g ^ (code & 3) inside its chunk) spreads the eight threads of a
            // quarter-warp over the eight 16-byte bank groups of a half-row, so the stores are conflict-free.  The empty slots of a
            // short group repeat query 0 (their byte lanes are summed like the others and never pass: threshold +inf), so all loads are
            // unconditional.
            constexpr int UPT = 3 * 256 * 2 / QNT;
            static_assert(UPT * QNT == 3 * 256 * 2, "the build's units divide evenly over the threads");
            uint4* dst = reinterpret_cast<uint4*>(smem);
#pragma unroll 1
            for (int tb = 0; tb < ntab; tb++) {
                const uint4* s0 = reinterpret_cast<const uint4*>(lut8 + (size_t)dsc->q[4 * tb + 0] * DPH_LUTQ8_BYTES);
                const uint4* s1 = reinterpret_cast<const uint4*>(lut8 + (size_t)dsc->q[4 * tb + 1] * DPH_LUTQ8_BYTES);
                const uint4* s2 = reinterpret_cast<const uint4*>(lut8 + (size_t)dsc->q[4 * tb + 2] * DPH_LUTQ8_BYTES);
                const uint4* s3 = reinterpret_cast<const uint4*>(lut8 + (size_t)dsc->q[4 * tb + 3] * DPH_LUTQ8_BYTES);
                uint4 va[UPT], vb[UPT], vc[UPT], vd[UPT];
#pragma unroll
                for (int e = 0; e < UPT; e++) {
                    const int u = tid + e * QNT;
                    va[e] = ldg_policy(s0 + u, pol_table); vb[e] = ldg_policy(s1 + u, pol_table);
                    vc[e] = ldg_policy(s2 + u, pol_table); vd[e] = ldg_policy(s3 + u, pol_table);
                }
#pragma unroll
                for (int e = 0; e < UPT; e++) {
                    const int u = tid + e * QNT, row = u >> 1, h = u & 1;
                    const int seg = row >> 8, code = row & 255, sw = code & 3;
                    const int region = seg < 2 ? tb : 2, half = seg < 2 ? seg : tb;
                    uint4* d = dst + region * 4096 + code * 16 + half * 8 + h * 4;
                    d[0 ^ sw] = quad_pack(va[e].x, vb[e].x, vc[e].x, vd[e].x);
                    d[1 ^ sw] = quad_pack(va[e].y, vb[e].y, vc[e].y, vd[e].y);
                    d[2 ^ sw] = quad_pack(va[e].z, vb[e].z, vc[e].z, vd[e].z);
                    d[3 ^ sw] = quad_pack(va[e].w, vb[e].w, vc[e].w, vd[e].w);
                }
            }
        }
        if (tid < DPH_QUAD_ITEM_Q) { sh->cnt[tid] = 0; sh->qs[tid] = (long long)dsc->q[tid]; sh->thr[tid] = gq; }
        if (tid == 0) { sh->ndone = 0; sh->ndone_snap = 0; sh->full = 0; sh->unit = next_u; }
        __syncthreads();
        QPH_MARK(0);
        // the next unit's record: its head to every warp's slot (for the run-out prefetch), all of it to the other descriptor slot
        const int nu = sh->unit;
        if (nu < total_units) {
            const unsigned char* rec = reinterpret_cast<const unsigned char*>(a.udesc + nu);
            if (lane == 0) { cp_async16(&sh->head[warp][0], rec); cp_async16(&sh->head[warp][1], rec + 16); }
            if (warp == 0 && lane < (int)(sizeof(DphUnit) / 16)) cp_async16(reinterpret_cast<unsigned char*>(&sh->desc[cur ^ 1]) + lane * 16, rec + lane * 16);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        const unsigned* mrow = FILT ? a.mask + a.mask_off[dsc->list] : nullptr;
        if (ntab == 2) quad_item_rounds<2, FILT>(a, sh, dsc, lbase, b, bp, nxt, rot, one, total_units, pol_stream, ph, ph_t, nmask, mrow);
        else quad_item_rounds<1, FILT>(a, sh, dsc, lbase, b, bp, nxt, rot, one, total_units, pol_stream, ph, ph_t, nmask, mrow);
        // every warp waited for its copies before the rounds' last barrier: the next record is visible
        any_unit = nu < total_units;
        if (any_unit) quad_first_block<FILT>(a, &sh->desc[cur ^ 1], nxt, pol_stream, nmask);
        // ---- publish the candidate sets: the (up to) eight region reservations go out together, one barrier ----
        if (tid < nq) sh->base[tid] = atomicAdd(a.cand_cnt + sh->qs[tid], sh->cnt[tid]);
        __syncthreads();
#pragma unroll 1
        for (int i = 0; i < nq; i++) {
            const long long q = sh->qs[i];
            const int cnt = sh->cnt[i];
            const long long off = a.cand_off[q], cap = a.cand_off[q + 1] - off;
            const int basep = sh->base[i];
            for (int c = tid; c < cnt; c += QNT)
                if (basep + c < cap) a.cand[off + basep + c] = sh->cbuf[i][c];
        }
        __syncthreads();             // buffers, counters, sh->unit and the descriptor slots are reused by the next item
        QPH_MARK(3);
        cur ^= 1;
    }
#ifdef DPH_SCAN_PHASES
    if (tid == 0) {
        for (int i = 0; i < 4; i++) atomicAdd(&g_quad_phase_ns[i], ph[i]);
        __threadfence();
        if (atomicAdd(&g_quad_phase_ctas, 1u) == gridDim.x - 1) {
            __threadfence();
            unsigned long long v[4];
            for (int i = 0; i < 4; i++) { v[i] = atomicExch(&g_quad_phase_ns[i], 0ull); }
            printf("scan_quad_kernel phases (ms, summed over %u CTAs): table build %.3f, scan rounds %.3f, compaction barriers %.3f, publish %.3f\n",
                   gridDim.x, v[0] * 1e-6, v[1] * 1e-6, v[2] * 1e-6, v[3] * 1e-6);
            g_quad_phase_ctas = 0;
        }
    }
#endif
}
#undef QPH_MARK

__global__ void smem_base_probe_kernel(unsigned* out) { *out = (unsigned)__cvta_generic_to_shared(dph_smem); }

static int dph_scan_setup_attrs() {
    static DphPerDeviceOnce once;
    if (!once.first()) return 0;
    {
        unsigned* d = nullptr; unsigned h = 0;
        DPH_CUDA(cudaMalloc((void**)&d, 4));
        smem_base_probe_kernel<<<1, 32, 1024>>>(d);
        DPH_CUDA(cudaMemcpy(&h, d, 4, cudaMemcpyDeviceToHost));
        cudaFree(d);
        // the quad scan also needs the window's top address byte to be 0 (its gather addresses are built without it)
        DPH_CHECK(h == DPH_DYN_SMEM_BASE, "dynamic shared memory window does not start at 0x400 on this driver; rebuild with the probed value");
    }
    for (auto f : {scan_kernel<DPH_SCAN_FAST, DPH_FILT_NONE>, scan_kernel<DPH_SCAN_FAST, DPH_FILT_MASK>, scan_kernel<DPH_SCAN_FAST, DPH_FILT_QUERY>})
        DPH_CUDA(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LUT_FAST + (int)sizeof(ScanShared)));
    for (auto f : {scan_kernel<DPH_SCAN_EXACT, DPH_FILT_NONE>, scan_kernel<DPH_SCAN_EXACT, DPH_FILT_MASK>, scan_kernel<DPH_SCAN_EXACT, DPH_FILT_QUERY>})
        DPH_CUDA(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LUT_EXACT + (int)sizeof(ScanShared)));
    for (auto f : {scan_pair_kernel<false>, scan_pair_kernel<true>})
        DPH_CUDA(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LUT_FAST + (int)sizeof(PairShared)));
    for (auto f : {scan_quad_kernel<false>, scan_quad_kernel<true>})
        DPH_CUDA(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_QUAD_TABLES + (int)sizeof(QuadShared)));
    return 0;
}

int dph_launch_scan(dph_index* ix, const DphSearchPlan& p, const DphCodeSrc& src, int64_t n, bool exact, cudaStream_t st) {
    if (n == 0) return 0;
    DPH_TRY(dph_scan_setup_attrs());
    const int grid = p.grid, group = p.pass_group(exact), keep = p.pass_keep(exact);
    const bool filt = src.mask != nullptr;          // the row mask is indexed in the shard's own block numbering (ix->blk_off)
    const bool qfilt = src.qf != nullptr;           // per-query selectors: the one-query scan only (search_plan)
    DPH_CHECK(group == 1 || !qfilt, "scan: a per-query filter runs the one-query scan only");
    if (group == 1) {
        ScanArgs a;
        a.codes = src.codes; a.qpre = ix->wpre.as<long long>(); a.segs = ix->segs.as<DphSeg>(); a.nseg = ix->nseg.as<int>(); a.work = ix->work.as<DphWork>();
        a.lut_canon = ix->lut_canon.as<float>(); a.gthr = ix->gthr.as<unsigned>();
        a.cand = ix->cand.as<unsigned long long>(); a.cand_off = ix->cand_off.as<long long>(); a.cand_cnt = ix->cand_cnt.as<int>();
        a.n = n; a.nprobe = ix->nprobe; a.keep = keep;
        a.mask = src.mask; a.mask_off = (const long long*)ix->blk_off; a.qf = src.qf;
        const size_t smem = (exact ? SMEM_LUT_EXACT : SMEM_LUT_FAST) + sizeof(ScanShared);
        auto f = exact ? (qfilt ? scan_kernel<DPH_SCAN_EXACT, DPH_FILT_QUERY> : filt ? scan_kernel<DPH_SCAN_EXACT, DPH_FILT_MASK> : scan_kernel<DPH_SCAN_EXACT, DPH_FILT_NONE>)
                       : (qfilt ? scan_kernel<DPH_SCAN_FAST, DPH_FILT_QUERY> : filt ? scan_kernel<DPH_SCAN_FAST, DPH_FILT_MASK> : scan_kernel<DPH_SCAN_FAST, DPH_FILT_NONE>);
        f<<<grid, NT, smem, st>>>(a);
    } else {
        GroupScanArgs a;
        a.codes = src.codes; a.blk_off = src.blk_off; a.list_len = ix->list_len; a.grp_cnt = ix->grp_cnt.as<int>();
        a.grp_off = ix->grp_off.as<int>(); a.units = ix->grp_units.as<unsigned long long>(); a.entries = ix->grp_entries.as<unsigned>();
        a.work = ix->groupwork.as<DphGroupWork>(); a.next_unit = &ix->groupwork.as<DphGroupWork>()->next_unit; a.lutq = ix->lutq.as<unsigned short>(); a.qparams = ix->qparams.as<float2>();
        a.cd = ix->cd.as<float>(); a.gdense = ix->gdense.as<unsigned>(); a.gthr = ix->gthr.as<unsigned>();
        a.cand = ix->cand.as<unsigned long long>(); a.cand_off = ix->cand_off.as<long long>(); a.cand_cnt = ix->cand_cnt.as<int>();
        a.list_lo = src.lo; a.list_hi = src.hi; a.nprobe = ix->nprobe; a.keep = keep;
        a.udesc = ix->grp_udesc.as<DphUnit>(); a.one = 1u;
        a.mask = src.mask; a.mask_off = (const long long*)ix->blk_off;
        if (group == 4) (filt ? scan_quad_kernel<true> : scan_quad_kernel<false>)<<<grid, QNT, SMEM_QUAD_TABLES + sizeof(QuadShared), st>>>(a);
        else (filt ? scan_pair_kernel<true> : scan_pair_kernel<false>)<<<grid, NT, SMEM_LUT_FAST + sizeof(PairShared), st>>>(a);
    }
    DPH_CUDA(cudaGetLastError());
    return 0;
}

// =================================================================================================
// merge: one CTA per query.  FAST: prove the filter, re-score survivors in canonical order, sort.
// EXACT: candidates already carry canonical scores.  Output: D (score desc), I (labels), G (scan position).
// =================================================================================================
struct MergeArgs {
    const unsigned long long* cand; const long long* cand_off; const int* cand_cnt; const unsigned* gthr; const float* eps;
    const DphSeg* segs; const int* nseg; int nprobe; int k; int mode;
    const uint8_t* codes; const float* lut_canon; const long long* ids; const long long* list_start;
    const long long* lab_off;       // the shard's first block of each list: labels follow its layout whatever `codes` is
    float* D; long long* I; unsigned* G; int* flags; const int* only_flagged;
};

// last segment r with gstart[r] <= gidx; gstart = the query's segment starts, staged in shared memory by the caller (a binary search
// over the descriptors in global memory is a chain of ~8 dependent L2 round trips per survivor)
__device__ __forceinline__ int find_seg(const unsigned* gstart, int nsg, unsigned gidx) {
    int lo = 0, hi = nsg;
    while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (gstart[mid] <= gidx) lo = mid; else hi = mid; }
    return lo;
}

__global__ void __launch_bounds__(256) merge_kernel(MergeArgs a) {
    __shared__ SelectScratch sc;
    __shared__ unsigned long long surv[DPH_SURV_CAP];
    __shared__ unsigned sgs[DPH_MAX_NPROBE];
    __shared__ int scnt, sflag;
    const long long q = blockIdx.x;
    const int tid = threadIdx.x;
    if (a.only_flagged && a.only_flagged[q] == 0) return;
    const unsigned long long* E = a.cand + a.cand_off[q];
    long long cap = a.cand_off[q + 1] - a.cand_off[q];
    int n = a.cand_cnt[q];
    const bool overflow = n > cap;          // cannot happen with the plan's capacity bound; if it ever does the query goes to the exact kernel
    if (n > cap) n = (int)cap;
    const DphSeg* segs = a.segs + q * a.nprobe;
    const int nsg = a.nseg[q];
    const int k = a.k;
    if (tid == 0) { scnt = 0; sflag = 0; }
    for (int i = tid; i < nsg; i += blockDim.x) sgs[i] = segs[i].gstart;
    __syncthreads();
    auto get = [&](int i) { return E[i]; };
    unsigned long long pivot = 0ull;   // gather keys >= pivot
    int flag = overflow ? 1 : 0;
    if (a.mode == DPH_SCAN_FAST) {
        const float eps2 = 2.0f * a.eps[q];
        const unsigned gt = a.gthr[q];
        if (n > k) {
            unsigned long long pk = block_radix_select(get, n, k, &sc);
            const float Tk = dph_ckey_score(pk);
            if (gt != 0u && !(Tk - dph_fkey_inv(gt) > eps2)) flag = 1;
            pivot = (unsigned long long)dph_fkey(Tk - eps2) << 32;       // every entry with filter score >= Tk - 2eps
        } else if (gt != 0u) flag = 1;
    } else {
        if (n > DPH_SURV_CAP) pivot = block_radix_select(get, n, k, &sc);
    }
    for (int i = tid; i < n; i += blockDim.x) {
        unsigned long long e = E[i];
        if (e >= pivot) { int p = atomicAdd(&scnt, 1); if (p < DPH_SURV_CAP) surv[p] = e; else sflag = 1; }
    }
    __syncthreads();
    int ns = scnt < DPH_SURV_CAP ? scnt : DPH_SURV_CAP;
    if (sflag) flag = 1;
    if (a.mode == DPH_SCAN_FAST) {
        // exact re-scoring, one WARP per survivor: lane l fetches the code byte and the LUT entry of sub-quantizers l, l+32, l+64
        // (96 independent loads in flight instead of a 96-long chain of dependent L2 round trips), then the lanes' values are added
        // in canonical m-ascending order (bit-exact with the oracle: dis = dis0; for m: dis += LUT[m][c[m]]).
        const float* lutc = a.lut_canon + (size_t)q * DPH_LUT_CANON_FLOATS;
        const int lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
        for (int i = warp; i < ns; i += nwarps) {
            const unsigned gidx = dph_ckey_gidx(surv[i]);
            const DphSeg s = segs[find_seg(sgs, nsg, gidx)];
            const unsigned j = gidx - s.gstart;
            const uint8_t* blk = a.codes + (s.blk + (long long)(j >> 5)) * DPH_BLK_BYTES;
            const int ln = (int)(j & 31u);
            float v[3];
#pragma unroll
            for (int h = 0; h < 3; h++) {
                const int m = h * 32 + lane;
                v[h] = __ldg(lutc + DPH_LUTC_IDX(m, (int)blk[dph_blk_addr(ln, m)]));
            }
            float dis = s.dis0;
#pragma unroll
            for (int h = 0; h < 3; h++)
#pragma unroll
                for (int l2 = 0; l2 < 32; l2++) dis += __shfl_sync(0xffffffffu, v[h], l2);
            __syncwarp();
            if (lane == 0) surv[i] = dph_ckey(dis, gidx);
        }
    }
    const int p2 = dph_next_pow2(ns > 1 ? ns : 1);
    for (int i = ns + tid; i < p2; i += blockDim.x) surv[i] = 0ull;
    __syncthreads();
    block_bitonic_sort_desc(surv, p2);
    for (int i = tid; i < k; i += blockDim.x) {
        float d = DPH_NEUTRAL; long long id = -1; unsigned gi = 0xFFFFFFFFu;
        if (i < ns) {
            const unsigned long long e = surv[i];
            gi = dph_ckey_gidx(e); d = dph_ckey_score(e);
            const DphSeg s = segs[find_seg(sgs, nsg, gi)];
            const unsigned j = gi - s.gstart;
            id = a.ids ? a.ids[a.lab_off[s.list] * 32 + j] : a.list_start[s.list] + (long long)j;
        }
        a.D[q * k + i] = d; a.I[q * k + i] = id; a.G[q * k + i] = gi;
    }
    if (a.mode == DPH_SCAN_FAST && tid == 0) a.flags[q] = flag;
}

int dph_launch_merge(dph_index* ix, const uint8_t* codes, int64_t n, int k, int mode, const int32_t* only_flagged, float* D, int64_t* I,
                     uint32_t* G, cudaStream_t st) {
    if (n == 0) return 0;
    MergeArgs a;
    a.cand = ix->cand.as<unsigned long long>(); a.cand_off = ix->cand_off.as<long long>(); a.cand_cnt = ix->cand_cnt.as<int>();
    a.gthr = ix->gthr.as<unsigned>(); a.eps = ix->eps.as<float>(); a.segs = ix->segs.as<DphSeg>(); a.nseg = ix->nseg.as<int>(); a.nprobe = ix->nprobe; a.k = k; a.mode = mode;
    a.codes = codes; a.lut_canon = ix->lut_canon.as<float>(); a.ids = (const long long*)ix->ids; a.list_start = (const long long*)ix->list_start;
    a.lab_off = (const long long*)ix->blk_off;
    a.D = D; a.I = (long long*)I; a.G = G; a.flags = ix->flags.as<int>(); a.only_flagged = only_flagged;
    merge_kernel<<<(unsigned)n, 256, 0, st>>>(a);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

// =================================================================================================
// pack / merge of the per-shard partial top-k for ONE all-gather:  P[q][i] = { ckey(score, scan position), label }.
// =================================================================================================
__global__ void pack_topk_kernel(const float* D, const long long* I, const unsigned* G, long long total, longlong2* P) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    longlong2 v;
    v.x = I[i] >= 0 ? (long long)dph_ckey(D[i], G[i]) : 0ll;
    v.y = I[i];
    P[i] = v;
}
__global__ void __launch_bounds__(256) merge_packed_kernel(const longlong2* Pg, int nshards, long long n, int k, float* D, long long* I) {
    extern __shared__ unsigned long long mp[];      // [p2] keys, then [p2] labels
    const long long q = blockIdx.x;
    const int tot = nshards * k, p2 = dph_next_pow2(tot);
    unsigned long long* keys = mp;
    for (int i = threadIdx.x; i < p2; i += blockDim.x) {
        unsigned long long key = 0ull;
        if (i < tot) key = (unsigned long long)Pg[((long long)(i / k) * n + q) * k + (i % k)].x;
        keys[i] = key;
    }
    __syncthreads();
    block_bitonic_sort_desc(keys, p2);
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        float d = DPH_NEUTRAL; long long id = -1;
        const unsigned long long key = keys[i];
        if (key != 0ull) {
            d = dph_ckey_score(key);
            for (int j = 0; j < tot && id < 0; j++) {          // scan positions are unique per query: find the owner (<= nshards*k entries)
                const longlong2 e = Pg[((long long)(j / k) * n + q) * k + (j % k)];
                if ((unsigned long long)e.x == key) id = e.y;
            }
        }
        D[q * k + i] = d; I[q * k + i] = id;
    }
}
DPH_API int dph_pack_topk(const float* D, const int64_t* I, const uint32_t* G, int64_t n, int k, int64_t* P, void* cuda_stream) {
    const long long total = (long long)n * k;
    if (total == 0) return 0;
    pack_topk_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(D, (const long long*)I, G, total, (longlong2*)P);
    DPH_CUDA(cudaGetLastError());
    return 0;
}
DPH_API int dph_merge_shards_packed(const int64_t* Pg, int nshards, int64_t n, int k, float* D, int64_t* I, void* cuda_stream) {
    if (n == 0) return 0;
    DPH_CHECK(nshards >= 1 && k >= 1 && (long long)nshards * k <= 8192, "merge_shards: nshards*k must be <= 8192");
    int p2 = 1; while (p2 < nshards * k) p2 <<= 1;
    static DphPerDeviceOnce once;
    if (once.first()) { DPH_CUDA(cudaFuncSetAttribute(merge_packed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8)); }
    merge_packed_kernel<<<(unsigned)n, 256, p2 * 8, (cudaStream_t)cuda_stream>>>((const longlong2*)Pg, nshards, n, k, D, (long long*)I);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

// =================================================================================================
// merge_shards: all-gathered per-shard top-k -> global top-k, order (score desc, scan position asc).
// =================================================================================================
__global__ void __launch_bounds__(256) merge_shards_kernel(const float* Dg, const long long* Ig, const unsigned* Gg, int nshards, long long n,
                                                            int k, float* D, long long* I, unsigned* G) {
    extern __shared__ unsigned long long ms[];     // keys [p2] then payload index is recovered from a parallel array
    const long long q = blockIdx.x;
    const int tid = threadIdx.x;
    const int tot = nshards * k;
    const int p2 = dph_next_pow2(tot);
    unsigned long long* keys = ms;
    // key = (fkey(score), ~gidx); payload looked up afterwards by matching (shard, slot) stored in a side table:
    // gidx is unique per real entry, so re-find the source by scanning the <= nshards*k inputs (tiny).
    for (int i = tid; i < p2; i += blockDim.x) {
        unsigned long long key = 0ull;
        if (i < tot) {
            int s = i / k, r = i % k;
            long long id = Ig[((long long)s * n + q) * k + r];
            if (id >= 0) key = dph_ckey(Dg[((long long)s * n + q) * k + r], Gg[((long long)s * n + q) * k + r]);
        }
        keys[i] = key;
    }
    __syncthreads();
    block_bitonic_sort_desc(keys, p2);
    for (int i = tid; i < k; i += blockDim.x) {
        float d = DPH_NEUTRAL; long long id = -1;
        unsigned long long key = keys[i];
        unsigned gi = 0xFFFFFFFFu;
        if (key != 0ull) {
            gi = dph_ckey_gidx(key);
            d = dph_ckey_score(key);
            for (int s = 0; s < nshards && id < 0; s++)
                for (int r = 0; r < k; r++) {
                    long long o = ((long long)s * n + q) * k + r;
                    if (Gg[o] == gi && Ig[o] >= 0) { id = Ig[o]; break; }
                }
        }
        D[q * k + i] = d; I[q * k + i] = id;
        if (G) G[q * k + i] = gi;
    }
}

int dph_launch_merge_shards(const float* Dg, const int64_t* Ig, const uint32_t* Gg, int nshards, int64_t n, int k, float* D, int64_t* I,
                            uint32_t* G, cudaStream_t st) {
    if (n == 0) return 0;
    DPH_CHECK(nshards >= 1 && k >= 1 && (long long)nshards * k <= 8192, "merge_shards: nshards*k must be <= 8192");
    int p2 = 1; while (p2 < nshards * k) p2 <<= 1;
    static DphPerDeviceOnce once;
    if (once.first()) { DPH_CUDA(cudaFuncSetAttribute(merge_shards_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8)); }
    merge_shards_kernel<<<(unsigned)n, 256, p2 * 8, st>>>(Dg, (const long long*)Ig, Gg, nshards, n, k, D, (long long*)I, G);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

DPH_API int dph_merge_shards(const float* Dg, const int64_t* Ig, const uint32_t* Gg, int nshards, int64_t n, int k, float* D, int64_t* I,
                                void* cuda_stream) {
    return dph_launch_merge_shards(Dg, Ig, Gg, nshards, n, k, D, I, nullptr, (cudaStream_t)cuda_stream);
}
