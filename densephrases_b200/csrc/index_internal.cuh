// index_internal.cuh -- the dph_index handle, the search plan and the internal kernel-launch prototypes.
#pragma once
#include "common.cuh"
#include "../../include/dph_b200.h"
#include <algorithm>
#include <functional>
#include <string.h>
#include <vector>

#define DPH_SCAN_THREADS 512
#define DPH_SCAN_WARPS (DPH_SCAN_THREADS / 32)
#define DPH_CAND_CAP 3072          // one-query scan: shared-memory candidate buffer (u64 keys) per CTA; holds every k's keep (scan.cu)
#define DPH_PAIR_KEEP_MAX 1024      // pair mode: PCAP (1536) - pair scan threads (512), see scan.cu
#define DPH_QUAD_KEEP_MAX 256       // quad mode: QCAP (512) - quad scan threads (256), see scan.cu

#define DPH_KEEP_SLACK 32          // fast mode keeps k + slack candidates per CTA
#define DPH_MAX_K 1024
#define DPH_PROF_RING 64
#define DPH_MAX_NPROBE 1024
#define DPH_SURV_CAP 2048          // merge kernel: survivors re-scored exactly per query
#define DPH_LUT_SCAN_FLOATS (3 * 256 * 64)   // per query: 3 segments x 256 codes x (32 + 31 dup + 1 pad)
#define DPH_LUTQ8_BYTES (3 * 256 * 32)       // per query: the quad scan's compact 8-bit table source (prep.cu, lutq_kernel)
#define DPH_LUT_CANON_FLOATS (96 * 256)
// The canonical fp32 table of a query, LUT[m][code] = <xr[8m..8m+8), pq[m][code]>, is stored segment-major, code-major,
// sub-quantizer-minor: [3 segments of 32 sub-quantizers][256 codes][32] -- i.e. already in the row order the conflict-free scan
// layout needs (scan.cu), so ONE 96 KB table per query serves the one-query scan (staged with its wrap copies), the quantised
// pair / quad tables, the exact kernel and the exact re-scoring in the merge.
#define DPH_LUTC_IDX(m, code) ((((m) >> 5) << 13) + ((code) << 5) + ((m) & 31))
#define DPH_SEG_SMEM 256            // segment descriptors of one query kept in shared memory by the scan kernel
#define DPH_L2_PREFETCH_ROUNDS 2    // scan kernels: bulk L2 prefetch distance, in rounds (one 3 KB block per warp per round; tools/scan_floor.cu)

struct DevBuf {            // grow-only device buffer; freed with its owner, on the owner's device (which must be current)
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    int ensure(size_t bytes);
    template <class T> T* as() const { return (T*)p; }
};

// The shard's lists as tightly packed 32-row code blocks, derived from the lengths of all lists (DESIGN.md 3).  set_lists, add,
// remove and sync_list_len build one; dph_commit_layout makes it the handle's (dph_index::lay).
struct DphLayout {
    int64_t lo = 0, hi = 0;             // the shard's lists
    std::vector<int32_t> len;           // [nlist]
    std::vector<int64_t> start;         // [nlist+1] global list-major row of each list's first vector
    std::vector<int64_t> blk_off;       // [nlist]   first code block of the list in the shard (-1 outside it)
    std::vector<int64_t> row_start;     // [max(hi-lo, 1)] shard-local row of each shard list's first vector
    int64_t nblocks = 0, rows = 0;      // of the shard
    // Fails with `what` (the index unchanged) unless 0 <= list_len[l] < 2^31 for every list.
    int build(const dph_index* ix, const int64_t* list_len, const char* what);
    // Staging chunks: runs of whole lists of at most dph_chunk_rows() rows (a longer list is a chunk alone), no empty chunk.
    struct Chunk { int64_t row0, rows, blk0, blk1; };      // shard-local rows [row0, row0 + rows), blocks [blk0, blk1)
    std::vector<Chunk> chunks(int64_t* max_rows) const;
};
struct dph_index {
    int device = 0;
    int d = DPH_D, M = DPH_M;
    int64_t nlist = 0;
    int nprobe = 256;
    int scan_mode = DPH_SCAN_FAST;
    cudaStream_t stream = 0;
    int num_sms = 132;

    // model
    float* A = nullptr;         // [d,d]
    float* C = nullptr;         // [nlist,d]
    float* pq = nullptr;        // [M,256,dsub]
    // lists
    int64_t list_lo = 0, list_hi = 0;   // shard range
    int64_t ntotal = 0, ntotal_local = 0, nblocks_local = 0;
    int32_t* list_len = nullptr;        // [nlist]   (all lists)
    int64_t* list_start = nullptr;      // [nlist+1] global list-major row of each list's first vector
    int64_t* blk_off = nullptr;         // [nlist]   first code block in `codes` (-1 when not in shard)
    uint8_t* codes = nullptr;           // [nblocks_local * 3072] interleaved blocks
    int64_t* ids = nullptr;             // [nblocks_local * 32] labels (or nullptr: sequential)
    // direct map for explicit ids (sorted labels -> local padded row); built at set_lists
    int64_t* dm_ids = nullptr;
    int64_t* dm_rows = nullptr;
    int64_t dm_n = 0;
    int64_t dm_cap = 0;                 // entries allocated for dm_ids / dm_rows
    int64_t blk_cap = 0;                // blocks allocated for codes / ids (a remove does not shrink them)
    DphLayout lay;                      // host copy of the committed layout

    // per-batch workspace
    DevBuf xdev, xr, S, key, cd, lut_canon, lutmax, segs, wpre, qinfo, cand, cand_off, cand_cnt, gthr, flags,
        work, Dp, Ip, Gp, eps, nseg,
        lutmin, lutmaxv, lutq, qparams, gdense,
        grp_cnt, grp_fill, grp_off, grp_blockpre, grp_entries, grp_unitpre, grp_units, grp_udesc, groupwork,   // grouped plan (prep.cu)
        csplit, xsplit, candkeys, cflags, selkeys,
        rb_ids, rb_out, rb_found, ws_q, ws_id, ws_out, ws_xq,        // reconstruct_batch / window_scores staging (host-buffer calls)
        enc_key, enc_cd, enc_list, enc_codes, enc_q8,                // encode / add: top-1 coarse result, host-call staging
        qfview;                                                      // the search chunk's DphQfView (per-query filter)
    int64_t csplit_lo = -1, csplit_nl = -1;
    int coarse_tc = 1;                 // tensor-core coarse quantizer with exact re-rank (0: always the SIMT sequential-k GEMM)
    int last_group = 1;                // queries per gather used by the last search (1, 2 or 4)
    int64_t last_coarse_n = -1;
    bool profile = false;              // CUDA events around the scan kernel of the last search chunk
    cudaEvent_t ev0[DPH_PROF_RING] = {}, ev1[DPH_PROF_RING] = {};
    int64_t prof_n = 0;
    cudaEvent_t aev[6] = {};           // profiled adds, removes and merges: stage boundaries (encode.cu, lists.cu, remove.cu, merge.cu)
    float add_ms[4] = {};              // last add: rotation, coarse, PQ encode, re-layout + scatter (ms)
    float remove_ms[3] = {};           // last remove: mark + plan, row moves + block shift, direct map (ms)
    float merge_ms[4] = {};            // last merge: plan + alloc, block moves, source rows, direct map (ms)
    float train_ms[3] = {};            // last train_coarse / train_pq: assign, sort + update, split + renorm (ms, summed over iterations)
    int64_t remove_tmp_peak = 0;       // last remove: largest total of its temporary device allocations (bytes)

    // Codes in host memory (host_codes.cu, DESIGN.md 3.5).  `codes` is then the device pointer of the mapped host array host_codes,
    // and `region` [region_blocks] holds in HBM the resident lists' blocks [0, res_blocks), then the stream region (the rest).
    // stream_blocks is the stream size the caller asked for; a mutation that empties the resident set leaves the whole region to the
    // stream.
    bool on_host = false;
    uint8_t* host_codes = nullptr;
    uint8_t* region = nullptr;
    int64_t res_blocks = 0, stream_blocks = 0, region_blocks = 0;
    // A reserved host capacity (host_move.cu): host_blocks = blocks allocated in host_codes (max(host_reserve, the shard's blocks) at
    // set_lists); host_mutable = reserve_host_codes was called, so add, remove, sync_list_len and merge run in place on host_codes.
    int64_t host_blocks = 0, host_reserve = 0;
    bool host_mutable = false;
    int64_t move_counts[3] = {};       // last host mutation: blocks read from and written to the host array, staging chunks
    float move_ms = 0.f;               // last host mutation: time of the in-place block mover
    std::vector<int64_t> res_off;      // [nlist] block of a resident list in `region`, else -1
    int64_t* res_off_dev = nullptr;    // [nlist] device copy
    int64_t max_stream_blocks = 0;     // the shard's largest non-resident list, in blocks
    int64_t fetch_counts[4] = {};      // last search: slices, lists fetched, blocks fetched, resident lists scanned
    float fetch_ms = 0.f;              // last search: time of its fetch kernels (profiling on)
    DevBuf view, fdesc, hs_D, hs_I, hs_G;   // per slice: block-offset view, fetch descriptors, the running top-k and the slice's

    // Filtered search (filter.cu, DESIGN.md 3.6): the committed layout's serial (process-wide unique, set by dph_commit_layout) and
    // the filter later searches apply (dph_index_set_filter; nullptr: none).
    uint64_t layout_version = 0;
    const dph_filter* filter = nullptr;
    // Per-query filtered search (query_filter.cu, DESIGN.md 3.7): the query filter later searches apply (dph_index_set_query_filter).
    // At most one of filter and qfilter is set.
    const dph_query_filter* qfilter = nullptr;
};

// A row mask of one shard: mask[b] bit l = row l of the shard's code block b is selected.  Valid for ix while ix->layout_version ==
// version.
struct dph_filter {
    dph_index* ix = nullptr;
    uint64_t version = 0;
    uint32_t* mask = nullptr;           // [nwords] device
    int64_t nwords = 0, rows = 0;
};

// Per-query selectors of one search chunk, on the device (dph_query_filter): assign[q] = query q's selector, -1 = none.  Selector f's
// blocks of shard list lo + i are entries base[f] + [off[f * stride + i], off[f * stride + i + 1]) of blk (the list's block numbers,
// ascending) and word (their mask words: bit l = lane l's row is selected).
struct DphQfView {
    const int32_t* assign; const uint32_t* off; const long long* base; const uint32_t* blk; const uint32_t* word;
    long long lo, stride;
};
// A per-query filter of one shard (query_filter.cu): F selectors in the CSR of DphQfView, and the selector of each of n queries.
// Valid for ix while ix->layout_version == version.
struct dph_query_filter {
    dph_index* ix = nullptr;
    uint64_t version = 0;
    int64_t nsel = 0, n = 0, lo = 0, nl = 0;     // selectors, queries, the shard's first list and its list count
    int32_t* assign = nullptr;                   // [n] device
    uint32_t* off = nullptr;                     // [nsel * (nl + 1)] device
    int64_t* base = nullptr;                     // [nsel + 1] device
    uint32_t *blk = nullptr, *word = nullptr;    // [nblk] device
    int64_t nblk = 0;
    std::vector<int64_t> h_base, rows;           // host copies: base [nsel + 1], selected rows per selector [nsel]
    DphQfView view(int64_t q0) const { return {assign + q0, off, (const long long*)base, blk, word, (long long)lo, (long long)nl + 1}; }
};

// Where the scan stage reads the codes of lists [lo, hi): the handle's own blocks, or in host mode the view of one slice.  mask: the
// active filter's row mask, indexed in the shard's own block numbering (ix->blk_off), or nullptr.  qf: the active per-query filter's
// selectors for the chunk's queries, indexed by list (a device copy of the view: the scan kernel's arguments gain one pointer only), or
// nullptr.
struct DphCodeSrc { const uint8_t* codes; const long long* blk_off; int64_t lo, hi; const uint32_t* mask; const DphQfView* qf; };

// Writes list_len / list_start / blk_off of `L` to the device and makes `L` the handle's layout, totals included; the only code
// that does.
int dph_commit_layout(dph_index* ix, DphLayout L);
void dph_free_lists(dph_index* ix);            // the handle's list arrays go; it then has no lists
int check_ready(dph_index* ix, int k);

__device__ __forceinline__ long long lower_bound_ll(const long long* a, long long n, long long key) {      // first i with a[i] >= key
    long long lo = 0, hi = n;
    while (lo < hi) { const long long mid = (lo + hi) >> 1; if (a[mid] < key) lo = mid + 1; else hi = mid; }
    return lo;
}
// Block -> list lookup inside the shard: last l in [lo,hi) with blk_off[l] <= blk.
__device__ __forceinline__ long long list_of_block(const long long* blk_off, long long lo, long long hi, long long blk) {
    while (hi - lo > 1) { long long mid = (lo + hi) >> 1; if (blk_off[mid] <= blk) lo = mid; else hi = mid; }
    return lo;
}
// One 96-byte code row -> the lane-rotated layout of fill_blocks_kernel / common.cuh:dph_blk_addr (six 16-byte stores of one lane).
__device__ __forceinline__ void dph_store_row(uint8_t* codes, long long blk, int lane, const unsigned char* row) {
#pragma unroll
    for (int c = 0; c < 6; c++) {
        unsigned char bytes[16];
#pragma unroll
        for (int b = 0; b < 16; b++) bytes[b] = row[dph_blk_sub(lane, c * 16 + b)];
        uint4 v;
        memcpy(&v, bytes, 16);
        *reinterpret_cast<uint4*>(codes + blk * DPH_BLK_BYTES + c * 512 + lane * 16) = v;
    }
}
// The inverse: the row of `lane` in block `blk`, m ascending.
__device__ __forceinline__ void dph_load_row(const uint8_t* codes, long long blk, int lane, unsigned char* row) {
#pragma unroll
    for (int c = 0; c < 6; c++) {
        const uint4 v = *reinterpret_cast<const uint4*>(codes + blk * DPH_BLK_BYTES + c * 512 + lane * 16);
        unsigned char bytes[16];
        memcpy(bytes, &v, 16);
#pragma unroll
        for (int b = 0; b < 16; b++) row[dph_blk_sub(lane, c * 16 + b)] = bytes[b];
    }
}

struct DevTmp {            // the device allocations of one call, freed on every exit path unless released
    std::vector<void*> ps;
    int64_t live = 0, peak = 0;             // bytes allocated through this object (released ones included), and the largest total
    ~DevTmp() { for (void* p : ps) if (p) cudaFree(p); }
    template <class T> int alloc(T** out, size_t count, const char* what) {
        const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
        cudaError_t e = cudaMalloc((void**)out, bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();                     // an allocation failure is not sticky: keep it out of later error checks
            *out = nullptr;
            dph_set_error(std::string(what) + ": " + cudaGetErrorString(e));
            return 1;
        }
        ps.push_back(*out);
        live += (int64_t)bytes; peak = std::max(peak, live);
        return 0;
    }
    void release(void* p) { for (void*& q : ps) if (q == p) q = nullptr; }
};

// A label-set selector on the device (remove.cu): ids [n] (mem: where they live) copied into a temporary of `tmp`, sorted and
// de-duplicated on st -> *out [*nu].  `what` prefixes the error.
int dph_label_set(DevTmp& tmp, const int64_t* ids, int64_t n, int mem, cudaStream_t st, long long** out, int64_t* nu, const char* what);
// Rows per staging chunk of set_lists / copy_lists / remove (about 256 MB of code rows; DPH_UPLOAD_CHUNK_ROWS overrides it for tests).
int64_t dph_chunk_rows();
// Block re-layout of the add (lists.cu), also the remove's block shift: blocks [blk0, blk0 + gridDim.x) of the layout boff_new are
// written to dst[0 ..) from the same list's block in boff_old (whole, same rows and lanes; zeros / -1 past the list's old end).
__global__ void relayout_codes_kernel(uint8_t* dst, long long blk0, const long long* boff_new, const long long* boff_old, const int* len_old,
                                      long long lo, long long hi, const uint8_t* codes_old);
__global__ void relayout_ids_kernel(long long* dst, long long blk0, const long long* boff_new, const long long* boff_old, const int* len_old,
                                    long long lo, long long hi, const long long* ids_old, const long long* list_start_old,
                                    const long long* lrs_old, long long* dm_ids, long long* dm_rows);

// What the scan stage of one batch runs (search.cu).  The FAST pass keeps `keep` candidates per scan CTA and query and its merge
// flags the queries it cannot prove exact; the EXACT pass (scan_kernel<EXACT>, keep = k) re-runs those, or runs alone in EXACT mode.
struct DphSearchPlan {
    int k;
    bool exact_only;    // EXACT scan mode: no fast pass, the exact pass scans every query
    int group;          // fast pass: queries per gather -- 1 (fp32 LUT), 2 (pair-packed u16 LUTs) or 4 (quad-packed u8 LUTs)
    int keep;           // fast pass: candidates kept per scan CTA and query
    int item_q;         // fast pass: queries per work item -- 2 (pair), DPH_QUAD_ITEM_Q (quad), 1 (one query: no items)
    int grid;           // scan CTAs: one persistent CTA per SM
    bool grouped() const { return group > 1; }
    int pass_group(bool exact) const { return exact ? 1 : group; }
    int pass_keep(bool exact) const { return exact ? k : keep; }
};

// ---- prep.cu ----
int dph_launch_sgemm_nt_seq(const float* X, int64_t n, const float* W, int64_t m, int K, float* out, cudaStream_t st);
int dph_launch_coarse_select(const float* S, int64_t n, int64_t nlist, int nprobe, int32_t* key, float* cd, cudaStream_t st,
                             unsigned long long* keys64 = nullptr, unsigned list_base = 0, const int* only_rows = nullptr, int64_t ld = 0,
                             DevBuf* tmp = nullptr);      // tmp: scratch for the chunked selection of long rows (nullptr: one CTA per row)
int dph_coarse_tc(dph_index* ix, int64_t n, int64_t lo, int64_t nl, int nprobe, unsigned long long* keys64, int32_t* key, float* cd, cudaStream_t st,
                  const float* xr = nullptr, const float* C = nullptr);
int dph_launch_coarse_merge(const unsigned long long* keys, int W, int64_t n, int nprobe, int32_t* key, float* cd, cudaStream_t st,
                            unsigned long long* keys64 = nullptr);
int dph_launch_lut(const float* xr, int64_t n, const float* pq, float* lut_canon, float* lutmax, float* lutmin, float* lutmaxv,
                   void* lutq, float2* qparams, cudaStream_t st, int group);
// One pass of plan p (only_flagged, nullable: only the queries whose flag is set): segments, work, candidate areas, eps, group queue.
int dph_launch_plan(dph_index* ix, const DphSearchPlan& p, const DphCodeSrc& src, int64_t n, bool exact, const int32_t* only_flagged,
                    cudaStream_t st);
// ---- scan.cu ----
// One pass: scan_kernel<EXACT> (exact), else by p.group scan_kernel<FAST>, scan_pair_kernel or scan_quad_kernel.
int dph_launch_scan(dph_index* ix, const DphSearchPlan& p, const DphCodeSrc& src, int64_t n, bool exact, cudaStream_t st);
// Labels are read through the shard's own layout (ix->blk_off), the codes of the exact re-scoring from `codes`.
int dph_launch_merge(dph_index* ix, const uint8_t* codes, int64_t n, int k, int mode, const int32_t* only_flagged, float* D, int64_t* I,
                     uint32_t* G, cudaStream_t st);
// Dg/Ig/Gg [nshards, n, k] -> D/I [n, k] and, when G is non-null, G [n, k] (0xFFFFFFFF on an empty slot); order score desc, scan
// position asc.
int dph_launch_merge_shards(const float* Dg, const int64_t* Ig, const uint32_t* Gg, int nshards, int64_t n, int k, float* D, int64_t* I,
                            uint32_t* G, cudaStream_t st);
// ---- search.cu ----
// The plan, scan and merge passes of the scan stage over the codes of src (the tables of the chunk are built).
int dph_scan_passes(dph_index* ix, const DphSearchPlan& p, const DphCodeSrc& src, int64_t n, int k, float* D, int64_t* I, uint32_t* G);
// ---- host_codes.cu ----
// Host mode: the scan stage of one chunk, slice by slice (DESIGN.md 3.5).
int dph_host_scan(dph_index* ix, const DphSearchPlan& p, int64_t n, int k, float* D, int64_t* I, uint32_t* G, const uint32_t* mask,
                  const DphQfView* qf);
// Host mode after set_lists: the HBM region (stream only) and the resident table (empty).
int dph_host_lists_ready(dph_index* ix);
// Host mode after a committed mutation: when a list of the shard changed (its length, so its blocks), the resident set empties and
// the whole region serves as the stream region; the largest non-resident list is recomputed either way.
int dph_host_after_mutation(dph_index* ix, bool shard_changed);
// ---- host_move.cu ----
// The in-place re-layout of a host index's page-locked code array (DESIGN.md 3.5, "Mutable host indexes").  prepare() allocates the
// two HBM staging buffers (through `tmp`), streams and events before the caller changes anything.  run() rewrites destination blocks
// [d_first, nw.nblocks) of the new layout nw from the same list's blocks of the committed layout ix->lay (whole, zeros past a list's
// old end), in chunks of whole blocks: descending when no list moves down (add, merge), ascending when none moves up (the remove's
// block shift).  stage(buf, c0, c1, stream), when set, writes the new rows whose destination block is in [c0, c1) into the staged
// chunk buf (block c0 at buf[0]) before it is written back.  Every host write is then a whole-block copy-engine transfer.
struct DphHostMover {
    using StageFn = std::function<int(uint8_t* buf, int64_t c0, int64_t c1, cudaStream_t st)>;
    uint8_t* buf[2] = {};
    cudaStream_t rs = nullptr, ws = nullptr;          // the gather (read) stream and the write-back stream
    cudaEvent_t ev[6] = {};                           // start, end, read[2], write[2]
    int64_t chunk_blocks = 0;
    ~DphHostMover();
    int prepare(dph_index* ix, DevTmp& tmp, int64_t blocks, const char* oom);
    int run(dph_index* ix, const DphLayout& nw, int64_t d_first, const long long* boff_new, bool grow, const StageFn& stage);
};
// The first block of layout nw whose content differs from the committed layout's (nw.nblocks when none): a list's first block when
// it moved, else its old tail block when its length changed.
int64_t dph_first_changed_block(const DphLayout& old, const DphLayout& nw);
// Host mode: rejects (the index unchanged) a layout that needs more blocks than the host array holds.
int dph_host_capacity_check(const dph_index* ix, const DphLayout& nw, const char* what);
// Whether a list of the shard has another length in nw than in the committed layout.
bool dph_shard_changed(const dph_index* ix, const DphLayout& nw);
// ---- lists.cu ----
__global__ void fill_blocks_kernel(uint8_t* codes, long long nblocks, const long long* blk_off, const int* list_len, long long list_lo,
                                   long long list_hi, const uint8_t* raw, const long long* local_row_start, uint64_t seed, long long blk0,
                                   long long raw_row0, long long out0);
// ---- encode.cu ----
int64_t dph_encode_chunk(const dph_index* ix);
int dph_encode_rows(dph_index* ix, const float* x_dev, int64_t n, int64_t* list_out, uint8_t* codes_out, int* bad);
// The input stage of add_int8: rows x = q / scale + offset of int8 q [n, d] (mem: device, or host, page-locked read in place or
// pageable staged as int8) dequantised chunk by chunk into xdev, then dph_encode_rows.
int dph_encode_int8(dph_index* ix, const int8_t* q, int64_t n, float offset, float scale, int mem, int64_t* list_out, uint8_t* codes_out,
                    int* bad);
// Top-1 coarse list of n <= dph_encode_chunk rows xr [n, d] against centroids C [nlist, d]: the encoding's assignment (tensor-core
// candidates + exact re-rank where the shape allows, else the SIMT sequential-k GEMM; smallest list id on a tie).  ix->S must hold
// the n x nlist (padded to 128) scores.  key [n] int32, cd [n] the top-1 score.
int dph_coarse_top1(dph_index* ix, const float* xr, const float* C, int64_t n, int32_t* key, float* cd, cudaStream_t st);
// PQ codes [n, 96] of the residuals xr - C[key] under the codebooks pq (pq_encode_kernel); list_out [n] int64 receives key.
int dph_pq_assign(dph_index* ix, const float* xr, const float* C, const int32_t* key, const float* pq, int64_t n, int64_t* list_out,
                  uint8_t* codes_out, cudaStream_t st);
__global__ void nonfinite_kernel(const float* __restrict__ x, long long count, int* __restrict__ bad);
