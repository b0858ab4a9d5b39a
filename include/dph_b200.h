/*
 * dph_b200.h -- C ABI of libdph_b200.so: the H100-native (sm_90a) replacement for the FAISS calls on the
 * DensePhrases retrieval hot path.  Plain pointers and sizes only (no torch / faiss types).
 *
 * Every entry point names the reference interface it replaces (paths relative to the reference DensePhrases repository):
 *
 *   dph_index_search            <- faiss.IndexPreTransform.search(x, k)      densephrases/index.py:200
 *   dph_index_reconstruct_batch <- faiss IndexIVFPQ.reconstruct(id) per id   densephrases/index.py:31,282-300
 *   dph_index_get_opq           <- faiss.vector_to_array(OPQMatrix.A)        densephrases/index.py:32
 *   dph_index_ntotal/d/nlist    <- index.ntotal / index.d / index_ivf.nlist  densephrases/index.py:33,128-133
 *   dph_index_set_nprobe        <- index_ivf.nprobe = 256                    densephrases/index.py:53,62
 *   dph_index_create/set_*      <- faiss.read_index(...) / IndexPreTransform(OPQMatrix, IndexIVFPQ(...))
 *                                  densephrases/index.py:30 ; build_phrase_index.py:113-116,149-150
 *   dph_index_add_with_ids      <- index.add_with_ids(vectors, ids)          build_phrase_index.py:145-150,156-279
 *   dph_index_add_int8          <- index.add_with_ids(int8_to_float(start, offset, scale), ids)   build_phrase_index.py:207-226
 *   dph_index_encode            <- the assignment + PQ encoding inside add_with_ids (IndexIVFPQ::encode_vectors)
 *   dph_index_copy_lists        <- the inverted lists faiss.write_index stores (invlists->get_codes / get_ids)
 *   dph_index_remove_ids        <- index.remove_ids(IDSelectorBatch(ids) | IDSelectorRange(lo, hi)) (faiss 1.6.x IndexIVF)
 *   dph_filter_create           <- faiss.SearchParametersIVF(sel=IDSelectorBatch | IDSelectorRange | IDSelectorNot) (faiss >= 1.7.3)
 *   dph_index_sync_list_len     <- (sharded remove) the list lengths faiss keeps in one process, exchanged between shards
 *   dph_index_merge_from        <- invlists.merge_from(sub_index.invlists, offset)            build_phrase_index.py:282-338
 *   dph_index_train_coarse      <- the coarse quantizer's k-means inside index.train(x)   build_phrase_index.py:96-142
 *   dph_index_train_pq          <- ProductQuantizer::train inside index.train(x) (and OPQMatrix::train's PQ)
 *   dph_index_encode_pq         <- OPQMatrix::train's pq_regular.compute_codes (PQ codes without a coarse residual)
 *   dph_index_get_centroids/pq  <- the trained tables faiss.write_index stores
 *
 * Conventions: every function returns 0 on success, non-zero on error (dph_last_error() gives the
 * message; the Python layer raises RuntimeError like faiss' SWIG layer does).  `mem` arguments say
 * where caller buffers live.  All device work is issued on the stream passed to dph_index_set_stream
 * (default: the legacy default stream).  Calls with host buffers are synchronous; calls with device
 * buffers are asynchronous on that stream.  Inputs are never modified.
 */
#ifndef DPH_B200_H
#define DPH_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define DPH_MEM_HOST 0
#define DPH_MEM_DEVICE 1

/* scan kernel selection (dph_index_set_scan_mode) */
#define DPH_SCAN_FAST 0   /* default: conflict-free gather filter + proof + exact fp32 re-scoring; picks QUAD / PAIR / SINGLE per batch */
#define DPH_SCAN_EXACT 1  /* canonical-order fp32 ADC for every code (slow; fallback + cross-check) */
#define DPH_SCAN_PAIR 2   /* force: two queries share every gather (int16-packed quantised LUTs), lists grouped by probing queries */
#define DPH_SCAN_SINGLE 3 /* force: one query per gather (fp32 LUT) */
#define DPH_SCAN_QUAD 4   /* force: four queries share every gather (int8-packed quantised LUTs), lists grouped by probing queries */

typedef struct dph_index dph_index;

const char* dph_last_error(void);
int dph_version(void);

/* ---- construction (replaces faiss.read_index / index build; build_phrase_index.py:113-116) ---- */
/* d = M*dsub, nbits must be 8 (ksub 256), M must be 96 (PQ96: code row = 96 bytes). */
int dph_index_create(dph_index** out, int d, int64_t nlist, int M, int nbits, int device);
void dph_index_free(dph_index* ix);
int dph_index_set_stream(dph_index* ix, void* cuda_stream);
/* OPQ matrix A [d,d] row-major (d_out rows), centroids [nlist,d], PQ codebooks [M,256,dsub]; fp32. */
int dph_index_set_opq(dph_index* ix, const float* A, int mem);
int dph_index_set_centroids(dph_index* ix, const float* C, int mem);
int dph_index_set_pq(dph_index* ix, const float* pq, int mem);
/* Synthetic centroids/PQ (bit-identical to oracle ref_gen_centroids / ref_gen_pq), generated on device. */
int dph_index_gen_centroids(dph_index* ix, uint64_t seed, float sigma);
int dph_index_gen_pq(dph_index* ix, uint64_t seed, float sigma);
/* This process holds only inverted lists [list_lo, list_hi) (list-range shard, SURVEY 8e). Call before set_lists. */
int dph_index_set_shard(dph_index* ix, int64_t list_lo, int64_t list_hi);
/* list_len [nlist] (ALL lists, host). codes: [ntotal,96] list-major rows of the lists in the shard only
 * (host), ids likewise [ntotal_shard] or NULL for sequential labels (label = global list-major row,
 * build_phrase_index.py:149-150). */
int dph_index_set_lists(dph_index* ix, const int64_t* list_len, const uint8_t* codes, const int64_t* ids);
/* Same but codes are generated on device from `seed` (bit-identical to oracle ref_gen_codes); ids sequential. */
int dph_index_set_lists_synthetic(dph_index* ix, const int64_t* list_len, uint64_t seed);

/* ---- growing the index (replaces index.add_with_ids, build_phrase_index.py:145-150,156-279; DESIGN.md 3 "Growing the index") ----
 * Encoding is IndexPreTransform(OPQ) -> IndexIVFPQ (by_residual) with a fixed fp32 order, bit-identical to the oracle's ref_encode:
 * rotation, top-1 coarse list (smallest list id on a tie), fp32 residual, per sub-quantizer squared-L2 as one fmaf chain, lowest
 * codeword on a tie.  Needs the OPQ matrix, centroids and PQ codebooks.  Uses the search workspace: dph_index_last_xr is not kept. */
/* x [n,d] -> list_no_out [n] int64, codes_out [n,96] uint8 (m ascending); the index is not modified. */
int dph_index_encode(dph_index* ix, const float* x, int64_t n, int64_t* list_no_out, uint8_t* codes_out, int mem);
/* Append x [n,d] with labels ids [n] (NULL -> ntotal + i, like IndexIVF::add) to their lists, in input order; needs set_lists first
 * (all-zero list lengths give an empty, trained index).  The device state afterwards is byte-identical to set_lists of the
 * concatenated list-major arrays.  On a shard, rows of lists outside [list_lo, list_hi) only count into the list lengths: every rank
 * that adds the same batch reaches the same global state.  An index with sequential labels turns them into explicit ones.  A label
 * added twice is found at every row that carries it; reconstruct returns the most recent row (faiss' hashtable direct map), except
 * for a label repeated across shards, which reconstruct leaves undefined.  Rejected, with the index unchanged: a negative label, a
 * non-finite input value, too little device memory for the old and the new code buffers at once (a host index with a reserved
 * capacity: for two staging buffers), a host index whose capacity the new layout exceeds.  Synchronises the stream. */
int dph_index_add_with_ids(dph_index* ix, const float* x, int64_t n, const int64_t* ids, int mem);
/* add_with_ids of the rows x = fl32(fl32(q / scale) + offset) of int8 q [n,d] (a phrase dump's `start` rows with its group's offset and
 * scale attributes cast to fp32): byte-identical to add_with_ids of those fp32 rows.  mem DPH_MEM_DEVICE: q and ids are device
 * pointers.  DPH_MEM_HOST: page-locked q is read in place through its device mapping, pageable q through a bounded device staging
 * chunk of int8; no fp32 copy of the rows is made on the host.  q may start at any byte offset.  Rejected, with the index
 * unchanged: scale zero or not finite, offset not finite, and every case add_with_ids rejects.  Synchronises the stream. */
int dph_index_add_int8(dph_index* ix, const int8_t* q, int64_t n, float offset, float scale, const int64_t* ids, int mem);
/* This shard's lists as list-major host arrays: codes_out [ntotal_local,96], ids_out [ntotal_local] (may be NULL); the inverse of
 * set_lists, for writing a grown index back to a faiss file (artifacts.write_faiss_index). */
int dph_index_copy_lists(dph_index* ix, uint8_t* codes_out, int64_t* ids_out);
/* list_len_out [nlist] (host): the length of every list, all shards. */
int dph_index_get_list_len(const dph_index* ix, int64_t* list_len_out);
/* Measurement hook: with profiling on, the stage times of the last add in ms: rotation, coarse, PQ encode, re-layout + scatter. */
int dph_index_last_add_ms(const dph_index* ix, float* ms_out /* [4] */);

/* ---- codes in host memory (DESIGN.md 3.5 "Codes in host memory") ----
 * on_host = 1: set_lists / set_lists_synthetic put the shard's code blocks in page-locked, device-mapped host memory (same 32-row block
 * layout); labels, direct map, list tables and model tables stay in device memory.  Device memory holds two code regions: the resident
 * lists (dph_index_set_resident_lists) and a stream region of stream_bytes (rounded down to whole 3 KB blocks).  Each search chunk is
 * scanned in slices: the probed lists in ascending id, a new slice whenever the next non-resident list would overflow the stream region;
 * a slice's non-resident probed lists are copied into the stream region and scanned, and the slices' partial top-k are merged (score
 * desc, scan position asc).  Results are bit-identical to the same index in device memory.  A search is rejected when the stream region
 * is smaller than the shard's largest non-resident list.  Host mode costs one copy of the probes to the host and one synchronisation
 * per search chunk.  Without a reserved host capacity (dph_index_reserve_host_codes) it is read-only after set_lists: add_with_ids,
 * remove_ids, sync_list_len and merge_from are rejected with the index unchanged; it is never a merge source.  on_host must be chosen
 * before set_lists (like set_shard); stream_bytes may be changed later (the region is reallocated, resident lists kept); on_host = 0
 * needs stream_bytes = 0.  set_lists drops the resident set. */
int dph_index_set_code_residency(dph_index* ix, int on_host, int64_t stream_bytes);
/* Host mode, after set_lists: copy lists [n] (this shard's; any order, duplicates ignored) into an exact-size device region that replaces
 * the previous resident set (n = 0 empties it).  Rejected, with the index unchanged: a list outside [list_lo, list_hi), too little device
 * memory for the new resident region next to the old one.  Synchronises the stream. */
int dph_index_set_resident_lists(dph_index* ix, const int64_t* lists, int64_t n);
/* Host mode: what the last search call fetched, summed over its chunks: counts [4] = slices, lists fetched, blocks fetched, resident
 * lists scanned; ms (may be NULL) = time of its fetch kernels with profiling on (0 otherwise). */
int dph_index_last_fetch(const dph_index* ix, int64_t* counts, float* ms);
/* Bytes of page-locked host memory holding the codes (0 unless host mode). */
int64_t dph_index_host_bytes(const dph_index* ix);
/* Host mode: reserve a host capacity of bytes (rounded down to whole 3 KB blocks), which makes the index mutable.  add_with_ids,
 * remove_ids, sync_list_len and merge_from (from device-resident sources) then behave exactly as on a device-resident index, re-laying
 * the page-locked array in place through two HBM staging buffers (DESIGN.md 3.5 "Mutable host indexes"); an add or merge whose layout
 * needs more than the capacity is rejected with the index unchanged.  A mutation that changes a list of the shard empties the
 * resident set: the region keeps its size and serves as the stream region until dph_index_set_resident_lists is called again.
 * Before set_lists: set_lists allocates max(capacity, its blocks).  After: a larger capacity allocates a new page-locked array, copies
 * the blocks and frees the old one (the only time two host arrays exist; rejected with the index unchanged if the allocation fails);
 * a capacity at or below the allocation only makes the index mutable.  The capacity never shrinks.  Synchronises the stream. */
int dph_index_reserve_host_codes(dph_index* ix, int64_t bytes);
/* Host mode, measurement hook: the last add, remove or merge's in-place block mover: counts [3] = blocks read from the host array,
 * blocks written to it, staging chunks; ms (may be NULL) = its time from the first gather to the last write-back. */
int dph_index_last_host_move(const dph_index* ix, int64_t* counts, float* ms);

/* ---- removing vectors (replaces index.remove_ids(faiss.IDSelectorBatch(ids)) / remove_ids(faiss.IDSelectorRange(lo, hi)) of faiss
 * 1.6.x IndexIVF; DESIGN.md 3.2 "Removing vectors") ----
 * Selector: the label set ids [n_ids] (mem says where it lives; any order, duplicates allowed, absent or negative labels match nothing)
 * when ids is non-NULL, with range_lo = range_hi = 0; else the label range [range_lo, range_hi), with n_ids = 0.  Every row of this
 * shard whose label is selected is removed.  Each list keeps the survivors in the order of faiss' IndexIVF::remove_ids loop without a
 * direct map (the last row fills each hole); the device state afterwards is byte-identical to set_lists of the resulting list-major
 * arrays.  An empty selector (n_ids == 0, or range_lo >= range_hi) changes nothing; any other turns sequential labels into explicit
 * ones, as the first add does.  The shard compacts in place: extra device memory is one staging buffer of <= ~256 MB plus
 * O(nlist + n_ids + rows removed), and 24 B per row for an index that gains labels; the code allocation is not shrunk.  Rejected,
 * with the index unchanged: n_ids < 0, both or neither selector forms, too little device memory for those buffers.
 * n_removed_out: rows removed from this shard; removed_per_list_out [nlist] (host, may be NULL): per list, zero outside the shard.
 * On a shard, the lengths of other shards' lists are left as they were: see dph_index_sync_list_len.  Synchronises the stream. */
int dph_index_remove_ids(dph_index* ix, const int64_t* ids, int64_t n_ids, int64_t range_lo, int64_t range_hi, int mem,
                         int64_t* n_removed_out, int64_t* removed_per_list_out);
/* Sharded remove (sharded.py): after every shard removed the same selector, list_len [nlist] (host) = the old lengths minus the
 * all-reduced per-list counts.  Sets the lengths (and list starts, which order ties in the sharded merge) of the lists outside
 * [list_lo, list_hi); refuses, with the index unchanged, when an entry of this shard differs from its own length, or when other lists
 * change on a shard whose labels are still sequential (they would move). */
int dph_index_sync_list_len(dph_index* ix, const int64_t* list_len);
/* Measurement hooks: with profiling on, the stage times of the last remove in ms: mark + plan, row moves + block shift, direct map;
 * and the largest total of its temporary device allocations in bytes (the device sorts' own scratch not included).  A call with an
 * empty selector resets both to zero. */
int dph_index_last_remove_ms(const dph_index* ix, float* ms_out /* [3] */);
int64_t dph_index_last_remove_tmp_bytes(const dph_index* ix);

/* ---- merging indexes (replaces the merge stage of build_phrase_index.py:282-338: invlists.merge_from of every sub-index, and
 * faiss IndexIVF::merge_from(other, add_id); DESIGN.md 3.4 "Merging indexes") ----
 * Appends the rows of the n_src sources src[0 .. n_src) to this index: for every list l the result holds this index's rows, then
 * source 0's rows of l, then source 1's, and so on, each in its stored order.  A source row's label is its stored label (sequential:
 * list_start_src[l] + j) plus add_id.  The device state afterwards is byte-identical to set_lists of the concatenated list-major
 * arrays.  The sources are not modified (faiss empties `other`).  An index with sequential labels turns them into explicit ones on any
 * merge that adds rows; the direct map is the stable merge of this index's map and each source's map in argument order, so
 * reconstruct returns the latest source's row of a label present twice.  Sources with no rows make the call a no-op.  On a shard,
 * every source must hold the same list range; the other lists' rows only count into the list lengths, so every rank merging its
 * shards of the same sources reaches the same global state.  Rejected, with the index unchanged: a source with another d, nlist, M,
 * device or shard range, or whose OPQ matrix, centroids or PQ codebooks differ in any bit (compared on the device); this index as its
 * own source; a label + add_id that is negative or overflows; a list longer than 2^31 - 1 rows; too little device memory for the old
 * and the new code, label and direct-map buffers of the shard at once (the peak of an add).  Synchronises the streams of this index
 * and of the sources. */
int dph_index_merge_from(dph_index* ix, const dph_index* const* src, int n_src, int64_t add_id);
/* Measurement hook: with profiling on, the stage times of the last merge in ms: plan + alloc, block moves, source rows, direct map. */
int dph_index_last_merge_ms(const dph_index* ix, float* ms_out /* [4] */);

/* ---- training (replaces index.train(x) of build_phrase_index.py:96-142: faiss Clustering with cp.spherical over IndexFlatIP and
 * ProductQuantizer::train on residuals; DESIGN.md 3.3 "Training the index") ----
 * The trained tables are bit-identical to the oracle's ref_train_coarse / ref_train_pq: a sample of at most max_points_per_centroid
 * x k rows drawn from rnd64(seed, ...), rotated by the handle's OPQ matrix; init from sample rows ranked by rnd64 (unless hot_start,
 * which starts from the handle's current table); per iteration the encoding's own assignment, per-cluster sums in ascending row order,
 * faiss' split of empty clusters with the repo's draws, and (coarse) renormalisation to unit norm.  x [n, d] fp32 (mem: host or
 * device).  Only the rotated sample stays on the device.  Rejected, with the index unchanged: a handle that holds vectors, no OPQ
 * matrix, n < k (nlist, or 256 for the PQ), a non-finite value in a sampled row, too little device memory for the sample and the
 * workspace; hot start without the table, train_pq with residual = 1 without centroids.  Synchronise the stream. */
/* Coarse centroids [nlist, d]: niter iterations of spherical k-means (faiss' IVF default 10).  obj_out [niter] (may be NULL): the sum
 * of the assigned inner products in fp64 before each update; nsplit_out [niter] (may be NULL): empty clusters re-seeded by a split. */
int dph_index_train_coarse(dph_index* ix, const float* x, int64_t n, int niter, uint64_t seed, int64_t max_points_per_centroid,
                           int hot_start, int mem, double* obj_out, int64_t* nsplit_out);
/* PQ codebooks [96, 256, 8]: 96 independent L2 k-means of niter iterations (faiss default 25), assignment = the encoding's argmin.
 * residual = 1: on xr - C[top-1 list] (IndexIVFPQ by_residual); 0: on xr itself (OPQ's PQ). */
int dph_index_train_pq(dph_index* ix, const float* x, int64_t n, int niter, uint64_t seed, int64_t max_points_per_centroid,
                       int hot_start, int residual, int mem);
/* codes_out [n, 96] = PQ codes of x A^T without a coarse residual (the encoding's argmin, lowest codeword on a tie). */
int dph_index_encode_pq(dph_index* ix, const float* x, int64_t n, uint8_t* codes_out, int mem);
/* Read the tables back (for artifacts.write_faiss_index / save_container): C_out [nlist, d], pq_out [96, 256, 8]. */
int dph_index_get_centroids(const dph_index* ix, float* C_out, int mem);
int dph_index_get_pq(const dph_index* ix, float* pq_out, int mem);
/* Measurement hook: with profiling on, the stage times of the last train_coarse / train_pq in ms, summed over its iterations:
 * assignment, sort + update, split + renorm. */
int dph_index_last_train_ms(const dph_index* ix, float* ms_out /* [3] */);

/* ---- getters ---- */
int64_t dph_index_ntotal(const dph_index* ix);       /* all shards */
int64_t dph_index_ntotal_local(const dph_index* ix); /* this shard */
int dph_index_d(const dph_index* ix);
int64_t dph_index_nlist(const dph_index* ix);
int dph_index_nprobe(const dph_index* ix);
int dph_index_set_nprobe(dph_index* ix, int nprobe);
int dph_index_set_scan_mode(dph_index* ix, int mode);
/* Coarse quantizer on the tensor cores (3xTF32 candidate pass + exact sequential-FMA re-rank + proof; bit-identical probes).
 * 1 (default): used when the shape allows (lists % 128 == 0, batch >= 32, nprobe + margin <= 1024); 0: always the exact SIMT GEMM. */
int dph_index_set_coarse_tc(dph_index* ix, int on);
int dph_index_get_opq(const dph_index* ix, float* A_out, int mem);
/* Bytes of the index's resident arrays (model tables, lists, labels, direct map; in host mode the resident and stream regions instead
 * of the codes), without the per-batch workspace. */
int64_t dph_index_device_bytes(const dph_index* ix);
/* Measurement hook: when on, CUDA events bracket the scan kernel of each search (last chunk); last_scan_ms waits
 * for it and returns the kernel's duration in milliseconds (bench.py roofline). */
int dph_index_set_profile(dph_index* ix, int on);
int dph_index_last_scan_ms(dph_index* ix, float* ms);
/* Durations of the scan kernels of the last (up to 64) searches since profiling was switched on, oldest first;
 * dph_index_profile_count gives how many.  Lets bench.py time the kernel inside a back-to-back step loop. */
int dph_index_profile_scan_ms(dph_index* ix, float* ms_out, int max_out);
int dph_index_profile_count(const dph_index* ix);

/* ---- search (replaces index.search at index.py:200) ----
 * x [n,d] fp32; D [n,k] fp32, I [n,k] int64 labels; sorted by descending score; unfilled slots are
 * (-FLT_MAX, -1) like faiss' CMin heap.  Uses the index's nprobe (default 256, index.py:53,62). */
int dph_index_search(dph_index* ix, const float* x, int64_t n, int k, float* D, int64_t* I, int mem);
/* Sharded search: per-shard partial top-k.  G [n,k] uint32 = canonical scan position (tie-break key,
 * global over all shards).  Buffers on device.  After an all-gather over shards feed dph_merge_shards. */
int dph_index_search_partial(dph_index* ix, const float* x_dev, int64_t n, int k, float* D_dev, int64_t* I_dev,
                             uint32_t* G_dev);
/* Sharded coarse quantizer (scales the IndexFlatIP coarse search with the number of shards): every shard scores only its own
 * lists' centroids and emits its best nprobe as keys (score key << 32 | ~global list id, 0 = empty) [n,nprobe];
 * after an all-gather of the keys [nshards,n,nprobe], search_preassigned merges them into the global top-nprobe (identical to
 * the unsharded selection) and runs the rest of the search on this shard's lists.  n must fit one chunk (<= 4096). */
int dph_index_coarse_local(dph_index* ix, const float* x_dev, int64_t n, uint64_t* keys_dev);
int dph_index_search_preassigned(dph_index* ix, const uint64_t* keys_gathered_dev, int nshards, int64_t n, int k, float* D_dev,
                                 int64_t* I_dev, uint32_t* G_dev);
/* Query-split variant of the same step (large batches): every shard rotates and assigns only ITS SLICE of the batch (n_local queries),
 * but over ALL lists (the coarse quantizer is replicated, index.py:200 runs it once per batch), and emits one record per query:
 * rec [n_local, dph_index_record_floats()] = [768 f32 rotated query | nprobe i32 list numbers | nprobe f32 coarse scores].  After an
 * all-gather of the records, search_assigned (rec [n, ...], all queries in batch order) runs the rest of the search on this shard's
 * lists.  Same probes and scores as the unsharded search; the rotation and the exact re-rank of the tensor-core coarse quantizer are
 * done once per query instead of once per query and shard.  Records and candidate keys are an exchange format between ranks running
 * THIS library on replicas of the same coarse quantizer: list numbers inside them are trusted, not validated (a caller that
 * fabricates them must keep them in [-1, nlist)). */
int dph_index_record_floats(const dph_index* ix);
int dph_index_coarse_split(dph_index* ix, const float* x_dev, int64_t n_local, float* rec_dev);
int dph_index_search_assigned(dph_index* ix, const float* rec_dev, int64_t n, int k, float* D_dev, int64_t* I_dev, uint32_t* G_dev);
/* Dg/Ig/Gg [nshards,n,k] (all-gathered, device) -> D/I [n,k] (device).  Order: score desc, scan position asc. */
int dph_merge_shards(const float* Dg, const int64_t* Ig, const uint32_t* Gg, int nshards, int64_t n, int k, float* D,
                     int64_t* I, void* cuda_stream);
/* Same exchange as ONE buffer: pack (D, I, G) [n,k] into P [n,k,2] int64 = {candidate key (score, scan position), label};
 * all-gather P; merge Pg [nshards,n,k,2] -> D/I [n,k]. */
int dph_pack_topk(const float* D, const int64_t* I, const uint32_t* G, int64_t n, int k, int64_t* P, void* cuda_stream);
int dph_merge_shards_packed(const int64_t* Pg, int nshards, int64_t n, int k, float* D, int64_t* I, void* cuda_stream);

/* ---- filtered search (replaces index.search(x, k, params=faiss.SearchParametersIVF(sel=IDSelectorBatch(ids) |
 * IDSelectorRange(lo, hi) | IDSelectorNot(...))), faiss >= 1.7.3; DESIGN.md 3.6 "Filtered search") ----
 * A filter is a row mask of one shard: one uint32 per 32-row code block, bit l = lane l's row is selected.  A search with a filter set
 * (dph_index_set_filter) has the same probes as without it; every probed row whose label is not selected is skipped before it can
 * become a candidate, so its result is the unfiltered canonical ranking of the probed rows restricted to the selected ones, cut at k
 * (short results padded with (-FLT_MAX, -1)).  A row is selected exactly when its label is. */
typedef struct dph_filter dph_filter;
/* Selector forms and rejections as dph_index_remove_ids: the label set ids [n_ids] (mem says where it lives; any order, duplicates
 * allowed, absent or negative labels match nothing) with range_lo = range_hi = 0, or the label range [range_lo, range_hi) with ids =
 * NULL and n_ids = 0.  exclude != 0 selects every real row whose label is NOT in the selector (padding rows never).  The index is not
 * changed (sequential labels stay sequential).  The mask is built on the device and owned by the filter (dph_index_device_bytes does
 * not count it).  It belongs to ix and to ix's current list layout: after set_lists, add, remove, merge or sync_list_len on ix a
 * search with it is rejected until it is rebuilt.  Synchronises the stream. */
int dph_filter_create(dph_filter** out, dph_index* ix, const int64_t* ids, int64_t n_ids, int64_t range_lo, int64_t range_hi, int exclude,
                      int mem);
/* Frees the mask; a filter set on its index is cleared there.  Free a filter before its index. */
void dph_filter_free(dph_filter* f);
int64_t dph_filter_rows(const dph_filter* f);            /* selected rows of the shard */
int64_t dph_filter_bytes(const dph_filter* f);           /* device bytes of the mask */
/* The mask [nblocks of the shard] uint32 into host memory (block order of the shard's code array). */
int dph_filter_copy_mask(const dph_filter* f, uint32_t* out_host);
/* Applies f (NULL clears) to every later search of ix -- dph_index_search, search_partial, search_preassigned, search_assigned -- like
 * dph_index_set_nprobe.  Rejected when f was built for another index.  A search with a stale filter is rejected. */
int dph_index_set_filter(dph_index* ix, const dph_filter* f);

/* ---- per-query filters (a different IDSelector per query of one batch; DESIGN.md 3.7 "Per-query filters") ----
 * A query filter holds nsel label selectors and the selector assign[q] of each of the n queries of one batch (-1: the query is not
 * filtered).  A search of those n queries with it set (dph_index_set_query_filter) computes row q exactly as the search of query q alone
 * with the row mask of its selector (dph_filter_create, exclude = 0), or unfiltered for -1: D bits and I.  Each selector is held sparse:
 * per list of the shard, the ascending numbers of the list's blocks that hold a selected row, with their mask words -- 8 bytes per
 * selected block, plus a 4-byte offset per list of the shard per selector.  Selector s is the label set labels[label_off[s] ..
 * label_off[s + 1]) (labels in `mem`; any order, duplicates allowed, absent or negative labels match nothing), or, when ranges is not
 * NULL and (ranges[2s], ranges[2s + 1]) != (0, 0), the label range [ranges[2s], ranges[2s + 1]) -- not both; neither selects nothing.
 * label_off [nsel + 1], ranges [2 nsel] and assign [n] are host arrays; label_off may be NULL when every selector is a range.
 * Rejected (nothing created) when an assign entry is outside [-1, nsel) or a selector has both forms.  Built on the device in one
 * call for all selectors; the index is not changed.  It belongs to ix and ix's current list layout, as a dph_filter does.
 * Synchronises the stream.  exclude has no per-query form: use a dph_filter for it. */
typedef struct dph_query_filter dph_query_filter;
int dph_query_filter_create(dph_query_filter** out, dph_index* ix, const int64_t* labels, const int64_t* label_off, const int64_t* ranges,
                            int64_t nsel, const int32_t* assign, int64_t n, int mem);
void dph_query_filter_free(dph_query_filter* f);          /* a query filter set on its index is cleared there */
int64_t dph_query_filter_bytes(const dph_query_filter* f);                  /* device bytes of the filter */
int64_t dph_query_filter_rows(const dph_query_filter* f, int64_t s);        /* selected rows of the shard by selector s */
int64_t dph_query_filter_blocks(const dph_query_filter* f, int64_t s);      /* blocks held for selector s */
/* Selector s's CSR into host memory: off [lists of the shard + 1] (list lo + i's entries are [off[i], off[i + 1])), blk and word
 * [dph_query_filter_blocks(f, s)]: the list's block number and its mask word. */
int dph_query_filter_copy_selector(const dph_query_filter* f, int64_t s, uint32_t* off_out, uint32_t* blk_out, uint32_t* word_out);
/* Applies f (NULL clears) to every later search of ix, as dph_index_set_filter; it replaces a dph_filter set on ix (and that one
 * replaces it).  A search whose batch is not f's n queries is rejected, and so is one with a stale filter. */
int dph_index_set_query_filter(dph_index* ix, const dph_query_filter* f);

/* Per-query flags of the last search (device pointer, int32 [n]): bit0 = fast filter could not prove
 * exactness and the query was re-run through the exact kernel. */
const int32_t* dph_index_last_flags(const dph_index* ix);
/* Intermediate results of the last search, for tests (device pointers): probed lists [n,nprobe] int32,
 * coarse scores [n,nprobe] fp32, rotated queries [n,d]. */
const int32_t* dph_index_last_probes(const dph_index* ix);
const float* dph_index_last_coarse(const dph_index* ix);
const float* dph_index_last_xr(const dph_index* ix);
int dph_index_last_used_pair_mode(const dph_index* ix);   /* 1 when the last search shared gathers between queries (pair or quad) */
int dph_index_last_group_size(const dph_index* ix);       /* queries per gather of the last search: 1, 2 or 4 */
/* Copy one of them to the host (synchronises): which = 0 flags, 1 probes, 2 coarse scores, 3 rotated queries. */
int dph_index_copy_last(dph_index* ix, int which, void* dst_host, int64_t bytes);

/* ---- reconstruct (replaces reconst_fn loop, index.py:282-300) ----
 * out [m,d] fp32 in ROTATED space (caller un-rotates with R = OPQ matrix, index.py:340,365);
 * found [m] u8: 0 -> label not in this shard / not in the index, row is zeros (index.py:287-288). */
int dph_index_reconstruct_batch(dph_index* ix, const int64_t* ids, int64_t m, float* out, uint8_t* found, int mem);

/* ---- phrase re-scoring (replaces index.py:323-371: end.matmul(R); (q*end).sum; argmax with mask) ----
 * For each of m hits: window of L consecutive labels starting at first_id[i]; score[i,l] =
 * <q[i], R^T-unrotated reconstruct(first_id[i]+l)> computed as <A q[i] , reconstruct> (A orthonormal);
 * out_scores [m,L] fp32 (missing label -> 0, like the zero vector at index.py:287-288). */
int dph_index_window_scores(dph_index* ix, const float* q /*[m,d]*/, const int64_t* first_id /*[m]*/, int64_t m, int L,
                            float* out_scores, int mem);

/* ---- encoder (replaces Encoder.forward(return_query=True) -> embed_query, densephrases/encoder.py:146-152,101-118, and
 * Encoder.forward(input_ids=..., return_phrase=True) -> embed_phrase + filter_linear, encoder.py:92-99,130-144) ----
 * BERT-base towers (12 layers, 768 hidden, 12 heads, 3072 FFN; SpanBERT-base-cased geometry, options.py:23).
 * tower 0 = query_start_encoder.*, tower 1 = query_end_encoder.*, tower 2 = phrase_encoder.* (encoder.py:50-52).  Weight blob
 * layout: encoder.cu.  An encoder needs only the towers of the calls it serves. */
typedef struct dph_encoder dph_encoder;
int dph_encoder_create(dph_encoder** out, int device, int vocab_size, int max_position_embeddings, int type_vocab_size);
void dph_encoder_free(dph_encoder* e);
int dph_encoder_set_stream(dph_encoder* e, void* cuda_stream);
int64_t dph_encoder_tower_floats(const dph_encoder* e);
int dph_encoder_load_tower(dph_encoder* e, int tower, const float* blob, int mem);
/* filter_linear (encoder.py:32): weight fp32 [2,768], bias fp32 [2] */
int dph_encoder_load_filter(dph_encoder* e, const float* weight, const float* bias, int mem);
/* 0 (default): GEMMs as one TF32 MMA per product -- what torch 1.9 (the reference's pin) does for fp32 matmuls on Ampere+;
 * 1: 3xTF32 split GEMMs, fp32-accurate (matches the reference's CPU/fp32 path to ~1e-5);
 * 2: bf16x3 split GEMMs (operands as (hi, lo) bf16 planes, three kind::f16 MMAs per product, ~2^-17 relative): meets the 1e-3
 *    tolerance on the query vectors at the speed of mode 0. */
int dph_encoder_set_precision(dph_encoder* e, int precise);
/* 1 (default): self-attention on the tensor cores -- S <= 64 on both paths, every S on the phrase path (key blocks streamed with an
 * online softmax above 64); TF32 operands in precision mode 0, bf16 (hi, lo) planes with three MMAs per contraction (fp32-accurate)
 * in modes 1 and 2; fp32 accumulation and softmax.  0: always the fp32 SIMT attention kernels (S <= 384). */
int dph_encoder_set_attention(dph_encoder* e, int tensor_core);
/* One BERT-base self-attention (12 heads x 64; HF BertSelfAttention as used by encoder.py:101-118) on device buffers:
 * qkv fp32 [B*S, 2304] = (Q | K | V), mask int64 [B,S] -> ctx fp32 [B*S, 768].  tensor_core: 0 SIMT fp32, 1 wgmma TF32,
 * 2 wgmma on bf16 (hi, lo) operand planes, three MMAs per contraction (fp32-accurate); S <= 512 for 1 and 2, S <= 384 for 0. */
int dph_attention_bert(const float* qkv, const int64_t* attention_mask, int B, int S, float* ctx, int tensor_core, void* cuda_stream);
/* input_ids / attention_mask / token_type_ids int64 [B,S] (S <= 384); start_out / end_out fp32 [B,768] = hidden state at
 * position 0 of each tower (the reference returns them as [B,1,768]). */
int dph_encoder_embed_query(dph_encoder* e, const int64_t* input_ids, const int64_t* attention_mask, const int64_t* token_type_ids,
                            int B, int S, float* start_out, float* end_out, int mem);
/* input_ids / attention_mask / token_type_ids int64 [B,S] (S <= min(512, max_position_embeddings), B <= 65535); out fp32 [B,S,768] = the
 * phrase tower's last hidden state (the reference's start == end); filter_out (nullable) fp32 [B,S,2] = filter_linear(out) as
 * (start logit, end logit).  Host buffers: synchronous; device buffers: asynchronous on the encoder's stream. */
int dph_encoder_embed_phrase(dph_encoder* e, const int64_t* input_ids, const int64_t* attention_mask, const int64_t* token_type_ids,
                             int B, int S, float* out, float* filter_out, int mem);
/* Encoder.forward with a context and a question (encoder.py:120-153, 206-208, 260): context ids / mask / token types int64 [B,S]
 * (S <= min(512, max_position_embeddings), B <= 65535), question ids / mask / token types int64 [B,Sq] (Sq <= 384) ->
 * start_out, end_out fp32 [B,S] = each token's phrase vector . its question's q_start / q_end, filter_out fp32 [B,S,2] = the
 * filter head as in dph_encoder_embed_phrase (bit-identical).  The [B,S,768] phrase vectors are never written.  Needs all three
 * towers and the filter head.  Host buffers: synchronous; device buffers: asynchronous on the encoder's stream. */
int dph_encoder_read(dph_encoder* e, const int64_t* input_ids, const int64_t* attention_mask, const int64_t* token_type_ids, int B, int S,
                     const int64_t* input_ids_, const int64_t* attention_mask_, const int64_t* token_type_ids_, int Sq,
                     float* start_out, float* end_out, float* filter_out, int mem);

/* ---- span decoding of compute_predictions_logits (densephrases/utils/squad_metrics.py:408-684), spans.cu ----
 * start / end / sft / eft fp32 [F,S] (S <= 512), n_tokens int32 [F] (<= S), start_ok / end_ok uint32 bit masks [F, ceil(S/32)]
 * (bit s of row f: token s of feature f may start / end a span), ex_off int64 [E+1] (the features of example x are
 * ex_off[x] .. ex_off[x+1]-1, at least one each).  Per example: cand int32 [E,K,3] = the first n_cand[x] (<= K) prelim
 * candidates (feature within the example, start, end) in the reference's order (score double(start)+double(end) descending,
 * ties in enumeration order), total_count / vec_count int64 [E] = valid spans before / after the filter test, and for
 * version_2 the null feature int32 [E] (within the example; -1 if no feature scores below 1e6) with its (start, end) logits
 * fp32 [E,2].  1 <= max_answer_length <= 64, 1 <= K <= 1024.  mem: every buffer on the host or every buffer on the device.
 * Synchronous on cuda_stream. */
int dph_rc_spans(const float* start, const float* end, const float* sft, const float* eft, int F, int S, const int32_t* n_tokens,
                 const uint32_t* start_ok, const uint32_t* end_ok, const int64_t* ex_off, int E, int max_answer_length,
                 double filter_threshold, int K, int version_2, int32_t* cand, int32_t* n_cand, int64_t* total_count,
                 int64_t* vec_count, int32_t* null_feature, float* null_logits, int mem, void* cuda_stream);

/* ---- phrase dump (generate_phrase_vecs.py --do_dump; embed_utils.py get_metadata -> filter_metadata -> compress_metadata) ----
 * dph_dump_layout: byte offsets [7] inside the output buffer of one dph_dump_select call with R valid rows, n_doc documents and
 * L = max_answer_length -- n_kept int64, doc_kept int32 [n_doc], fallback f2o int64 [n_doc], kept rows int8 [R,768], f2o int64 [R],
 * start2end int32 [R,L], fallback rows int8 [n_doc,768] -- and returns the buffer size (-1 on bad arguments).
 * dph_dump_select: start fp32 [B,S,768] and filter logits fp32 [B,S,2] on the device (Encoder's phrase outputs); feat int32 [B,4]
 * on the host: per feature its valid rows [row_lo, row_hi), its document slot (0, 1, ... over consecutive features) and the
 * document-level index of row_lo; doc int32 [n_doc,2] on the host: rows the document kept in earlier batches, and 1 when it still
 * needs filter_metadata's fallback row (the first row with filter_start > -999999, looked for only when the document keeps no row
 * in this batch either; written to the fallback slot, f2o -1 if none).
 * A row is kept when filter_start or filter_end > fp32(filter_threshold); kept rows are written in batch order, quantised as
 * rint(clip((x - offset) * scale, -128, 127)), with their document-level f2o index and start2end remapped to the document's short
 * indices (-1 for ends outside the feature or failing the filter_end test).  out: page-locked host memory of at least
 * dph_dump_layout bytes, written by the kernels through its device mapping.  start 16-byte, filt and out 8-byte aligned.
 * S <= 512, 1 <= L <= 64.  Synchronous on cuda_stream. */
int64_t dph_dump_layout(int64_t R, int n_doc, int L, int64_t* offsets);
int dph_dump_select(const float* start, const float* filt, int B, int S, const int32_t* feat, int n_doc, const int32_t* doc,
                    int max_answer_length, double filter_threshold, double dense_offset, double dense_scale, void* out,
                    int64_t out_bytes, void* cuda_stream);

/* ---- exact sequential-k fp32 GEMM (the inner-product definition shared with the oracle): out [n,m] = X [n,K] . W [m,K]^T,
 * acc = fmaf(x[t], w[t], acc) for t ascending; device pointers; K % 32 == 0.  Used for the OPQ rotation and the coarse quantizer. */
int dph_sgemm_nt_seq(const float* X, int64_t n, const float* W, int64_t m, int64_t K, float* out, void* cuda_stream);

/* ---- dense fp32 GEMM on the Hopper tensor cores (wgmma tf32), the encoder's building block ----
 * out [M,N] = act(A [M,K] . W [N,K]^T + bias [N]) + residual [M,N]; act: 0 none, 1 erf-GELU; device pointers;
 * N % 128 == 0, K % 32 == 0.  == torch.nn.functional.linear (HF BertSelfAttention/BertOutput/BertIntermediate). */
int dph_gemm_tf32_nt(const float* A, const float* W, const float* bias, const float* residual, float* out, int64_t M, int64_t N,
                     int64_t K, int act, int precise /* 0: 1xTF32, 1: 3xTF32 split (fp32-accurate), 2: bf16x3 split (N % 256 == 0) */,
                     void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif
