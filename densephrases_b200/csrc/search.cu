// search.cu -- the search: the per-batch plan, its workspace, and the coarse and scan stages that the entry points compose (the whole
// search and the two sharded protocols of sharded.py).  C ABI declared in include/dph_b200.h; kernel launchers live by their kernels.
#include "index_internal.cuh"

// Candidates kept per CTA: k + slack.  The proof needs T_k - (k+slack)-th score > 2 eps; the pair filter's eps is dominated by
// the 10-bit quantisation, so its slack grows with k (order statistics: the gap between ranks k and 1.5k is ~0.1 sigma).
static int keep_single(int k) { return k + DPH_KEEP_SLACK; }
static int keep_pair(int k) { return k + std::max(k / 2, DPH_KEEP_SLACK); }
// Quad filter: 8-bit entries, eps ~2.7x the pair filter's: 2 eps ~ 0.26 sigma of the scores.  The drop threshold is some unit's
// keep-th best, i.e. at global rank >= keep; the proof needs score(rank k) - score(rank keep) > 2 eps.  Order statistics of the
// top of ~6 M scores: rank 10 -> rank 110 is ~0.5 sigma, which leaves a 2x margin (7-bit entries would need keep ~ 400).
static int keep_quad(int k) { return k + std::max(2 * k, 100); }

// The scan of a batch of n queries.  A grouped mode runs while its keep fits its kernel's candidate buffers: quad for k <= 85,
// pair for k <= 683, one query per gather above.  A per-query filter always runs the one-query scan (DESIGN.md 3.7): its queries
// read few blocks, mostly not the same ones.
static DphSearchPlan search_plan(const dph_index* ix, int64_t n, int k) {
    // sharing gathers between the queries that probe a list pays when lists are probed by >= ~1.5 queries of the batch on average
    const int64_t eff_probe = std::min<int64_t>(ix->nprobe, ix->nlist);
    // ... and when lists are long enough to amortise rebuilding the packed 192 KB LUT at every (list, query group) item
    const int64_t nl_local = std::max<int64_t>(ix->list_hi - ix->list_lo, 1);
    const bool long_lists = ix->ntotal_local / nl_local >= 4096;
    const bool shared = long_lists && n * eff_probe * 2 >= ix->nlist * 3;
    DphSearchPlan p;
    p.k = k; p.exact_only = ix->scan_mode == DPH_SCAN_EXACT; p.grid = ix->num_sms;
    p.group = 1;
    if (ix->scan_mode == DPH_SCAN_PAIR) p.group = 2;
    else if (ix->scan_mode == DPH_SCAN_QUAD || (ix->scan_mode == DPH_SCAN_FAST && shared)) p.group = 4;
    if (p.group == 4 && keep_quad(k) > DPH_QUAD_KEEP_MAX) p.group = 2;
    if (p.group == 2 && keep_pair(k) > DPH_PAIR_KEEP_MAX) p.group = 1;
    if (ix->qfilter) p.group = 1;
    p.keep = p.group == 4 ? keep_quad(k) : p.group == 2 ? keep_pair(k) : keep_single(k);     // one query: every k fits (scan.cu)
    p.item_q = p.group == 4 ? DPH_QUAD_ITEM_Q : p.group;      // quad: an item runs one code read through two packed tables
    return p;
}

// Entries (u64 keys) of the candidate area ix->cand, which both passes of a search use.  plan_scan_kernel gives query q parts_q * keep
// entries, parts_q = the scan CTAs or work units that may flush q's candidates.  Summed over the batch (T = sum_q blocks_q):
//  - one query per gather (either pass): parts_q = min(blocks_q / per + 2, grid), per = max(T / grid, 1): sum < 2 grid + 2n;
//  - grouped fast pass: parts_q = nseg_q + blocks_q / per + 1, per = the blocks of a list segment (group_scan_kernel).  q's blocks
//    lie in items of <= item_q queries whose blocks number <= per * UNITS_PER_CTA * grid: sum <= n nprobe + item_q UNITS_PER_CTA grid + n.
// The area holds the first bound, plus the second when the fast pass is grouped, at the largest keep of any mode at this k.
static size_t cand_entries(const DphSearchPlan& p, int64_t n, int nprobe) {
    const size_t keep_max = std::max(keep_quad(p.k), keep_pair(p.k));
    size_t parts = (size_t)(2 * p.grid + 2 * n + 2);
    if (p.grouped()) parts += (size_t)(n * nprobe + (int64_t)p.item_q * DPH_GROUP_UNITS_PER_CTA * p.grid + 2 * n + 16);
    return parts * keep_max;
}

// Coarse stage workspace: rotated queries, coarse scores and probes of n queries (the sharded entry points also receive probes here).
static int size_coarse(dph_index* ix, int64_t n) {
    DPH_TRY(ix->xr.ensure((size_t)n * ix->d * 4));
    DPH_TRY(ix->S.ensure((size_t)n * ix->nlist * 4));
    for (DevBuf* b : {&ix->key, &ix->cd}) DPH_TRY(b->ensure((size_t)n * ix->nprobe * 4));
    return 0;
}

// Scan stage workspace: tables, plans, candidates and flags of n queries under plan p, for both passes.
static int size_scan(dph_index* ix, const DphSearchPlan& p, int64_t n) {
    const size_t nq = (size_t)n, np = nq * ix->nprobe, nl = (size_t)ix->nlist;
    for (DevBuf* b : {&ix->qinfo, &ix->eps, &ix->nseg, &ix->cand_cnt, &ix->gthr, &ix->flags}) DPH_TRY(b->ensure(nq * 4));
    for (DevBuf* b : {&ix->lutmax, &ix->lutmin, &ix->lutmaxv}) DPH_TRY(b->ensure(nq * DPH_M * 4));
    DPH_TRY(ix->lut_canon.ensure(nq * DPH_LUT_CANON_FLOATS * 4));
    DPH_TRY(ix->segs.ensure(np * sizeof(DphSeg)));
    for (DevBuf* b : {&ix->wpre, &ix->cand_off}) DPH_TRY(b->ensure((nq + 1) * 8));
    DPH_TRY(ix->cand.ensure(cand_entries(p, n, ix->nprobe) * 8));
    DPH_TRY(ix->work.ensure(sizeof(DphWork)));
    if (!p.grouped()) return 0;
    DPH_TRY(ix->lutq.ensure(nq * (p.group == 4 ? DPH_LUTQ8_BYTES : DPH_LUT_SCAN_FLOATS * 2)));
    DPH_TRY(ix->qparams.ensure(nq * 8));
    for (DevBuf* b : {&ix->gdense, &ix->grp_entries}) DPH_TRY(b->ensure(np * 4));
    for (DevBuf* b : {&ix->grp_cnt, &ix->grp_fill}) DPH_TRY(b->ensure(nl * 4));
    for (DevBuf* b : {&ix->grp_off, &ix->grp_unitpre}) DPH_TRY(b->ensure((nl + 1) * 4));
    DPH_TRY(ix->grp_blockpre.ensure((nl + 1) * 8));
    // units <= sum_l items_l * (blocks_l / seg + 1) <= total_blocks / seg + items <= UNITS_PER_CTA * grid + n * nprobe
    const size_t units = np + (size_t)DPH_GROUP_UNITS_PER_CTA * p.grid + 16;
    DPH_TRY(ix->grp_units.ensure(units * 8));
    if (p.group == 4) DPH_TRY(ix->grp_udesc.ensure(units * sizeof(DphUnit)));
    DPH_TRY(ix->groupwork.ensure(sizeof(DphGroupWork)));
    return 0;
}

// Coarse stage: OPQ rotation of x [n, d] into xr, then the nprobe best lists of every query -- over ALL lists into (key, cd) when
// keys64 is null, else over this shard's lists into keys64 as (score, list) keys (the list-split sharded coarse quantizer).
static int coarse_stage(dph_index* ix, const float* x_dev, int64_t n, unsigned long long* keys64) {
    cudaStream_t st = ix->stream;
    const int nprobe = ix->nprobe;
    const int64_t lo = keys64 ? ix->list_lo : 0, nl = keys64 ? ix->list_hi - ix->list_lo : ix->nlist;
    DPH_TRY(size_coarse(ix, n));
    int32_t* key = keys64 ? nullptr : ix->key.as<int32_t>();
    float* cd = keys64 ? nullptr : ix->cd.as<float>();
    DPH_TRY(dph_launch_sgemm_nt_seq(x_dev, n, ix->A, ix->d, ix->d, ix->xr.as<float>(), st));                   // OPQ rotation
    const int rc = ix->coarse_tc ? dph_coarse_tc(ix, n, lo, nl, nprobe, keys64, key, cd, st) : 1;
    if (rc != 1) return rc;                                                                  // 0: done on the tensor cores
    DPH_TRY(dph_launch_sgemm_nt_seq(ix->xr.as<float>(), n, ix->C + lo * ix->d, nl, ix->d, ix->S.as<float>(), st));   // coarse scores
    if (keys64) DPH_TRY(dph_launch_coarse_select(ix->S.as<float>(), n, nl, nprobe, nullptr, nullptr, st, keys64, (unsigned)lo));
    else DPH_TRY(dph_launch_coarse_select(ix->S.as<float>(), n, nl, nprobe, key, cd, st, nullptr, 0u, nullptr, 0, &ix->selkeys));
    return 0;
}

// The fast pass (plan, scan, merge) over the codes of src and the exact re-run of the queries its merge flagged (launches that exit
// at once when none is), or the exact pass alone in EXACT mode.  Writes D, I, G [n, k]; the profiling events bracket the first
// pass's scan kernel.
int dph_scan_passes(dph_index* ix, const DphSearchPlan& p, const DphCodeSrc& src, int64_t n, int k, float* D, int64_t* I, uint32_t* G) {
    cudaStream_t st = ix->stream;
    const bool exact = p.exact_only;
    if (exact) DPH_CUDA(cudaMemsetAsync(ix->flags.p, 0, (size_t)n * 4, st));
    DPH_TRY(dph_launch_plan(ix, p, src, n, exact, nullptr, st));
    if (ix->profile) DPH_CUDA(cudaEventRecord(ix->ev0[ix->prof_n % DPH_PROF_RING], st));
    DPH_TRY(dph_launch_scan(ix, p, src, n, exact, st));
    if (ix->profile) { DPH_CUDA(cudaEventRecord(ix->ev1[ix->prof_n % DPH_PROF_RING], st)); ix->prof_n++; }
    DPH_TRY(dph_launch_merge(ix, src.codes, n, k, exact ? DPH_SCAN_EXACT : DPH_SCAN_FAST, nullptr, D, I, G, st));
    if (exact) return 0;
    DPH_TRY(dph_launch_plan(ix, p, src, n, true, ix->flags.as<int32_t>(), st));
    DPH_TRY(dph_launch_scan(ix, p, src, n, true, st));
    DPH_TRY(dph_launch_merge(ix, src.codes, n, k, DPH_SCAN_EXACT, ix->flags.as<int32_t>(), D, I, G, st));
    return 0;
}

// The row mask of the filter set on ix (nullptr: none).  Rejects a filter of another handle or of an earlier layout of this one.
static int active_mask(const dph_index* ix, const uint32_t** mask) {
    const dph_filter* f = ix->filter;
    *mask = nullptr;
    if (ix->qfilter) {
        const dph_query_filter* qf = ix->qfilter;
        DPH_CHECK(qf->ix == ix, "search: the query filter was built for another index; build it with this index's make_query_filters");
        DPH_CHECK(qf->version == ix->layout_version,
                  "search: the query filter is stale (the index's lists changed since it was built: set_lists, add, remove, merge or "
                  "sync_list_len); rebuild the filter");
    }
    if (!f) return 0;
    DPH_CHECK(f->ix == ix, "search: the filter was built for another index; build it with this index's make_filter");
    DPH_CHECK(f->version == ix->layout_version,
              "search: the filter is stale (the index's lists changed since it was built: set_lists, add, remove, merge or sync_list_len); "
              "rebuild the filter");
    *mask = f->mask;
    return 0;
}

// A search of n queries with a per-query filter set needs the filter's n (checked before the search changes anything).
static int check_query_filter_n(const dph_index* ix, int64_t n) {
    if (!ix->qfilter) return 0;
    DPH_CHECK(ix->qfilter->n == n, "search: the query filter was built for " + std::to_string(ix->qfilter->n) + " queries, the batch has " +
                                   std::to_string(n));
    return 0;
}

// Scan stage, from the rotated queries in xr and the probes in (key, cd): the tables, then the passes over the shard's codes -- in
// host mode slice by slice, the tables built once for all slices.  Every search path passes here, so the active filter applies here.
// q0: the chunk's first query in the batch (the row of a per-query filter's assignment).
static int scan_stage(dph_index* ix, int64_t n, int k, float* D, int64_t* I, uint32_t* G, int64_t q0 = 0) {
    cudaStream_t st = ix->stream;
    const uint32_t* mask;
    DPH_TRY(active_mask(ix, &mask));
    const DphQfView* qf = nullptr;
    if (ix->qfilter) {
        const DphQfView v = ix->qfilter->view(q0);
        DPH_TRY(ix->qfview.ensure(sizeof(DphQfView)));
        DPH_CUDA(cudaMemcpyAsync(ix->qfview.p, &v, sizeof v, cudaMemcpyHostToDevice, st));
        qf = ix->qfview.as<DphQfView>();
    }
    const DphSearchPlan p = search_plan(ix, n, k);
    DPH_TRY(size_scan(ix, p, n));
    ix->last_group = p.group;
    DPH_TRY(dph_launch_lut(ix->xr.as<float>(), n, ix->pq, ix->lut_canon.as<float>(), ix->lutmax.as<float>(),
                           ix->lutmin.as<float>(), ix->lutmaxv.as<float>(), p.grouped() ? ix->lutq.p : nullptr,
                           p.grouped() ? ix->qparams.as<float2>() : nullptr, st, p.group));
    if (ix->on_host) return dph_host_scan(ix, p, n, k, D, I, G, mask, qf);
    const DphCodeSrc src{ix->codes, (const long long*)ix->blk_off, ix->list_lo, ix->list_hi, mask, qf};
    return dph_scan_passes(ix, p, src, n, k, D, I, G);
}

// Host mode: the fetch counters describe the last search call.
static void reset_fetch(dph_index* ix) {
    std::fill(ix->fetch_counts, ix->fetch_counts + 4, 0);
    ix->fetch_ms = 0.f;
}

static int64_t chunk_size(const dph_index* ix, int64_t n) {
    int64_t c = (1ll << 28) / std::max<int64_t>(ix->nlist, 1);   // S chunk <= 1 GiB
    c = std::max<int64_t>(1, std::min<int64_t>(c, 4096));
    return std::min(c, n);
}

DPH_API int dph_index_search_partial(dph_index* ix, const float* x_dev, int64_t n, int k, float* D, int64_t* I, uint32_t* G) {
    DPH_TRY(check_ready(ix, k));
    DPH_TRY(check_query_filter_n(ix, n));
    DPH_CUDA(cudaSetDevice(ix->device));
    reset_fetch(ix);
    const int64_t cs = chunk_size(ix, n);
    for (int64_t o = 0; o < n; o += cs) {
        const int64_t m = std::min(cs, n - o);
        DPH_TRY(coarse_stage(ix, x_dev + o * ix->d, m, nullptr));
        DPH_TRY(scan_stage(ix, m, k, D + o * k, I + o * k, G + o * k, o));
    }
    return 0;
}

DPH_API int dph_index_search(dph_index* ix, const float* x, int64_t n, int k, float* D, int64_t* I, int mem) {
    DPH_TRY(check_ready(ix, k));
    DPH_TRY(check_query_filter_n(ix, n));
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n == 0) return 0;
    DPH_TRY(ix->Gp.ensure((size_t)n * k * 4));
    if (mem == DPH_MEM_DEVICE) return dph_index_search_partial(ix, x, n, k, D, I, ix->Gp.as<uint32_t>());
    DPH_TRY(ix->xdev.ensure((size_t)n * ix->d * 4));
    DPH_TRY(ix->Dp.ensure((size_t)n * k * 4));
    DPH_TRY(ix->Ip.ensure((size_t)n * k * 8));
    DPH_CUDA(cudaMemcpyAsync(ix->xdev.p, x, (size_t)n * ix->d * 4, cudaMemcpyHostToDevice, ix->stream));
    DPH_TRY(dph_index_search_partial(ix, ix->xdev.as<float>(), n, k, ix->Dp.as<float>(), ix->Ip.as<int64_t>(), ix->Gp.as<uint32_t>()));
    DPH_CUDA(cudaMemcpyAsync(D, ix->Dp.p, (size_t)n * k * 4, cudaMemcpyDeviceToHost, ix->stream));
    DPH_CUDA(cudaMemcpyAsync(I, ix->Ip.p, (size_t)n * k * 8, cudaMemcpyDeviceToHost, ix->stream));
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    return 0;
}

// ---- sharded coarse quantizer (every rank scores only its own lists' centroids; SURVEY.md 8e "Partitioning") ----
DPH_API int dph_index_coarse_local(dph_index* ix, const float* x_dev, int64_t n, uint64_t* keys_dev) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_CHECK(n <= chunk_size(ix, n), "coarse_local: batch too large for one chunk");
    ix->last_coarse_n = n;
    return coarse_stage(ix, x_dev, n, (unsigned long long*)keys_dev);
}
DPH_API int dph_index_search_preassigned(dph_index* ix, const uint64_t* keys_gathered_dev, int nshards, int64_t n, int k, float* D_dev,
                                         int64_t* I_dev, uint32_t* G_dev) {
    DPH_TRY(check_ready(ix, k));
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_CHECK(n == ix->last_coarse_n, "search_preassigned must follow coarse_local with the same batch");
    DPH_TRY(check_query_filter_n(ix, n));
    reset_fetch(ix);
    DPH_TRY(size_coarse(ix, n));
    DPH_TRY(dph_launch_coarse_merge((const unsigned long long*)keys_gathered_dev, nshards, n, ix->nprobe, ix->key.as<int32_t>(), ix->cd.as<float>(),
                                    ix->stream));
    return scan_stage(ix, n, k, D_dev, I_dev, G_dev);
}

// ---- query-split sharded search (sharded.py): every rank rotates and assigns ITS SLICE of the batch over ALL lists, the ranks
// exchange one record per query -- [768 f32 rotated query | nprobe i32 lists | nprobe f32 coarse scores] -- and then scan their own
// lists.  Against the list-split coarse quantizer above it removes the replicated rotation and exact re-rank (each done for n / W
// queries instead of n) and the merge of per-shard candidates; it needs the full centroid table on every rank (it is replicated).
__global__ void pack_records_kernel(const float* __restrict__ xr, const int* __restrict__ key, const float* __restrict__ cd, int nprobe, float* __restrict__ rec) {
    const long long q = blockIdx.x;
    const int R = DPH_D + 2 * nprobe;
    float* o = rec + q * R;
    for (int t = threadIdx.x; t < R; t += blockDim.x)
        o[t] = t < DPH_D ? xr[q * DPH_D + t] : (t < DPH_D + nprobe ? __int_as_float(key[q * nprobe + t - DPH_D]) : cd[q * nprobe + t - DPH_D - nprobe]);
}
__global__ void unpack_records_kernel(const float* __restrict__ rec, int nprobe, float* __restrict__ xr, int* __restrict__ key, float* __restrict__ cd) {
    const long long q = blockIdx.x;
    const int R = DPH_D + 2 * nprobe;
    const float* r = rec + q * R;
    for (int t = threadIdx.x; t < R; t += blockDim.x) {
        const float v = r[t];
        if (t < DPH_D) xr[q * DPH_D + t] = v;
        else if (t < DPH_D + nprobe) key[q * nprobe + t - DPH_D] = __float_as_int(v);
        else cd[q * nprobe + t - DPH_D - nprobe] = v;
    }
}
DPH_API int dph_index_record_floats(const dph_index* ix) { return ix->d + 2 * ix->nprobe; }
DPH_API int dph_index_coarse_split(dph_index* ix, const float* x_dev, int64_t n_local, float* rec_dev) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n_local == 0) return 0;
    DPH_CHECK(n_local <= chunk_size(ix, n_local), "coarse_split: slice too large for one chunk");
    DPH_TRY(coarse_stage(ix, x_dev, n_local, nullptr));
    pack_records_kernel<<<(unsigned)n_local, 256, 0, ix->stream>>>(ix->xr.as<float>(), ix->key.as<int>(), ix->cd.as<float>(), ix->nprobe, rec_dev);
    DPH_CUDA(cudaGetLastError());
    return 0;
}
DPH_API int dph_index_search_assigned(dph_index* ix, const float* rec_dev, int64_t n, int k, float* D_dev, int64_t* I_dev, uint32_t* G_dev) {
    DPH_TRY(check_ready(ix, k));
    DPH_CUDA(cudaSetDevice(ix->device));
    DPH_TRY(check_query_filter_n(ix, n));
    if (n == 0) return 0;
    reset_fetch(ix);
    DPH_TRY(size_coarse(ix, n));
    unpack_records_kernel<<<(unsigned)n, 256, 0, ix->stream>>>(rec_dev, ix->nprobe, ix->xr.as<float>(), ix->key.as<int>(), ix->cd.as<float>());
    DPH_CUDA(cudaGetLastError());
    return scan_stage(ix, n, k, D_dev, I_dev, G_dev);
}
