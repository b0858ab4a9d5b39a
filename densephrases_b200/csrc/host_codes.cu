// host_codes.cu -- codes in host memory (DESIGN.md 3.5): the shard's code blocks live in page-locked, device-mapped host memory; a
// set of resident lists and a fixed-size stream region live in HBM.  Every search chunk is scanned in slices: each slice's probed,
// non-resident lists are fetched into the stream region, the unchanged plan / scan / merge passes run over a per-slice block-offset
// view, and the slices' partial top-k are folded into a running top-k with the shard merge.  Bit-identical to the resident index.
#include "index_internal.cuh"

// Gathers the blocks of lists[0 .. nf) from src (block src_off[list] on) into dst, packed in descriptor order: list i's blocks go to
// dst blocks [pre[i], pre[i+1]).  One warp per 3 KB block; each lane issues its six 16-byte loads before any store, so that a warp
// keeps a whole block in flight over PCIe when src is mapped host memory.
__global__ void __launch_bounds__(256) fetch_lists_kernel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src,
                                                          const long long* __restrict__ src_off, const long long* __restrict__ lists,
                                                          const long long* __restrict__ pre, int nf) {
    const long long total = pre[nf];
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long b = w0; b < total; b += nw) {
        int lo = 0, hi = nf;                       // last descriptor i with pre[i] <= b (as list_of_block)
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pre[mid] <= b) lo = mid; else hi = mid; }
        const uint4* s = reinterpret_cast<const uint4*>(src + (src_off[lists[lo]] + b - pre[lo]) * DPH_BLK_BYTES) + lane;
        uint4 v[6];
#pragma unroll
        for (int c = 0; c < 6; c++) v[c] = s[c * 32];
        uint4* d = reinterpret_cast<uint4*>(dst + b * DPH_BLK_BYTES) + lane;
#pragma unroll
        for (int c = 0; c < 6; c++) d[c * 32] = v[c];
    }
}

// The view of one slice: for every list l in [lo, hi), its first block in the HBM region -- resident (res_off[l]) or fetched into the
// stream region (stream0 + its descriptor's prefix) -- or -1 (not probed in this slice, never read).
__global__ void view_kernel(long long* view, long long lo, long long hi, const long long* res_off, const long long* lists, const long long* pre,
                            int nf, long long stream0) {
    const long long l = lo + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= hi) return;
    long long v = res_off[l];
    if (v < 0) {
        int a = 0, b = nf;                         // first descriptor with lists[i] >= l
        while (a < b) { const int m = (a + b) >> 1; if (lists[m] < l) a = m + 1; else b = m; }
        if (a < nf && lists[a] == l) v = stream0 + pre[a];
    }
    view[l] = v;
}

static int launch_fetch(dph_index* ix, uint8_t* dst, const long long* lists, const long long* pre, int64_t nf, int64_t blocks) {
    if (blocks == 0) return 0;
    const unsigned grid = (unsigned)std::min<int64_t>((blocks + 7) / 8, (int64_t)ix->num_sms * 8);
    fetch_lists_kernel<<<grid, 256, 0, ix->stream>>>(dst, ix->codes, (const long long*)ix->blk_off, lists, pre, (int)nf);
    DPH_CUDA(cudaGetLastError());
    return 0;
}

static void update_max_stream_blocks(dph_index* ix) {
    int64_t m = 0;
    for (int64_t l = ix->list_lo; l < ix->list_hi; l++)
        if (ix->res_off[l] < 0) m = std::max<int64_t>(m, (ix->lay.len[l] + 31) / 32);
    ix->max_stream_blocks = m;
}

static int alloc_region(uint8_t** out, int64_t blocks, const char* what) {
    const cudaError_t e = cudaMalloc((void**)out, (size_t)std::max<int64_t>(blocks, 1) * DPH_BLK_BYTES);
    if (e != cudaSuccess) {
        cudaGetLastError();
        *out = nullptr;
        dph_set_error(std::string(what) + ": " + cudaGetErrorString(e));
        return 1;
    }
    return 0;
}

int dph_host_lists_ready(dph_index* ix) {
    const int64_t nlist = ix->nlist;
    ix->res_off.assign(nlist, -1);
    ix->res_blocks = 0;
    DPH_CUDA(cudaMalloc((void**)&ix->res_off_dev, nlist * 8));
    DPH_CUDA(cudaMemcpy(ix->res_off_dev, ix->res_off.data(), nlist * 8, cudaMemcpyHostToDevice));
    DPH_TRY(alloc_region(&ix->region, ix->stream_blocks, "set_lists: the stream region"));
    ix->region_blocks = ix->stream_blocks;
    update_max_stream_blocks(ix);
    return 0;
}

int dph_host_after_mutation(dph_index* ix, bool shard_changed) {
    if (shard_changed) {                           // the region keeps its size; the stream region takes all of it
        std::fill(ix->res_off.begin(), ix->res_off.end(), (int64_t)-1);
        ix->res_blocks = 0;
        DPH_CUDA(cudaMemcpy(ix->res_off_dev, ix->res_off.data(), ix->nlist * 8, cudaMemcpyHostToDevice));
    }
    update_max_stream_blocks(ix);
    return 0;
}

DPH_API int dph_index_set_code_residency(dph_index* ix, int on_host, int64_t stream_bytes) {
    DPH_CHECK(ix != nullptr, "null index");
    DPH_CHECK(stream_bytes >= 0 && (on_host || stream_bytes == 0),
              "set_code_residency: stream_bytes must be >= 0, and 0 when the codes stay in device memory; the index is unchanged");
    DPH_CHECK((on_host != 0) == ix->on_host || ix->list_len == nullptr,
              "set_code_residency: where the codes live must be chosen before set_lists; the index is unchanged");
    DPH_CUDA(cudaSetDevice(ix->device));
    const int64_t sb = stream_bytes / DPH_BLK_BYTES;
    if (on_host && ix->list_len) {                 // a new region: the resident blocks move over, the old region goes
        uint8_t* r;
        DPH_TRY(alloc_region(&r, ix->res_blocks + sb, "set_code_residency: not enough device memory for the new region; the index is unchanged"));
        if (ix->res_blocks > 0)
            DPH_CUDA(cudaMemcpyAsync(r, ix->region, (size_t)ix->res_blocks * DPH_BLK_BYTES, cudaMemcpyDeviceToDevice, ix->stream));
        DPH_CUDA(cudaStreamSynchronize(ix->stream));
        cudaFree(ix->region);
        ix->region = r;
        ix->region_blocks = ix->res_blocks + sb;
    }
    if (!on_host) { ix->host_reserve = 0; ix->host_mutable = false; }
    ix->on_host = on_host != 0;
    ix->stream_blocks = sb;
    return 0;
}

DPH_API int dph_index_set_resident_lists(dph_index* ix, const int64_t* lists, int64_t n) {
    DPH_CHECK(ix && ix->on_host && ix->list_len, "set_resident_lists: needs an index whose codes are in host memory, after set_lists");
    DPH_CHECK(n >= 0 && (lists != nullptr || n == 0), "set_resident_lists: bad list array; the index is unchanged");
    const int64_t lo = ix->list_lo, hi = ix->list_hi, nlist = ix->nlist;
    std::vector<int64_t> ls(lists, lists + n);
    for (int64_t l : ls)
        if (l < lo || l >= hi) {
            dph_set_error("set_resident_lists: list " + std::to_string(l) + " is not in this shard [" + std::to_string(lo) + ", " +
                          std::to_string(hi) + "); the index is unchanged");
            return 1;
        }
    std::sort(ls.begin(), ls.end());
    ls.erase(std::unique(ls.begin(), ls.end()), ls.end());
    std::vector<int64_t> off(nlist, -1), desc, pre{0};
    int64_t nb = 0;
    for (int64_t l : ls) {
        off[l] = nb;
        const int64_t b = (ix->lay.len[l] + 31) / 32;
        if (b > 0) { desc.push_back(l); nb += b; pre.push_back(nb); }
    }
    DPH_CUDA(cudaSetDevice(ix->device));
    const char* oom = "set_resident_lists: not enough device memory for the resident lists and the stream region; the index is unchanged";
    DevTmp tmp;
    uint8_t* r; int64_t* d_desc;
    DPH_TRY(tmp.alloc(&r, (size_t)(nb + ix->stream_blocks) * DPH_BLK_BYTES, oom));
    DPH_TRY(tmp.alloc(&d_desc, desc.size() + pre.size(), oom));
    desc.insert(desc.end(), pre.begin(), pre.end());
    DPH_CUDA(cudaMemcpyAsync(d_desc, desc.data(), desc.size() * 8, cudaMemcpyHostToDevice, ix->stream));
    const int64_t nf = (int64_t)pre.size() - 1;
    DPH_TRY(launch_fetch(ix, r, (const long long*)d_desc, (const long long*)d_desc + nf, nf, nb));
    DPH_CUDA(cudaMemcpyAsync(ix->res_off_dev, off.data(), nlist * 8, cudaMemcpyHostToDevice, ix->stream));
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    tmp.release(r);
    cudaFree(ix->region);
    ix->region = r;
    ix->res_blocks = nb;
    ix->region_blocks = nb + ix->stream_blocks;
    ix->res_off = std::move(off);
    update_max_stream_blocks(ix);
    return 0;
}

int dph_host_scan(dph_index* ix, const DphSearchPlan& p, int64_t n, int k, float* D, int64_t* I, uint32_t* G, const uint32_t* mask,
                  const DphQfView* qf) {
    cudaStream_t st = ix->stream;
    const int64_t lo = ix->list_lo, hi = ix->list_hi, np = n * ix->nprobe, sb = ix->region_blocks - ix->res_blocks;
    if (ix->max_stream_blocks > sb) {
        dph_set_error("search: the stream region holds " + std::to_string(sb) + " blocks; the largest non-resident list of the shard needs " +
                      std::to_string(ix->max_stream_blocks) + " (raise stream_bytes or make that list resident)");
        return 1;
    }
    // 1. the chunk's probed lists: one copy of the probes to the host and one synchronisation
    std::vector<int32_t> key(np);
    DPH_CUDA(cudaMemcpyAsync(key.data(), ix->key.p, (size_t)np * 4, cudaMemcpyDeviceToHost, st));
    DPH_CUDA(cudaStreamSynchronize(st));
    std::vector<uint8_t> probed(std::max<int64_t>(hi - lo, 1), 0);
    for (const int32_t l : key)
        if (l >= lo && l < hi && ix->lay.len[l] > 0) probed[l - lo] = 1;
    // 2. slices: probed lists in ascending id; a new slice starts when the next list's blocks would overflow the stream region.  Slice
    // s covers lists [s_lo[s], s_lo[s + 1]) (the last one up to hi), fetches descriptors [d0[s], d0[s + 1]) whose destination prefix
    // starts at pre[d0[s] + s] (one more entry per slice: its total).  A chunk that probes nothing is one empty slice.
    std::vector<int64_t> s_lo, d0, desc, pre;
    int64_t used = 0, resident = 0, fetched_blocks = 0;
    for (int64_t l = lo; l < hi; l++) {
        if (!probed[l - lo]) continue;
        const int64_t cost = ix->res_off[l] >= 0 ? 0 : (ix->lay.len[l] + 31) / 32;
        if (s_lo.empty() || used + cost > sb) {
            if (!s_lo.empty()) { pre.push_back(used); fetched_blocks += used; }
            s_lo.push_back(s_lo.empty() ? lo : l);
            d0.push_back((int64_t)desc.size());
            used = 0;
        }
        if (cost > 0) { desc.push_back(l); pre.push_back(used); used += cost; }
        else resident++;
    }
    if (s_lo.empty()) { s_lo.push_back(lo); d0.push_back(0); }
    pre.push_back(used); fetched_blocks += used;
    d0.push_back((int64_t)desc.size());
    const int64_t ns = (int64_t)s_lo.size(), nd = (int64_t)desc.size();
    desc.insert(desc.end(), pre.begin(), pre.end());
    DPH_TRY(ix->fdesc.ensure(desc.size() * 8));
    DPH_TRY(ix->view.ensure((size_t)ix->nlist * 8));
    DPH_CUDA(cudaMemcpyAsync(ix->fdesc.p, desc.data(), desc.size() * 8, cudaMemcpyHostToDevice, st));
    const size_t nk = (size_t)n * k;
    if (ns > 1) {                                  // [2, n, k]: the running top-k, then the slice's
        DPH_TRY(ix->hs_D.ensure(2 * nk * 4)); DPH_TRY(ix->hs_I.ensure(2 * nk * 8)); DPH_TRY(ix->hs_G.ensure(2 * nk * 4));
    }
    // 3. per slice: fetch, view, the passes, the fold into the running top-k (in D, I, G)
    const long long* d_desc = ix->fdesc.as<long long>();
    long long* view = ix->view.as<long long>();
    const bool prof = ix->profile && ix->aev[0];
    for (int64_t s = 0; s < ns; s++) {
        const int64_t a = d0[s], nf = d0[s + 1] - a, slo = s_lo[s], shi = s + 1 < ns ? s_lo[s + 1] : hi;
        const long long *lists = d_desc + a, *spre = d_desc + nd + a + s;
        if (prof) DPH_CUDA(cudaEventRecord(ix->aev[0], st));
        DPH_TRY(launch_fetch(ix, ix->region + ix->res_blocks * DPH_BLK_BYTES, lists, spre, nf, pre[a + s + nf]));
        if (prof) {
            DPH_CUDA(cudaEventRecord(ix->aev[1], st));
            DPH_CUDA(cudaEventSynchronize(ix->aev[1]));
            float ms = 0.f;
            DPH_CUDA(cudaEventElapsedTime(&ms, ix->aev[0], ix->aev[1]));
            ix->fetch_ms += ms;
        }
        if (shi > slo)
            view_kernel<<<(unsigned)((shi - slo + 255) / 256), 256, 0, st>>>(view, slo, shi, (const long long*)ix->res_off_dev, lists, spre,
                                                                           (int)nf, ix->res_blocks);
        DPH_CUDA(cudaGetLastError());
        const DphCodeSrc src{ix->region, view, slo, shi, mask, qf};     // the filters are indexed by the shard's blocks / lists, not the view's
        if (s == 0) { DPH_TRY(dph_scan_passes(ix, p, src, n, k, D, I, G)); continue; }
        float* hD = ix->hs_D.as<float>(); int64_t* hI = ix->hs_I.as<int64_t>(); uint32_t* hG = ix->hs_G.as<uint32_t>();
        DPH_CUDA(cudaMemcpyAsync(hD, D, nk * 4, cudaMemcpyDeviceToDevice, st));
        DPH_CUDA(cudaMemcpyAsync(hI, I, nk * 8, cudaMemcpyDeviceToDevice, st));
        DPH_CUDA(cudaMemcpyAsync(hG, G, nk * 4, cudaMemcpyDeviceToDevice, st));
        DPH_TRY(dph_scan_passes(ix, p, src, n, k, hD + nk, hI + nk, hG + nk));
        DPH_TRY(dph_launch_merge_shards(hD, hI, hG, 2, n, k, D, I, G, st));
    }
    ix->fetch_counts[0] += ns; ix->fetch_counts[1] += nd; ix->fetch_counts[2] += fetched_blocks; ix->fetch_counts[3] += resident;
    return 0;
}

DPH_API int dph_index_last_fetch(const dph_index* ix, int64_t* counts, float* ms) {
    DPH_CHECK(ix && ix->on_host, "last_fetch: the codes of this index are in device memory");
    std::copy(ix->fetch_counts, ix->fetch_counts + 4, counts);
    if (ms) *ms = ix->fetch_ms;
    return 0;
}

DPH_API int64_t dph_index_host_bytes(const dph_index* ix) {
    return ix->host_codes ? std::max<int64_t>(ix->host_blocks, 1) * DPH_BLK_BYTES : 0;
}
