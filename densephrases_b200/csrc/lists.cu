// lists.cu -- the resident lists: their layout, set_lists / set_lists_synthetic, add_with_ids, copy_lists (DESIGN.md 3, 3.1).
// remove.cu holds remove_ids and sync_list_len; both commit their layout through dph_commit_layout below.
#include "index_internal.cuh"
#include <stdlib.h>
#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/sequence.h>
#include <thrust/sort.h>

int64_t dph_chunk_rows() {
    int64_t chunk_rows = (256ll << 20) / DPH_CODE;
    if (const char* ev = getenv("DPH_UPLOAD_CHUNK_ROWS")) chunk_rows = std::max<int64_t>(1, atoll(ev));      // tests: force many chunks
    return chunk_rows;
}

int DphLayout::build(const dph_index* ix, const int64_t* list_len, const char* what) {
    const int64_t nlist = ix->nlist;
    lo = ix->list_lo; hi = ix->list_hi;
    len.assign(nlist, 0); start.assign(nlist + 1, 0); blk_off.assign(nlist, -1); row_start.assign(std::max<int64_t>(hi - lo, 1), 0);
    for (int64_t l = 0; l < nlist; l++) {
        DPH_CHECK(list_len[l] >= 0 && list_len[l] < (1ll << 31), what);
        len[l] = (int32_t)list_len[l];
        start[l + 1] = start[l] + list_len[l];
    }
    nblocks = rows = 0;
    for (int64_t l = lo; l < hi; l++) {
        blk_off[l] = nblocks; row_start[l - lo] = rows;
        nblocks += (list_len[l] + 31) / 32; rows += list_len[l];
    }
    return 0;
}

std::vector<DphLayout::Chunk> DphLayout::chunks(int64_t* max_rows) const {
    const int64_t chunk_rows = dph_chunk_rows();
    std::vector<Chunk> out;
    *max_rows = 0;
    for (int64_t l0 = lo, l1; l0 < hi; l0 = l1) {
        int64_t acc = 0;
        for (l1 = l0; l1 < hi && (acc == 0 || acc + len[l1] <= chunk_rows); l1++) acc += len[l1];
        if (acc == 0) break;                                 // only empty lists are left
        out.push_back({row_start[l0 - lo], acc, blk_off[l0], l1 < hi ? blk_off[l1] : nblocks});
        *max_rows = std::max(*max_rows, acc);
    }
    return out;
}

int dph_commit_layout(dph_index* ix, DphLayout L) {
    const int64_t nlist = ix->nlist;
    DPH_CUDA(cudaMemcpy(ix->list_len, L.len.data(), nlist * 4, cudaMemcpyHostToDevice));
    DPH_CUDA(cudaMemcpy(ix->list_start, L.start.data(), (nlist + 1) * 8, cudaMemcpyHostToDevice));
    DPH_CUDA(cudaMemcpy(ix->blk_off, L.blk_off.data(), nlist * 8, cudaMemcpyHostToDevice));
    ix->ntotal = L.start[nlist]; ix->ntotal_local = L.rows; ix->nblocks_local = L.nblocks;
    ix->lay = std::move(L);
    return 0;
}

// One thread per (block, lane, 16-byte chunk): writes the interleaved/rotated layout (common.cuh).
// raw != nullptr: gather from list-major rows [*,96] (row index = local_row_start[l] + j); else synthesise from seed.
__global__ void __launch_bounds__(192) fill_blocks_kernel(uint8_t* codes, long long nblocks, const long long* blk_off, const int* list_len,
                                                          long long list_lo, long long list_hi, const uint8_t* raw,
                                                          const long long* local_row_start, uint64_t seed, long long blk0, long long raw_row0) {
    const long long blk = blk0 + blockIdx.x;                  // this launch covers blocks [blk0, nblocks)
    if (blk >= nblocks) return;
    const int lane = threadIdx.x & 31, c = threadIdx.x >> 5;   // c in 0..5
    __shared__ long long s_l;
    if (threadIdx.x == 0) s_l = list_of_block(blk_off, list_lo, list_hi, blk);
    __syncthreads();
    const long long l = s_l;
    const long long j = (blk - blk_off[l]) * 32 + lane;
    const bool valid = j < (long long)list_len[l];
    const int seg = c >> 1;
    unsigned char bytes[16];
    if (!valid) {
#pragma unroll
        for (int b = 0; b < 16; b++) bytes[b] = 0;
    } else if (raw) {
        const uint8_t* row = raw + (local_row_start[l - list_lo] + j - raw_row0) * DPH_CODE;      // raw holds rows [raw_row0, ...) of the shard
#pragma unroll
        for (int b = 0; b < 16; b++) bytes[b] = row[dph_blk_sub(lane, c * 16 + b)];
    } else {
        uint64_t w[4];
#pragma unroll
        for (int i = 0; i < 4; i++) w[i] = dph_rnd64(seed, DPH_STREAM_CODES, (uint64_t)l, (uint64_t)(j * 12 + seg * 4 + i));
#pragma unroll
        for (int b = 0; b < 16; b++) {
            const int ml = dph_blk_sub(lane, c * 16 + b) & 31;     // byte within the 32-byte segment
            bytes[b] = (unsigned char)(w[ml >> 3] >> (8 * (ml & 7)));
        }
    }
    uint4 v;
    memcpy(&v, bytes, 16);
    *reinterpret_cast<uint4*>(codes + blk * DPH_BLK_BYTES + c * 512 + lane * 16) = v;
}

// labels of the padded rows of blocks [blk0, nblocks) + the direct-map pairs (label, padded row) of the real rows
__global__ void fill_ids_kernel(long long* ids, long long nblocks, const long long* blk_off, const int* list_len, long long list_lo,
                                long long list_hi, const long long* raw_ids, const long long* local_row_start, long long blk0, long long raw_row0,
                                long long* dm_ids, long long* dm_rows) {
    const long long blk = blk0 + blockIdx.x;
    if (blk >= nblocks) return;
    const long long l = list_of_block(blk_off, list_lo, list_hi, blk);
    const long long j = (blk - blk_off[l]) * 32 + threadIdx.x;
    const bool real = j < (long long)list_len[l];
    const long long row = local_row_start[l - list_lo] + j;
    const long long id = real ? raw_ids[row - raw_row0] : -1;
    ids[blk * 32 + threadIdx.x] = id;
    if (real) { dm_ids[row] = id; dm_rows[row] = blk * 32 + threadIdx.x; }
}

void dph_free_lists(dph_index* ix) {
    void** ptrs[] = {(void**)&ix->list_len, (void**)&ix->list_start, (void**)&ix->blk_off, (void**)&ix->codes, (void**)&ix->ids,
                     (void**)&ix->dm_ids, (void**)&ix->dm_rows};
    for (void** p : ptrs) { if (*p) cudaFree(*p); *p = nullptr; }
    ix->blk_cap = ix->dm_cap = ix->dm_n = 0;
}

static int set_lists_common(dph_index* ix, const int64_t* list_len, const uint8_t* codes, const int64_t* ids, bool synthetic, uint64_t seed) {
    DPH_CUDA(cudaSetDevice(ix->device));
    DphLayout L;
    DPH_TRY(L.build(ix, list_len, "bad list length"));
    const int64_t nlist = ix->nlist, lo = ix->list_lo, hi = ix->list_hi, nb = L.nblocks, rows = L.rows;
    if (!synthetic && nb > 0) DPH_CHECK(codes != nullptr, "codes is null");
    const bool labels = ids && nb > 0;           // no ids: sequential labels (list_start[l] + j)
    // The call is valid: from here on the index changes.  The old arrays are freed before the new ones are allocated, so a re-set
    // needs room for one copy of the codes; if an allocation fails, the handle is left without lists.
    dph_free_lists(ix);
    auto alloc = [](auto** p, int64_t count) { return cudaMalloc((void**)p, std::max<int64_t>(count, 1) * sizeof(**p)); };
    DPH_CUDA(alloc(&ix->codes, nb * DPH_BLK_BYTES));
    if (labels) {
        DPH_CUDA(alloc(&ix->ids, nb * 32));
        DPH_CUDA(alloc(&ix->dm_ids, rows));
        DPH_CUDA(alloc(&ix->dm_rows, rows));
        ix->dm_cap = ix->dm_n = rows;
    }
    DPH_CUDA(alloc(&ix->list_len, nlist));
    DPH_CUDA(alloc(&ix->list_start, nlist + 1));
    DPH_CUDA(alloc(&ix->blk_off, nlist));
    ix->blk_cap = nb;
    DPH_TRY(dph_commit_layout(ix, std::move(L)));
    if (nb == 0) return 0;
    const DphLayout& lay = ix->lay;
    const long long* bo = (const long long*)ix->blk_off;
    if (synthetic) {
        for (int64_t b0 = 0; b0 < nb; b0 += (1ll << 30)) {          // grid.x limit
            const unsigned g = (unsigned)std::min<int64_t>(nb - b0, 1ll << 30);
            fill_blocks_kernel<<<g, 192, 0, ix->stream>>>(ix->codes, std::min<int64_t>(nb, b0 + g), bo, ix->list_len, lo, hi, nullptr, nullptr, seed, b0, 0);
        }
        DPH_CUDA(cudaGetLastError());
    } else {
        // Upload in chunks of whole lists through a bounded staging buffer (<= ~256 MB of rows): the raw list-major copy never
        // sits on the device next to the blocked one.  Labels go the same way; the direct map (faiss DirectMap::Hashtable,
        // build_phrase_index.py:139-141) is filled by the same kernel and sorted ON THE DEVICE.
        int64_t max_rows;
        const std::vector<DphLayout::Chunk> chunks = lay.chunks(&max_rows);
        DevTmp tmp;
        const char* oom = "set_lists: staging";
        uint8_t* d_raw; int64_t *d_lrs, *d_rawids = nullptr;
        DPH_TRY(tmp.alloc(&d_raw, (size_t)max_rows * DPH_CODE, oom));
        DPH_TRY(tmp.alloc(&d_lrs, lay.row_start.size(), oom));
        if (labels) DPH_TRY(tmp.alloc(&d_rawids, (size_t)max_rows, oom));
        DPH_CUDA(cudaMemcpy(d_lrs, lay.row_start.data(), lay.row_start.size() * 8, cudaMemcpyHostToDevice));
        for (const DphLayout::Chunk& c : chunks) {
            DPH_CUDA(cudaMemcpyAsync(d_raw, codes + (size_t)c.row0 * DPH_CODE, (size_t)c.rows * DPH_CODE, cudaMemcpyHostToDevice, ix->stream));
            fill_blocks_kernel<<<(unsigned)(c.blk1 - c.blk0), 192, 0, ix->stream>>>(ix->codes, c.blk1, bo, ix->list_len, lo, hi, d_raw,
                                                                                     (const long long*)d_lrs, 0, c.blk0, c.row0);
            if (labels) {
                DPH_CUDA(cudaMemcpyAsync(d_rawids, ids + c.row0, (size_t)c.rows * 8, cudaMemcpyHostToDevice, ix->stream));
                fill_ids_kernel<<<(unsigned)(c.blk1 - c.blk0), 32, 0, ix->stream>>>((long long*)ix->ids, c.blk1, bo, ix->list_len, lo, hi,
                                                                                     (const long long*)d_rawids, (const long long*)d_lrs, c.blk0,
                                                                                     c.row0, (long long*)ix->dm_ids, (long long*)ix->dm_rows);
            }
            DPH_CUDA(cudaGetLastError());
            DPH_CUDA(cudaStreamSynchronize(ix->stream));       // the staging buffers are reused by the next chunk
        }
        if (labels) {
            thrust::device_ptr<long long> kp((long long*)ix->dm_ids), vp((long long*)ix->dm_rows);
            thrust::sort_by_key(thrust::cuda::par.on(ix->stream), kp, kp + rows, vp);
        }
    }
    DPH_CUDA(cudaStreamSynchronize(ix->stream));
    return 0;
}
DPH_API int dph_index_set_lists(dph_index* ix, const int64_t* list_len, const uint8_t* codes, const int64_t* ids) {
    return set_lists_common(ix, list_len, codes, ids, false, 0);
}
DPH_API int dph_index_set_lists_synthetic(dph_index* ix, const int64_t* list_len, uint64_t seed) {
    return set_lists_common(ix, list_len, nullptr, nullptr, true, seed);
}

// -------------------------------------------------------------------------------------------------
// add_with_ids (DESIGN.md 3, "Growing the index").  The batch is encoded (encode.cu), then the shard's lists are laid out again into
// buffers of the exact new size.  Old rows keep their offsets j inside their list, so every old 3 KB block moves whole; the new rows
// follow in input order.  The result is byte-identical to set_lists of the concatenated list-major arrays.
// -------------------------------------------------------------------------------------------------
__global__ void iota_kernel(long long* out, long long n, long long base) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = base + i;
}
// flag bits: 2 = negative label, 4 = unassigned vector; cnt[l] += new rows of list l
__global__ void add_validate_kernel(const long long* list_no, const long long* ids, long long n, int* flag, int* cnt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long l = list_no[i];
    if (l < 0) atomicOr(flag, 4);
    else atomicAdd(&cnt[l], 1);
    if (ids[i] < 0) atomicOr(flag, 2);
}

// one CTA per block of the new layout: old blocks move whole (same rows, same lanes), blocks past a list's old end start as zeros
__global__ void __launch_bounds__(192) relayout_codes_kernel(uint8_t* dst, long long blk0, const long long* boff_new, const long long* boff_old,
                                                             const int* len_old, long long lo, long long hi, const uint8_t* codes_old) {
    const long long blk = blk0 + blockIdx.x;
    __shared__ long long s_l;
    if (threadIdx.x == 0) s_l = list_of_block(boff_new, lo, hi, blk);
    __syncthreads();
    const long long l = s_l, b = blk - boff_new[l];
    uint4 v = make_uint4(0, 0, 0, 0);
    if (b < ((long long)len_old[l] + 31) / 32) v = reinterpret_cast<const uint4*>(codes_old + (boff_old[l] + b) * DPH_BLK_BYTES)[threadIdx.x];
    reinterpret_cast<uint4*>(dst + (long long)blockIdx.x * DPH_BLK_BYTES)[threadIdx.x] = v;
}
// labels of the new layout's old rows (-1 elsewhere; the new rows are written by add_scatter_kernel).  Implicit labels (ids_old null)
// become explicit: list_start_old[l] + j, with their direct-map pairs at the row's old local position (already in label order) unless
// dm_ids is null (the merge builds its direct map from the labels' order instead).
__global__ void relayout_ids_kernel(long long* dst, long long blk0, const long long* boff_new, const long long* boff_old, const int* len_old,
                                    long long lo, long long hi, const long long* ids_old, const long long* list_start_old,
                                    const long long* lrs_old, long long* dm_ids, long long* dm_rows) {
    const long long blk = blk0 + blockIdx.x;
    const long long l = list_of_block(boff_new, lo, hi, blk), b = blk - boff_new[l];
    const long long j = b * 32 + threadIdx.x;
    long long id = -1;
    if (j < (long long)len_old[l]) {
        if (ids_old) id = ids_old[(boff_old[l] + b) * 32 + threadIdx.x];
        else {
            id = list_start_old[l] + j;
            if (dm_ids) {
                dm_ids[lrs_old[l - lo] + j] = id;
                dm_rows[lrs_old[l - lo] + j] = blk * 32 + threadIdx.x;
            }
        }
    }
    dst[(long long)blockIdx.x * 32 + threadIdx.x] = id;
}
// existing direct-map pairs (explicit labels): old padded row -> the same (list, j) in the new layout
__global__ void remap_dm_kernel(const long long* dm_ids_old, const long long* dm_rows_old, long long cnt, const long long* boff_old,
                                const long long* boff_new, long long lo, long long hi, long long* dm_ids_new, long long* dm_rows_new) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    const long long prow = dm_rows_old[i], ob = prow >> 5;
    const long long l = list_of_block(boff_old, lo, hi, ob);
    dm_ids_new[i] = dm_ids_old[i];
    dm_rows_new[i] = ((boff_new[l] + ob - boff_old[l]) << 5) | (prow & 31);
}
// new row of sorted position s (rows sorted stably by list: input order inside a list) -> j = old length + rank inside the batch.
// Its direct-map pair goes to slot dm0 + (input row), so that equal labels keep insertion order through the stable sort; rows of
// lists outside the shard get a sentinel label that sorts past the live entries.
__global__ void add_scatter_kernel(long long n, const long long* sorted_list, const long long* perm, const long long* bstart, const int* len_old,
                                   const long long* boff_new, long long lo, long long hi, const uint8_t* codes_all, const long long* ids_all,
                                   uint8_t* codes_new, long long* ids_new, long long* dm_ids, long long* dm_rows, long long dm0) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const long long l = sorted_list[s], r = perm[s];
    if (l < lo || l >= hi) { dm_ids[dm0 + r] = 0x7FFFFFFFFFFFFFFFll; dm_rows[dm0 + r] = -1; return; }
    const long long j = (long long)len_old[l] + (s - bstart[l]);
    const long long blk = boff_new[l] + (j >> 5);
    const int lane = (int)(j & 31);
    uint4 row4[6];
#pragma unroll
    for (int c = 0; c < 6; c++) row4[c] = reinterpret_cast<const uint4*>(codes_all + r * DPH_CODE)[c];
    dph_store_row(codes_new, blk, lane, reinterpret_cast<const unsigned char*>(row4));
    const long long id = ids_all[r];
    ids_new[blk * 32 + lane] = id;
    dm_ids[dm0 + r] = id;
    dm_rows[dm0 + r] = blk * 32 + lane;
}

DPH_API int dph_index_add_with_ids(dph_index* ix, const float* x, int64_t n, const int64_t* ids, int mem) {
    DPH_TRY(check_ready(ix, 1));
    DPH_CHECK(n >= 0, "add_with_ids: n must be >= 0");
    DPH_CUDA(cudaSetDevice(ix->device));
    if (n == 0) return 0;
    cudaStream_t st = ix->stream;
    const int64_t nlist = ix->nlist, lo = ix->list_lo, hi = ix->list_hi;
    for (float& a : ix->add_ms) a = 0.f;
    DevTmp tmp;
    const char* oom = "add_with_ids: not enough device memory for the batch; the index is unchanged";
    int64_t *list_all, *ids_all; uint8_t* codes_all; int *flag, *cnt;
    DPH_TRY(tmp.alloc(&list_all, n, oom)); DPH_TRY(tmp.alloc(&ids_all, n, oom)); DPH_TRY(tmp.alloc(&codes_all, (size_t)n * DPH_M, oom));
    DPH_TRY(tmp.alloc(&flag, 1, oom)); DPH_TRY(tmp.alloc(&cnt, nlist, oom));
    DPH_CUDA(cudaMemsetAsync(flag, 0, 4, st));
    DPH_CUDA(cudaMemsetAsync(cnt, 0, nlist * 4, st));
    // 1. assign + encode (host input: bounded staging, one encode chunk at a time)
    if (mem == DPH_MEM_DEVICE) DPH_TRY(dph_encode_rows(ix, x, n, list_all, codes_all, flag));
    else {
        const int64_t cs = std::min(dph_encode_chunk(ix), n);
        DPH_TRY(ix->xdev.ensure((size_t)cs * ix->d * 4));
        for (int64_t o = 0; o < n; o += cs) {
            const int64_t m = std::min(cs, n - o);
            DPH_CUDA(cudaMemcpyAsync(ix->xdev.p, x + o * ix->d, (size_t)m * ix->d * 4, cudaMemcpyHostToDevice, st));
            DPH_TRY(dph_encode_rows(ix, ix->xdev.as<float>(), m, list_all + o, codes_all + o * DPH_M, flag));
        }
    }
    if (ids) DPH_CUDA(cudaMemcpyAsync(ids_all, ids, (size_t)n * 8, mem == DPH_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, st));
    else iota_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((long long*)ids_all, n, ix->ntotal);        // IndexIVF::add: ntotal + i
    add_validate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const long long*)list_all, (const long long*)ids_all, n, flag, cnt);
    DPH_CUDA(cudaGetLastError());
    int h_flag = 0;
    std::vector<int32_t> h_cnt(nlist);
    DPH_CUDA(cudaMemcpyAsync(&h_flag, flag, 4, cudaMemcpyDeviceToHost, st));
    DPH_CUDA(cudaMemcpyAsync(h_cnt.data(), cnt, nlist * 4, cudaMemcpyDeviceToHost, st));
    DPH_CUDA(cudaStreamSynchronize(st));
    DPH_CHECK(!(h_flag & 1), "add_with_ids: the input holds a non-finite value; the index is unchanged");
    DPH_CHECK(!(h_flag & 2), "add_with_ids: negative label (-1 marks padding rows); the index is unchanged");
    DPH_CHECK(!(h_flag & 4), "add_with_ids: a vector has no best list; the index is unchanged");

    // 2. the new layout: every list's length (all shards), this shard's tightly packed blocks
    std::vector<int64_t> len_new(nlist), bstart(nlist, 0);
    for (int64_t l = 0; l < nlist; l++) {
        len_new[l] = ix->lay.len[l] + h_cnt[l];
        if (l + 1 < nlist) bstart[l + 1] = bstart[l] + h_cnt[l];
    }
    DphLayout L;
    DPH_TRY(L.build(ix, len_new.data(), "add_with_ids: a list would exceed 2^31 - 1 rows; the index is unchanged"));
    const DphLayout& old = ix->lay;
    const int64_t nb = L.nblocks;
    const bool was_explicit = ix->ids != nullptr;
    const int64_t dm_old = was_explicit ? ix->dm_n : ix->ntotal_local;       // pairs carried over
    const int64_t dm_cap = dm_old + n, dm_n = dm_old + (L.rows - old.rows);

    // 3. every new buffer before anything changes: a failed allocation leaves the index as it was
    const char* oom2 = "add_with_ids: not enough device memory for the re-layout (the old and the new code buffers of the shard are live "
                       "together); the index is unchanged";
    uint8_t* codes_new; int64_t *ids_new, *dm_ids_new, *dm_rows_new, *d_boff_new, *d_bstart, *d_lrs, *perm;
    DPH_TRY(tmp.alloc(&codes_new, (size_t)nb * DPH_BLK_BYTES, oom2)); DPH_TRY(tmp.alloc(&ids_new, (size_t)nb * 32, oom2));
    DPH_TRY(tmp.alloc(&dm_ids_new, dm_cap, oom2)); DPH_TRY(tmp.alloc(&dm_rows_new, dm_cap, oom2));
    DPH_TRY(tmp.alloc(&d_boff_new, nlist, oom2)); DPH_TRY(tmp.alloc(&d_bstart, nlist, oom2));
    DPH_TRY(tmp.alloc(&d_lrs, old.row_start.size(), oom2)); DPH_TRY(tmp.alloc(&perm, n, oom2));
    DPH_CUDA(cudaMemcpyAsync(d_boff_new, L.blk_off.data(), nlist * 8, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemcpyAsync(d_bstart, bstart.data(), nlist * 8, cudaMemcpyHostToDevice, st));
    DPH_CUDA(cudaMemcpyAsync(d_lrs, old.row_start.data(), old.row_start.size() * 8, cudaMemcpyHostToDevice, st));

    // 4. move the old blocks, scatter the new rows, merge the direct map
    const bool prof = ix->profile && ix->aev[0];
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[4], st));
    const long long *bo_new = (const long long*)d_boff_new, *bo_old = (const long long*)ix->blk_off;
    if (nb > 0) {
        relayout_codes_kernel<<<(unsigned)nb, 192, 0, st>>>(codes_new, 0, bo_new, bo_old, ix->list_len, lo, hi, ix->codes);
        relayout_ids_kernel<<<(unsigned)nb, 32, 0, st>>>((long long*)ids_new, 0, bo_new, bo_old, ix->list_len, lo, hi, (const long long*)ix->ids,
                                                       (const long long*)ix->list_start, (const long long*)d_lrs, (long long*)dm_ids_new,
                                                       (long long*)dm_rows_new);
    }
    if (was_explicit && ix->dm_n > 0)
        remap_dm_kernel<<<(unsigned)((ix->dm_n + 255) / 256), 256, 0, st>>>((const long long*)ix->dm_ids, (const long long*)ix->dm_rows, ix->dm_n,
                                                                           bo_old, bo_new, lo, hi, (long long*)dm_ids_new, (long long*)dm_rows_new);
    DPH_CUDA(cudaGetLastError());
    try {
        thrust::device_ptr<long long> kp((long long*)list_all), pp((long long*)perm);
        thrust::sequence(thrust::cuda::par.on(st), pp, pp + n);
        thrust::stable_sort_by_key(thrust::cuda::par.on(st), kp, kp + n, pp);
        add_scatter_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n, (const long long*)list_all, (const long long*)perm, (const long long*)d_bstart,
                                                                       ix->list_len, bo_new, lo, hi, codes_all, (const long long*)ids_all, codes_new,
                                                                       (long long*)ids_new, (long long*)dm_ids_new, (long long*)dm_rows_new, dm_old);
        DPH_CUDA(cudaGetLastError());
        thrust::device_ptr<long long> dk((long long*)dm_ids_new), dv((long long*)dm_rows_new);
        thrust::stable_sort_by_key(thrust::cuda::par.on(st), dk, dk + dm_cap, dv);       // equal labels keep insertion order
    } catch (const std::exception& e) {
        cudaGetLastError();
        dph_set_error(std::string("add_with_ids: device sort failed; the index is unchanged: ") + e.what());
        return 1;
    }
    if (prof) DPH_CUDA(cudaEventRecord(ix->aev[5], st));
    DPH_CUDA(cudaStreamSynchronize(st));

    // 5. commit: tables, then the buffers
    DPH_TRY(dph_commit_layout(ix, std::move(L)));
    void* olds[] = {ix->codes, ix->ids, ix->dm_ids, ix->dm_rows};
    for (void* p : olds) if (p) cudaFree(p);
    ix->codes = codes_new; ix->ids = ids_new; ix->dm_ids = dm_ids_new; ix->dm_rows = dm_rows_new;
    for (void* p : {(void*)codes_new, (void*)ids_new, (void*)dm_ids_new, (void*)dm_rows_new}) tmp.release(p);
    ix->dm_n = dm_n; ix->dm_cap = dm_cap; ix->blk_cap = nb;
    if (prof) DPH_CUDA(cudaEventElapsedTime(&ix->add_ms[3], ix->aev[4], ix->aev[5]));
    return 0;
}

// The inverse of set_lists: this shard's rows as list-major host arrays, through the same bounded staging.
__global__ void __launch_bounds__(192) read_blocks_kernel(const uint8_t* codes, long long nblocks, const long long* blk_off, const int* list_len,
                                                          long long list_lo, long long list_hi, const long long* ids, const long long* list_start,
                                                          const long long* local_row_start, long long blk0, long long raw_row0, uint8_t* raw,
                                                          long long* raw_ids) {
    const long long blk = blk0 + blockIdx.x;
    if (blk >= nblocks) return;
    const int lane = threadIdx.x & 31, c = threadIdx.x >> 5;
    __shared__ long long s_l;
    if (threadIdx.x == 0) s_l = list_of_block(blk_off, list_lo, list_hi, blk);
    __syncthreads();
    const long long l = s_l;
    const long long j = (blk - blk_off[l]) * 32 + lane;
    if (j >= (long long)list_len[l]) return;
    const long long row = local_row_start[l - list_lo] + j - raw_row0;
    const uint4 v = *reinterpret_cast<const uint4*>(codes + blk * DPH_BLK_BYTES + c * 512 + lane * 16);
    unsigned char bytes[16];
    memcpy(bytes, &v, 16);
#pragma unroll
    for (int b = 0; b < 16; b++) raw[row * DPH_CODE + dph_blk_sub(lane, c * 16 + b)] = bytes[b];
    if (c == 0 && raw_ids) raw_ids[row] = ids ? ids[blk * 32 + lane] : list_start[l] + j;
}

DPH_API int dph_index_copy_lists(dph_index* ix, uint8_t* codes_out, int64_t* ids_out) {
    DPH_CHECK(ix && ix->list_len, "copy_lists: lists are not set");
    DPH_CUDA(cudaSetDevice(ix->device));
    if (ix->ntotal_local == 0) return 0;
    const DphLayout& L = ix->lay;
    int64_t max_rows;
    const std::vector<DphLayout::Chunk> chunks = L.chunks(&max_rows);
    DevTmp tmp;
    uint8_t* d_raw; int64_t *d_ids, *d_lrs;
    DPH_TRY(tmp.alloc(&d_raw, (size_t)max_rows * DPH_CODE, "copy_lists: staging"));
    DPH_TRY(tmp.alloc(&d_ids, (size_t)max_rows, "copy_lists: staging"));
    DPH_TRY(tmp.alloc(&d_lrs, L.row_start.size(), "copy_lists: staging"));
    DPH_CUDA(cudaMemcpyAsync(d_lrs, L.row_start.data(), L.row_start.size() * 8, cudaMemcpyHostToDevice, ix->stream));
    for (const DphLayout::Chunk& c : chunks) {
        read_blocks_kernel<<<(unsigned)(c.blk1 - c.blk0), 192, 0, ix->stream>>>(ix->codes, c.blk1, (const long long*)ix->blk_off, ix->list_len,
                                                                                L.lo, L.hi, (const long long*)ix->ids, (const long long*)ix->list_start,
                                                                                (const long long*)d_lrs, c.blk0, c.row0, d_raw,
                                                                                ids_out ? (long long*)d_ids : nullptr);
        DPH_CUDA(cudaGetLastError());
        DPH_CUDA(cudaMemcpyAsync(codes_out + (size_t)c.row0 * DPH_CODE, d_raw, (size_t)c.rows * DPH_CODE, cudaMemcpyDeviceToHost, ix->stream));
        if (ids_out) DPH_CUDA(cudaMemcpyAsync(ids_out + c.row0, d_ids, (size_t)c.rows * 8, cudaMemcpyDeviceToHost, ix->stream));
        DPH_CUDA(cudaStreamSynchronize(ix->stream));          // the staging buffers are reused by the next chunk
    }
    return 0;
}

DPH_API int dph_index_get_list_len(const dph_index* ix, int64_t* list_len_out) {
    DPH_CHECK(ix && ix->list_len, "lists are not set");
    std::copy(ix->lay.len.begin(), ix->lay.len.end(), list_len_out);
    return 0;
}
DPH_API int dph_index_last_add_ms(const dph_index* ix, float* ms_out) {
    DPH_CHECK(ix->aev[0] != nullptr, "profiling was never enabled");
    std::copy(ix->add_ms, ix->add_ms + 4, ms_out);
    return 0;
}
