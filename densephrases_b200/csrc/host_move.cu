// host_move.cu -- mutable host indexes (DESIGN.md 3.5, "Mutable host indexes"): the reserved host capacity and the in-place block
// mover that add, remove and merge use to re-lay the page-locked code array without a second copy of it.
//
// Why in place is safe.  The new layout of an add or a merge only grows lists, so every list's first block moves up or stays
// (blk_off_new[l] >= blk_off_old[l]): each destination block's source is at or below it.  The remove's block shift only shrinks them,
// so each source is at or above its destination.  The destination blocks [d_first, nblocks) are rewritten in chunks of whole blocks,
// descending for growth and ascending for the shift, each chunk gathered into an HBM staging buffer before any of it is written back.
// Ordering rule: a chunk's write-back starts only after its own gather and after the gathers of every earlier chunk.  For growth,
// chunk i + 1 gathers only below d0(i) while chunk i writes at or above d0(i); an earlier chunk may gather from below its own d0, i.e.
// from a later chunk's destinations, which the rule keeps intact until that gather is done.  A chunk's own sources may overlap its
// destinations: it is staged whole first.  The shift is the mirror image.  Two buffers, a gather stream and a write-back stream: chunk
// i + 1's gather (PCIe host-to-device) overlaps chunk i's write-back (device-to-host).
#include "index_internal.cuh"

// One warp per destination block [blk0, blk0 + nblk) of the layout boff_new: the same list's block of boff_old in src (whole, same rows
// and lanes; zeros past the list's old end) into dst[0 ..).  Each lane issues its six 16-byte loads before any store
// (fetch_lists_kernel), so that a warp keeps a whole block in flight over PCIe when src is mapped host memory.
__global__ void __launch_bounds__(256) host_gather_kernel(uint8_t* __restrict__ dst, long long blk0, long long nblk,
                                                          const long long* __restrict__ boff_new, const long long* __restrict__ boff_old,
                                                          const int* __restrict__ len_old, long long lo, long long hi,
                                                          const uint8_t* __restrict__ src) {
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long i = w0; i < nblk; i += nw) {
        const long long blk = blk0 + i;
        const long long l = list_of_block(boff_new, lo, hi, blk), b = blk - boff_new[l];
        uint4 v[6];
        if (b < ((long long)len_old[l] + 31) / 32) {
            const uint4* s = reinterpret_cast<const uint4*>(src + (boff_old[l] + b) * DPH_BLK_BYTES) + lane;
#pragma unroll
            for (int c = 0; c < 6; c++) v[c] = s[c * 32];
        } else {
#pragma unroll
            for (int c = 0; c < 6; c++) v[c] = make_uint4(0, 0, 0, 0);
        }
        uint4* d = reinterpret_cast<uint4*>(dst + i * DPH_BLK_BYTES) + lane;
#pragma unroll
        for (int c = 0; c < 6; c++) d[c * 32] = v[c];
    }
}

int64_t dph_first_changed_block(const DphLayout& old, const DphLayout& nw) {
    for (int64_t l = nw.lo; l < nw.hi; l++) {
        if (nw.blk_off[l] != old.blk_off[l]) return nw.blk_off[l];
        if (nw.len[l] != old.len[l]) return nw.blk_off[l] + std::min(nw.len[l], old.len[l]) / 32;
    }
    return nw.nblocks;
}

bool dph_shard_changed(const dph_index* ix, const DphLayout& nw) {
    for (int64_t l = nw.lo; l < nw.hi; l++)
        if (nw.len[l] != ix->lay.len[l]) return true;
    return false;
}

int dph_host_capacity_check(const dph_index* ix, const DphLayout& nw, const char* what) {
    if (!ix->on_host || nw.nblocks <= ix->host_blocks) return 0;
    dph_set_error(std::string(what) + ": the new layout needs " + std::to_string(nw.nblocks * DPH_BLK_BYTES) +
                  " bytes of host codes; the reserved host capacity is " + std::to_string(ix->host_blocks * DPH_BLK_BYTES) +
                  " bytes (reserve_host_codes); the index is unchanged");
    return 1;
}

DphHostMover::~DphHostMover() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (ws) cudaStreamDestroy(ws);
    if (rs) cudaStreamDestroy(rs);
}

int DphHostMover::prepare(dph_index* ix, DevTmp& tmp, int64_t blocks, const char* oom) {
    if (blocks <= 0) return 0;
    chunk_blocks = std::max<int64_t>(1, std::min<int64_t>(dph_chunk_rows() * DPH_CODE / DPH_BLK_BYTES, blocks));
    DPH_TRY(tmp.alloc(&buf[0], (size_t)chunk_blocks * DPH_BLK_BYTES, oom));
    DPH_TRY(tmp.alloc(&buf[1], (size_t)chunk_blocks * DPH_BLK_BYTES, oom));
    DPH_CUDA(cudaStreamCreateWithFlags(&rs, cudaStreamNonBlocking));
    DPH_CUDA(cudaStreamCreateWithFlags(&ws, cudaStreamNonBlocking));
    DPH_CUDA(cudaEventCreate(&ev[0]));
    DPH_CUDA(cudaEventCreate(&ev[1]));
    for (int i = 2; i < 6; i++) DPH_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    return 0;
}

int DphHostMover::run(dph_index* ix, const DphLayout& nw, int64_t d_first, const long long* boff_new, bool grow, const StageFn& stage) {
    const DphLayout& old = ix->lay;
    const int64_t nb = nw.nblocks;
    for (int64_t& c : ix->move_counts) c = 0;
    ix->move_ms = 0.f;
    if (d_first >= nb) return 0;
    for (int64_t l = nw.lo; l < nw.hi; l++) {          // blocks gathered from the host array: those with an old source block
        const int64_t b0 = nw.blk_off[l], nbl = std::min((nw.len[l] + 31) / 32, (old.len[l] + 31) / 32);
        ix->move_counts[0] += std::max<int64_t>(0, b0 + nbl - std::max(b0, d_first));
    }
    cudaEvent_t &e_start = ev[0], &e_end = ev[1], *e_read = ev + 2, *e_write = ev + 4;
    const int64_t total = nb - d_first, nchunks = (total + chunk_blocks - 1) / chunk_blocks;
    DPH_CUDA(cudaEventRecord(e_start, ix->stream));    // the caller's earlier work on the array (hole fills, tail clears) is done
    DPH_CUDA(cudaStreamWaitEvent(rs, e_start, 0));
    DPH_CUDA(cudaStreamWaitEvent(ws, e_start, 0));
    for (int64_t i = 0; i < nchunks; i++) {
        const int64_t c0 = grow ? std::max(d_first, nb - (i + 1) * chunk_blocks) : d_first + i * chunk_blocks;
        const int64_t c1 = grow ? nb - i * chunk_blocks : std::min(nb, c0 + chunk_blocks);
        const int b = (int)(i & 1);
        if (i >= 2) DPH_CUDA(cudaStreamWaitEvent(rs, e_write[b], 0));      // buffer b's previous write-back is done
        const unsigned grid = (unsigned)std::min<int64_t>((c1 - c0 + 7) / 8, (int64_t)ix->num_sms * 8);
        host_gather_kernel<<<grid, 256, 0, rs>>>(buf[b], c0, c1 - c0, boff_new, (const long long*)ix->blk_off, ix->list_len, nw.lo, nw.hi,
                                                 ix->codes);
        DPH_CUDA(cudaGetLastError());
        if (stage) DPH_TRY(stage(buf[b], c0, c1, rs));
        // The gather stream runs in order, so this event marks chunk i's gather AND the gathers of every earlier chunk: the ordering
        // rule above.  (Waiting on chunk i's own gather only would let its write-back overwrite an earlier chunk's unread sources.)
        DPH_CUDA(cudaEventRecord(e_read[b], rs));
        DPH_CUDA(cudaStreamWaitEvent(ws, e_read[b], 0));
        DPH_CUDA(cudaMemcpyAsync(ix->host_codes + (size_t)c0 * DPH_BLK_BYTES, buf[b], (size_t)(c1 - c0) * DPH_BLK_BYTES, cudaMemcpyDeviceToHost, ws));
        DPH_CUDA(cudaEventRecord(e_write[b], ws));
    }
    DPH_CUDA(cudaEventRecord(e_end, ws));
    DPH_CUDA(cudaStreamWaitEvent(ix->stream, e_end, 0));
    DPH_CUDA(cudaEventSynchronize(e_end));
    DPH_CUDA(cudaEventElapsedTime(&ix->move_ms, e_start, e_end));
    ix->move_counts[1] = total; ix->move_counts[2] = nchunks;
    return 0;
}

DPH_API int dph_index_reserve_host_codes(dph_index* ix, int64_t bytes) {
    DPH_CHECK(ix && ix->on_host, "reserve_host_codes: needs an index whose codes are in host memory (set_code_residency first)");
    DPH_CHECK(bytes >= 0, "reserve_host_codes: bytes must be >= 0; the index is unchanged");
    DPH_CUDA(cudaSetDevice(ix->device));
    const int64_t want = bytes / DPH_BLK_BYTES;
    if (ix->host_codes && want > ix->host_blocks) {      // a larger array: the blocks move over, the old array goes
        uint8_t *h = nullptr, *d = nullptr;
        cudaError_t e = cudaHostAlloc((void**)&h, (size_t)want * DPH_BLK_BYTES, cudaHostAllocMapped);
        if (e == cudaSuccess) e = cudaHostGetDevicePointer((void**)&d, h, 0);
        if (e != cudaSuccess) {
            cudaGetLastError();
            if (h) cudaFreeHost(h);
            dph_set_error(std::string("reserve_host_codes: cannot allocate ") + std::to_string(want * DPH_BLK_BYTES) +
                          " bytes of page-locked host memory: " + cudaGetErrorString(e) + "; the index is unchanged");
            return 1;
        }
        DPH_CUDA(cudaStreamSynchronize(ix->stream));     // reads of the old array still in flight
        memcpy(h, ix->host_codes, (size_t)ix->nblocks_local * DPH_BLK_BYTES);
        cudaFreeHost(ix->host_codes);
        ix->host_codes = h; ix->codes = d; ix->host_blocks = want;
    }
    ix->host_reserve = std::max(ix->host_reserve, want);
    ix->host_mutable = true;
    return 0;
}

DPH_API int dph_index_last_host_move(const dph_index* ix, int64_t* counts, float* ms) {
    DPH_CHECK(ix && ix->on_host, "last_host_move: the codes of this index are in device memory");
    std::copy(ix->move_counts, ix->move_counts + 3, counts);
    if (ms) *ms = ix->move_ms;
    return 0;
}
