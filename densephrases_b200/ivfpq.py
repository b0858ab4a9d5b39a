"""IvfPqIndex: Python handle over the C-ABI index (include/dph_b200.h).

Mirrors the slice of the faiss Python API that reference densephrases/index.py uses on the hot path:
``search(x, k) -> (D, I)`` (index.py:200), ``reconstruct`` (index.py:31,286,296), ``ntotal``, ``d``, ``nprobe``
(index.py:33,53,62), the OPQ matrix (index.py:32).  numpy in -> numpy out through the C ABI with host buffers;
torch CUDA tensors in -> torch CUDA tensors out (device pointers, asynchronous on the current stream)."""
import contextlib
import ctypes as C

import numpy as np

from . import _lib as L


def _np_ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def default_stream_bytes(list_len, lo=0, hi=None):
    """The stream region a host-mode index gets when none is given: 1 GiB, or the largest list of lists [lo, hi) if that is more."""
    list_len = np.asarray(list_len, dtype=np.int64)[lo:hi]
    largest = int(list_len.max()) if len(list_len) else 0
    return max(1 << 30, (largest + 31) // 32 * 3072)


class IvfPqIndex:
    def __init__(self, nlist, d=768, M=96, nbits=8, device=0):
        self._h = C.c_void_p()
        L.check(L.lib().dph_index_create(C.byref(self._h), d, nlist, M, nbits, device))
        self.device = device
        self.shard = (0, nlist)             # this handle's lists [lo, hi) (set_shard)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and L is not None and getattr(L, "_lib", None) is not None:      # interpreter shutdown: the module may already be gone
            L._lib.dph_index_free(h)

    @classmethod
    def from_arrays(cls, A, centroids, pq, list_len, codes, ids=None, device=0, shard=None, codes_on_host=False, stream_bytes=None,
                    host_capacity_bytes=None):
        """Build from the arrays a faiss IndexPreTransform(OPQ)->IndexIVFPQ file holds (index.py:30).  codes_on_host: keep the codes in
        page-locked host memory and stream the probed lists through a device region of stream_bytes (None: default_stream_bytes);
        see set_code_residency.  host_capacity_bytes (host mode only): reserve that much page-locked memory for the codes, which makes
        the index mutable; see reserve_host_codes."""
        if host_capacity_bytes is not None and not codes_on_host:
            raise ValueError("host_capacity_bytes needs codes_on_host=True")
        ix = cls(len(list_len), device=device)
        ix.set_opq(A)
        ix.set_centroids(centroids)
        ix.set_pq(pq)
        if shard is not None:
            ix.set_shard(*shard)
        if codes_on_host:
            ix.set_code_residency(True, default_stream_bytes(list_len, *(shard or (0, None))) if stream_bytes is None else stream_bytes)
            if host_capacity_bytes is not None:
                ix.reserve_host_codes(host_capacity_bytes)
        ix.set_lists(list_len, codes, ids)
        return ix

    # ---- construction -----------------------------------------------------------------------
    def set_opq(self, A):
        A = np.ascontiguousarray(A, dtype=np.float32)
        assert A.shape == (self.d, self.d)
        L.check(L.lib().dph_index_set_opq(self._h, _np_ptr(A), L.MEM_HOST))

    def set_centroids(self, Cm):
        Cm = np.ascontiguousarray(Cm, dtype=np.float32)
        assert Cm.shape == (self.nlist, self.d)
        L.check(L.lib().dph_index_set_centroids(self._h, _np_ptr(Cm), L.MEM_HOST))

    def set_pq(self, pq):
        pq = np.ascontiguousarray(pq, dtype=np.float32)
        assert pq.shape == (96, 256, 8)
        L.check(L.lib().dph_index_set_pq(self._h, _np_ptr(pq), L.MEM_HOST))

    def gen_centroids(self, seed, sigma=0.5):
        L.check(L.lib().dph_index_gen_centroids(self._h, seed, sigma))

    def gen_pq(self, seed, sigma=0.25):
        L.check(L.lib().dph_index_gen_pq(self._h, seed, sigma))

    def set_shard(self, lo, hi):
        L.check(L.lib().dph_index_set_shard(self._h, lo, hi))
        self.shard = (int(lo), int(hi))

    def set_lists(self, list_len, codes, ids=None):
        list_len = np.ascontiguousarray(list_len, dtype=np.int64)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if ids is not None:
            ids = np.ascontiguousarray(ids, dtype=np.int64)
        L.check(L.lib().dph_index_set_lists(self._h, _np_ptr(list_len), _np_ptr(codes), None if ids is None else _np_ptr(ids)))

    def set_lists_synthetic(self, list_len, seed):
        list_len = np.ascontiguousarray(list_len, dtype=np.int64)
        L.check(L.lib().dph_index_set_lists_synthetic(self._h, _np_ptr(list_len), seed))

    # ---- codes in host memory (DESIGN.md 3.5) ---------------------------------------------------
    def set_code_residency(self, on_host, stream_bytes=0):
        """on_host=True (before set_lists): the codes live in page-locked host memory; every search copies the probed lists that are
        not resident into a device stream region of stream_bytes, slice by slice, with results bit-identical to a device-resident
        index.  stream_bytes may be changed later.  The index is then read-only (add, remove, sync_list_len and merge raise
        RuntimeError) unless a host capacity is reserved with reserve_host_codes; it is never a merge source."""
        L.check(L.lib().dph_index_set_code_residency(self._h, int(bool(on_host)), int(stream_bytes)))

    def set_resident_lists(self, lists):
        """Host mode: keep these lists of this shard in device memory (replaces the previous set; [] empties it).  To choose them,
        count the probes of a sample search: ``np.bincount(ix.last_probes(n).ravel() + 1, minlength=nlist + 1)[1:]`` after
        ``ix.search(sample, k)``, and take the most probed lists whose code bytes (ceil(len / 32) * 3072 each) fit the device memory
        you can spare.  Raises RuntimeError, leaving the index unchanged, on a list outside the shard or too little device memory.
        An add, remove or merge that changes a list of this shard empties the resident set: the region keeps its device memory and
        serves as the stream region (every list streams) until this is called again."""
        lists = np.ascontiguousarray(np.asarray(lists, dtype=np.int64).ravel())
        L.check(L.lib().dph_index_set_resident_lists(self._h, _np_ptr(lists), len(lists)))

    def last_fetch(self):
        """Host mode: what the last search fetched, summed over its chunks -> dict(slices, lists_fetched, blocks_fetched,
        resident_lists_scanned, fetch_ms); fetch_ms is measured with set_profile(True) only."""
        counts = np.zeros(4, dtype=np.int64)
        ms = C.c_float(0)
        L.check(L.lib().dph_index_last_fetch(self._h, _np_ptr(counts), C.byref(ms)))
        return dict(slices=int(counts[0]), lists_fetched=int(counts[1]), blocks_fetched=int(counts[2]), resident_lists_scanned=int(counts[3]),
                    fetch_ms=ms.value)

    @property
    def host_bytes(self):
        """Bytes of page-locked host memory holding the codes (0 unless the codes are in host memory)."""
        return L.lib().dph_index_host_bytes(self._h)

    def reserve_host_codes(self, nbytes):
        """Host mode: reserve a page-locked capacity of nbytes for the codes (rounded down to whole 3 KB blocks; it never shrinks) and
        make the index mutable.  add_with_ids / add, remove_ids, sync_list_len and merge_from (from device-resident sources) then give
        exactly what they give on a device-resident index, re-laying the host array in place through two device staging buffers of at
        most ~256 MB; an add or merge that needs more than the capacity raises RuntimeError, the index unchanged.  Host memory stays
        the capacity the caller chose.  Before set_lists, set_lists allocates max(capacity, what the lists need).  After it, a larger
        capacity allocates a new array, copies the codes and frees the old one (the one time two host arrays exist; if the allocation
        fails, RuntimeError and the index is unchanged); a capacity at or below host_bytes only makes the index mutable.  A mutation
        that changes a list of this shard empties the resident set (see set_resident_lists)."""
        L.check(L.lib().dph_index_reserve_host_codes(self._h, int(nbytes)))

    def last_host_move(self):
        """Host mode: the in-place block mover of the last add, remove or merge -> dict(blocks_read, blocks_written, chunks, ms): 3 KB
        blocks gathered from and written back to the host array, staging chunks, and its time (first gather to last write-back)."""
        counts = np.zeros(3, dtype=np.int64)
        ms = C.c_float(0)
        L.check(L.lib().dph_index_last_host_move(self._h, _np_ptr(counts), C.byref(ms)))
        return dict(blocks_read=int(counts[0]), blocks_written=int(counts[1]), chunks=int(counts[2]), ms=ms.value)

    # ---- growing the index (faiss add_with_ids, build_phrase_index.py:145-150) --------------------
    def _rows(self, x):
        if len(x.shape) != 2 or x.shape[1] != self.d:
            raise RuntimeError(f"expected vectors of shape [n, {self.d}], got {tuple(x.shape)}")
        return int(x.shape[0])

    def encode(self, x):
        """Assign + encode without changing the index: numpy [n,d] -> (list_no [n] i64, codes [n,96] u8) numpy | torch cuda -> torch
        cuda.  Bit-identical to the oracle's ref_encode (DESIGN.md 3, "Growing the index")."""
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x, dtype=np.float32)
            n = self._rows(x)
            list_no = np.empty(n, dtype=np.int64)
            codes = np.empty((n, 96), dtype=np.uint8)
            L.check(L.lib().dph_index_encode(self._h, _np_ptr(x), n, _np_ptr(list_no), _np_ptr(codes), L.MEM_HOST))
            return list_no, codes
        import torch
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        n = self._rows(x)
        list_no = torch.empty(n, dtype=torch.int64, device=x.device)
        codes = torch.empty((n, 96), dtype=torch.uint8, device=x.device)
        self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
        L.check(L.lib().dph_index_encode(self._h, x.data_ptr(), n, list_no.data_ptr(), codes.data_ptr(), L.MEM_DEVICE))
        return list_no, codes

    def add_with_ids(self, x, ids):
        """== faiss index.add_with_ids(x, ids): append x [n,d] (numpy or torch cuda) with labels ids [n] (None: ntotal + arange(n))
        to their lists, in input order.  Raises RuntimeError, leaving the index unchanged, on a negative label, a non-finite value,
        a shape mismatch or too little device memory for the re-layout.  A host-mode index needs a reserved host capacity
        (reserve_host_codes) that holds the new layout."""
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x, dtype=np.float32)
            n = self._rows(x)
            if ids is not None:
                ids = np.ascontiguousarray(np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids), dtype=np.int64)
                if ids.shape != (n,):
                    raise RuntimeError(f"ids has shape {ids.shape}, expected ({n},)")
            L.check(L.lib().dph_index_add_with_ids(self._h, _np_ptr(x), n, None if ids is None else _np_ptr(ids), L.MEM_HOST))
            return
        import torch
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        n = self._rows(x)
        if ids is not None:
            ids = torch.as_tensor(ids, dtype=torch.int64).to(x.device).contiguous()
            if tuple(ids.shape) != (n,):
                raise RuntimeError(f"ids has shape {tuple(ids.shape)}, expected ({n},)")
        self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
        L.check(L.lib().dph_index_add_with_ids(self._h, x.data_ptr(), n, None if ids is None else ids.data_ptr(), L.MEM_DEVICE))

    def add_int8(self, q, ids, offset, scale):
        """add_with_ids of the rows x = q / scale + offset of int8 q [n,d], computed in fp32 as the reference's int8_to_float did under
        numpy 1.x: fl32(fl32(float(q) / fl32(scale)) + fl32(offset)) (DESIGN.md 3.8).  The index afterwards is byte-identical to
        add_with_ids of those rows.  q is numpy (pageable, or a view of page-locked memory, read in place), a torch CPU tensor
        (pinned or not) or a torch CUDA tensor; ids as for add_with_ids, on the same side.  Only int8 crosses PCIe.  Raises
        RuntimeError, leaving the index unchanged, on a scale that is zero or not finite in fp32, an offset that is not finite, and
        everything add_with_ids rejects."""
        with np.errstate(over="ignore"):
            off32, scale32 = float(np.float32(offset)), float(np.float32(scale))
        if isinstance(q, np.ndarray):
            if q.dtype != np.int8:
                raise RuntimeError(f"add_int8: q must be int8, got {q.dtype}")
            q = np.ascontiguousarray(q)
            n = self._rows(q)
            if ids is not None:
                ids = np.ascontiguousarray(np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids), dtype=np.int64)
                if ids.shape != (n,):
                    raise RuntimeError(f"ids has shape {ids.shape}, expected ({n},)")
            L.check(L.lib().dph_index_add_int8(self._h, _np_ptr(q), n, off32, scale32, None if ids is None else _np_ptr(ids), L.MEM_HOST))
            return
        import torch
        if q.dtype != torch.int8 or not q.is_contiguous():
            raise RuntimeError(f"add_int8: q must be a contiguous int8 tensor, got {q.dtype}")
        n = self._rows(q)
        if ids is not None:
            ids = torch.as_tensor(ids, dtype=torch.int64).to(q.device).contiguous()
            if tuple(ids.shape) != (n,):
                raise RuntimeError(f"ids has shape {tuple(ids.shape)}, expected ({n},)")
        mem = L.MEM_DEVICE if q.is_cuda else L.MEM_HOST
        if q.is_cuda:
            self.set_stream(torch.cuda.current_stream(q.device).cuda_stream)
        L.check(L.lib().dph_index_add_int8(self._h, q.data_ptr(), n, off32, scale32, None if ids is None else ids.data_ptr(), mem))

    def add(self, x):
        """== faiss index.add(x): labels ntotal + arange(n)."""
        self.add_with_ids(x, None)

    def lists(self):
        """-> (list_len [nlist] i64 of ALL lists, codes [ntotal_local,96] u8, ids [ntotal_local] i64): this shard's lists, list-major
        (the arrays set_lists / from_arrays / artifacts.write_faiss_index take)."""
        list_len = np.empty(self.nlist, dtype=np.int64)
        L.check(L.lib().dph_index_get_list_len(self._h, _np_ptr(list_len)))
        n = self.ntotal_local
        codes = np.empty((n, 96), dtype=np.uint8)
        ids = np.empty(n, dtype=np.int64)
        L.check(L.lib().dph_index_copy_lists(self._h, _np_ptr(codes), _np_ptr(ids)))
        return list_len, codes, ids

    def last_add_ms(self):
        """With set_profile(True): stage times of the last add in ms (rotation, coarse, PQ encode, re-layout + scatter)."""
        out = np.zeros(4, dtype=np.float32)
        L.check(L.lib().dph_index_last_add_ms(self._h, _np_ptr(out)))
        return out

    # ---- removing vectors (faiss index.remove_ids with IDSelectorBatch / IDSelectorRange) ----------
    def _selector(self, sel, what):
        """A label selector (remove_ids, make_filter) -> the C arguments (ids, n_ids, range_lo, range_hi, mem) and the array they point
        into (keep it alive for the call).  sel: a numpy or torch int64 array of labels or a step-1 range of labels."""
        if isinstance(sel, range):
            if sel.step != 1:
                raise ValueError(f"{what}: a range selector must have step 1")
            # ctypes would wrap bounds past the int64 range: clamp them (a stop past it then reaches every label up to 2^63 - 2)
            lo, hi = (min(max(v, -2**63), 2**63 - 1) for v in (sel.start, sel.stop))
            return (None, 0, lo, hi, L.MEM_HOST), None
        if isinstance(sel, np.ndarray):
            if sel.dtype != np.int64:
                raise TypeError(f"{what}: labels must be int64, got {sel.dtype}")
            ids = np.ascontiguousarray(sel).ravel()
            return (_np_ptr(ids), len(ids), 0, 0, L.MEM_HOST), ids
        import torch
        if not isinstance(sel, torch.Tensor) or sel.dtype != torch.int64:
            raise TypeError(f"{what}: expected an int64 numpy array, an int64 torch tensor or a step-1 range, got %r" % type(sel))
        ids = sel.contiguous().view(-1)
        if ids.is_cuda:
            self.set_stream(torch.cuda.current_stream(ids.device).cuda_stream)
            return (ids.data_ptr(), ids.numel(), 0, 0, L.MEM_DEVICE), ids
        ids = ids.numpy()
        return (_np_ptr(ids), len(ids), 0, 0, L.MEM_HOST), ids

    def remove_ids_per_list(self, sel):
        """Remove every row whose label is selected -> rows removed per list [nlist] i64 (this shard's lists only).  sel: a numpy or
        torch int64 array of labels (any order, duplicates allowed, absent or negative labels match nothing) or a step-1 range of
        labels.  Survivor order and the rejected cases: DESIGN.md 3.2 / dph_index_remove_ids."""
        per = np.zeros(self.nlist, dtype=np.int64)
        n = C.c_int64(0)
        args, keep = self._selector(sel, "remove_ids")
        L.check(L.lib().dph_index_remove_ids(self._h, *args, C.byref(n), _np_ptr(per)))
        del keep
        return per

    # ---- filtered search (faiss SearchParametersIVF(sel=IDSelector...); DESIGN.md 3.6) ----------------------------------------
    def make_filter(self, sel, exclude=False):
        """A row filter of this index for search(..., filter=) -> IndexFilter.  sel: the selectors of remove_ids (an int64 numpy or
        torch label array, or a step-1 range); exclude=True selects every row whose label is NOT selected.  The index is not changed.
        The filter holds one 4-byte mask word per 32-row code block of this shard, in device memory of its own; it is valid until the
        index's lists change (set_lists, add, remove, merge, sync_list_len), after which a search with it raises RuntimeError."""
        h = C.c_void_p()
        args, keep = self._selector(sel, "make_filter")
        L.check(L.lib().dph_filter_create(C.byref(h), self._h, *args[:4], int(bool(exclude)), args[4]))
        del keep
        return IndexFilter(self, h)

    def make_query_filters(self, sels, assign=None):
        """Per-query filters for one batch, for search(..., filter=) -> QueryFilters (DESIGN.md 3.7).  sels: a list of selectors of
        make_filter (int64 numpy or torch label arrays, or step-1 ranges); assign: int array [n], query i uses sels[assign[i]], -1 = no
        filter (default: arange(len(sels))).  Row i of a search of n queries with it is exactly search(x[i:i+1], k,
        filter=make_filter(sels[assign[i]])), or the unfiltered search for -1.  Each selector is held as the blocks of this shard that
        hold a selected row, with their mask words (8 bytes each) and a 4-byte offset per list of the shard; the scan reads only those
        blocks.  There is no per-query exclude: make_filter(sel, exclude=True) serves it for the whole batch.  The index is not changed;
        the filter is valid until its lists change, as an IndexFilter."""
        sels = list(sels)
        nsel = len(sels)
        assign = np.arange(nsel) if assign is None else np.asarray(assign)
        if assign.ndim != 1 or (assign.size and not np.issubdtype(assign.dtype, np.integer)):
            raise TypeError("make_query_filters: assign must be a 1-d int array")
        if assign.size and (assign.min() < -1 or assign.max() >= nsel):
            raise ValueError(f"make_query_filters: assign entries must be in [-1, {nsel})")
        assign = np.ascontiguousarray(assign, dtype=np.int32)
        ranges = np.zeros((nsel, 2), dtype=np.int64)
        counts = np.zeros(nsel, dtype=np.int64)
        parts, dev = [], None
        for i, sel in enumerate(sels):
            args, keep = self._selector(sel, "make_query_filters")
            if isinstance(sel, range):
                ranges[i] = args[2], args[3]
                continue
            counts[i] = args[1]
            if args[4] == L.MEM_DEVICE:
                dev = keep.device
            parts.append(keep)
        label_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        if dev is not None:                     # device labels: concatenated on that device
            import torch
            labels = torch.cat([torch.as_tensor(p).to(dev) for p in parts]).contiguous() if parts else None
            ptr, mem = (labels.data_ptr() if labels is not None and labels.numel() else None), L.MEM_DEVICE
        else:
            labels = np.ascontiguousarray(np.concatenate(parts + [np.zeros(0, np.int64)]).astype(np.int64, copy=False))
            ptr, mem = (_np_ptr(labels) if len(labels) else None), L.MEM_HOST
        h = C.c_void_p()
        L.check(L.lib().dph_query_filter_create(C.byref(h), self._h, ptr, _np_ptr(label_off), _np_ptr(ranges), nsel, _np_ptr(assign),
                                                len(assign), mem))
        qf = QueryFilters(self, h, nsel, len(assign))
        qf._spec = (sels, assign)
        return qf

    @contextlib.contextmanager
    def _filtered(self, filter):
        """The filter (an IndexFilter or QueryFilters) applies to the searches inside the block, and to no other."""
        if filter is None:
            yield
            return
        if isinstance(filter, IndexFilter):
            set_filter = L.lib().dph_index_set_filter
        elif isinstance(filter, QueryFilters):
            set_filter = L.lib().dph_index_set_query_filter
        else:
            raise TypeError(f"filter: expected an IndexFilter from make_filter or QueryFilters from make_query_filters, got {type(filter)!r}")
        L.check(set_filter(self._h, filter._h))
        try:
            yield
        finally:
            set_filter(self._h, None)

    def remove_ids(self, sel):
        """== faiss index.remove_ids(IDSelectorBatch(sel)) for a label array, index.remove_ids(IDSelectorRange(lo, hi)) for
        range(lo, hi) -> the number of rows removed (on a shard: from this shard).  A host-mode index needs a reserved host capacity
        (reserve_host_codes); the array is compacted in place."""
        return int(self.remove_ids_per_list(sel).sum())

    def list_len(self):
        """-> [nlist] i64: the length of every list (all shards)."""
        out = np.empty(self.nlist, dtype=np.int64)
        L.check(L.lib().dph_index_get_list_len(self._h, _np_ptr(out)))
        return out

    def sync_list_len(self, list_len):
        """Sharded remove: set the lengths of the other shards' lists (this shard's entries must equal its own).  A host-mode index
        needs a reserved host capacity (reserve_host_codes)."""
        list_len = np.ascontiguousarray(list_len, dtype=np.int64)
        assert list_len.shape == (self.nlist,)
        L.check(L.lib().dph_index_sync_list_len(self._h, _np_ptr(list_len)))

    def last_remove_ms(self):
        """With set_profile(True): stage times of the last remove in ms (mark + plan, row moves + block shift, direct map)."""
        out = np.zeros(3, dtype=np.float32)
        L.check(L.lib().dph_index_last_remove_ms(self._h, _np_ptr(out)))
        return out

    def last_remove_tmp_bytes(self):
        """The largest total of the last remove's temporary device allocations, in bytes."""
        return int(L.lib().dph_index_last_remove_tmp_bytes(self._h))

    # ---- merging indexes (invlists.merge_from of build_phrase_index.py:282-338; DESIGN.md 3.4) --------------
    def merge_from(self, sources, add_id=0):
        """== faiss index.merge_from(other, add_id) for one IvfPqIndex or a list of them, in order: every list gets each source's rows
        of that list behind its own, labels shifted by add_id.  The sources are not modified (faiss empties `other`).  Raises
        RuntimeError, leaving the index unchanged, on an incompatible source (d, nlist, device, shard range, or any bit of the OPQ
        matrix, centroids or PQ codebooks), the index itself as a source, a label + add_id outside [0, 2^63) or too little device
        memory.  Sources with no rows make it a no-op.  Into a host-mode index with a reserved host capacity (reserve_host_codes) from
        device-resident sources: rejected, unchanged, when the merged layout exceeds the capacity; a host-mode source is rejected."""
        sources = [sources] if isinstance(sources, IvfPqIndex) else list(sources)
        for s in sources:
            if not isinstance(s, IvfPqIndex):
                raise TypeError(f"merge_from: sources must be IvfPqIndex handles, got {type(s)!r}")
        arr = (C.c_void_p * max(len(sources), 1))(*[s._h for s in sources])
        L.check(L.lib().dph_index_merge_from(self._h, arr, len(sources), int(add_id)))

    def last_merge_ms(self):
        """With set_profile(True): stage times of the last merge in ms (plan + alloc, block moves, source rows, direct map)."""
        out = np.zeros(4, dtype=np.float32)
        L.check(L.lib().dph_index_last_merge_ms(self._h, _np_ptr(out)))
        return out

    # ---- training (faiss index.train, build_phrase_index.py:96-142; DESIGN.md 3.3) -------------------------
    def _train_input(self, x):
        """-> (pointer, n, mem, keepalive) for numpy or a CUDA float32 tensor [n, d]."""
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x, dtype=np.float32)
            return _np_ptr(x), self._rows(x), L.MEM_HOST, x
        import torch
        if not (x.is_cuda and x.dtype == torch.float32):
            raise TypeError("train: expected a numpy array or a float32 CUDA tensor")
        x = x.contiguous()
        self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
        return x.data_ptr(), self._rows(x), L.MEM_DEVICE, x

    def train_coarse(self, x, niter=10, seed=1234, max_points_per_centroid=256, hot_start=False):
        """Spherical k-means of the coarse quantizer on x A^T (the handle's OPQ matrix) -> (obj [niter] f64, nsplit [niter] i64):
        the summed inner products of the assignment before each update and the empty clusters re-seeded by splits.  hot_start keeps
        the current centroids instead of drawing new ones."""
        p, n, mem, keep = self._train_input(x)
        if n < 39 * self.nlist:
            import warnings
            warnings.warn(f"train_coarse: {n} training points for {self.nlist} centroids; faiss wants at least {39 * self.nlist}")
        obj = np.zeros(max(niter, 1), dtype=np.float64)
        nsplit = np.zeros(max(niter, 1), dtype=np.int64)
        L.check(L.lib().dph_index_train_coarse(self._h, p, n, int(niter), C.c_uint64(seed), int(max_points_per_centroid), int(bool(hot_start)),
                                                mem, _np_ptr(obj), _np_ptr(nsplit)))
        del keep
        return obj[:niter], nsplit[:niter]

    def train_pq(self, x, niter=25, seed=1234, max_points_per_centroid=256, hot_start=False, residual=True):
        """96 L2 k-means of the PQ codebooks on the residuals x A^T - C[top-1 list] (residual=False: on x A^T, OPQ's case)."""
        p, n, mem, keep = self._train_input(x)
        L.check(L.lib().dph_index_train_pq(self._h, p, n, int(niter), C.c_uint64(seed), int(max_points_per_centroid), int(bool(hot_start)),
                                            int(bool(residual)), mem))
        del keep

    def encode_pq(self, x):
        """PQ codes of x A^T without a coarse residual: numpy [n,d] -> [n,96] u8 numpy | torch cuda -> torch cuda."""
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x, dtype=np.float32)
            codes = np.empty((self._rows(x), 96), dtype=np.uint8)
            L.check(L.lib().dph_index_encode_pq(self._h, _np_ptr(x), len(x), _np_ptr(codes), L.MEM_HOST))
            return codes
        import torch
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        codes = torch.empty((self._rows(x), 96), dtype=torch.uint8, device=x.device)
        self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
        L.check(L.lib().dph_index_encode_pq(self._h, x.data_ptr(), x.shape[0], codes.data_ptr(), L.MEM_DEVICE))
        return codes

    def train_opq(self, x, niter=10, seed=1234, niter_pq=40, niter_pq_hot=4, max_train_points=65536):
        """faiss OPQMatrix::train: from a seeded random rotation, alternate PQ training on x R^T (niter_pq passes the first time, then
        niter_pq_hot with hot start) and the orthogonal Procrustes update R = (U V^T)^T of svd(x^T y), y = decode(encode(x R^T)).  The
        PQ passes run on the GPU; the 768 x 768 cross-covariance and its SVD are fp64 torch.  Sets and returns the OPQ matrix."""
        import torch
        dev = torch.device("cuda", self.device)
        n = int(x.shape[0])
        rows = np.arange(n) if n <= max_train_points else np.sort(np.random.default_rng(seed).choice(n, max_train_points, replace=False))
        xs = torch.as_tensor(x[rows] if isinstance(x, np.ndarray) else x[torch.as_tensor(rows, device=x.device)]).to(dev, torch.float32).contiguous()
        g = torch.Generator().manual_seed(seed)
        R = torch.linalg.qr(torch.randn((self.d, self.d), generator=g, dtype=torch.float64))[0].to(dev)
        xd = xs.double()
        for it in range(niter):
            self.set_opq(R.float().cpu().numpy())
            self.train_pq(xs, niter=niter_pq if it == 0 else niter_pq_hot, seed=seed, max_points_per_centroid=max_train_points,
                          hot_start=it > 0, residual=False)
            torch.cuda.current_stream(dev).synchronize()
            codes = self.encode_pq(xs).long()
            pq = torch.from_numpy(self.pq_codebooks()).to(dev)
            y = pq[torch.arange(96, device=dev)[None, :], codes].reshape(len(xs), self.d)
            u, _, vt = torch.linalg.svd(xd.T @ y.double())
            R = (u @ vt).T.contiguous()
        A = R.float().cpu().numpy()
        self.set_opq(A)
        return A

    def train(self, x, niter=10, niter_pq=25, opq_niter=10, seed=1234, max_points_per_centroid=256):
        """== faiss index.train(x) of IndexPreTransform(OPQMatrix, IndexIVFPQ(IndexFlatIP)): OPQ (skipped with opq_niter=0, which
        keeps the current matrix), then the coarse quantizer, then the PQ on residuals, as IndexPreTransform::train does.  x: numpy or a
        CUDA float32 tensor [n, 768].  Leaves a trained, empty index -> dict(obj, nsplit) of the coarse iterations."""
        if self.ntotal:
            raise RuntimeError("train: the index holds vectors")
        if opq_niter > 0:
            self.train_opq(x, niter=opq_niter, seed=seed)
        obj, nsplit = self.train_coarse(x, niter=niter, seed=seed, max_points_per_centroid=max_points_per_centroid)
        self.train_pq(x, niter=niter_pq, seed=seed, max_points_per_centroid=max_points_per_centroid, residual=True)
        self.set_lists(np.zeros(self.nlist, np.int64), np.zeros((0, 96), np.uint8))
        return dict(obj=obj, nsplit=nsplit)

    def centroids(self):
        """-> [nlist, d] f32: the coarse centroids (rotated space)."""
        out = np.empty((self.nlist, self.d), dtype=np.float32)
        L.check(L.lib().dph_index_get_centroids(self._h, _np_ptr(out), L.MEM_HOST))
        return out

    def pq_codebooks(self):
        """-> [96, 256, 8] f32: the PQ codebooks."""
        out = np.empty((96, 256, 8), dtype=np.float32)
        L.check(L.lib().dph_index_get_pq(self._h, _np_ptr(out), L.MEM_HOST))
        return out

    def last_train_ms(self):
        """With set_profile(True): stage times of the last train_coarse / train_pq in ms (assign, sort + update, split + renorm)."""
        out = np.zeros(3, dtype=np.float32)
        L.check(L.lib().dph_index_last_train_ms(self._h, _np_ptr(out)))
        return out

    # ---- attributes ---------------------------------------------------------------------------
    @property
    def ntotal(self):
        return L.lib().dph_index_ntotal(self._h)

    @property
    def ntotal_local(self):
        return L.lib().dph_index_ntotal_local(self._h)

    @property
    def d(self):
        return L.lib().dph_index_d(self._h)

    @property
    def nlist(self):
        return L.lib().dph_index_nlist(self._h)

    @property
    def nprobe(self):
        return L.lib().dph_index_nprobe(self._h)

    @nprobe.setter
    def nprobe(self, v):
        L.check(L.lib().dph_index_set_nprobe(self._h, int(v)))

    def set_scan_mode(self, mode):
        L.check(L.lib().dph_index_set_scan_mode(self._h, mode))

    def last_used_pair_mode(self):
        return bool(L.lib().dph_index_last_used_pair_mode(self._h))

    def last_group_size(self):
        """Queries per shared-memory gather in the last search: 1 (fp32 LUT), 2 (pair-packed) or 4 (quad-packed)."""
        return int(L.lib().dph_index_last_group_size(self._h))

    def set_coarse_tc(self, on):
        L.check(L.lib().dph_index_set_coarse_tc(self._h, int(bool(on))))

    def set_stream(self, cuda_stream_ptr):
        L.check(L.lib().dph_index_set_stream(self._h, C.c_void_p(cuda_stream_ptr)))

    def opq_matrix(self):
        A = np.empty((self.d, self.d), dtype=np.float32)
        L.check(L.lib().dph_index_get_opq(self._h, _np_ptr(A), L.MEM_HOST))
        return A

    def set_profile(self, on):
        L.check(L.lib().dph_index_set_profile(self._h, int(bool(on))))

    def last_scan_ms(self):
        ms = C.c_float(0)
        L.check(L.lib().dph_index_last_scan_ms(self._h, C.byref(ms)))
        return ms.value

    def profile_scan_ms(self):
        n = L.lib().dph_index_profile_count(self._h)
        out = np.zeros(max(n, 1), dtype=np.float32)
        L.check(L.lib().dph_index_profile_scan_ms(self._h, _np_ptr(out), n))
        return out[:n]

    @property
    def device_bytes(self):
        return L.lib().dph_index_device_bytes(self._h)

    # ---- search -------------------------------------------------------------------------------
    def search(self, x, k, filter=None):
        """numpy [n,d] -> (D [n,k] f32, I [n,k] i64) numpy   |   torch cuda [n,d] -> torch cuda (D, I).  filter (make_filter): the
        same probes, and only selected rows can be results -- the unfiltered ranking of the probed rows restricted to the selected ones,
        cut at k; short results are padded with (-FLT_MAX, -1)."""
        with self._filtered(filter):
            return self._search(x, k)

    def _search(self, x, k):
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x, dtype=np.float32)
            n = x.shape[0]
            D = np.empty((n, k), dtype=np.float32)
            I = np.empty((n, k), dtype=np.int64)
            L.check(L.lib().dph_index_search(self._h, _np_ptr(x), n, k, _np_ptr(D), _np_ptr(I), L.MEM_HOST))
            return D, I
        import torch
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        n = x.shape[0]
        D = torch.empty((n, k), dtype=torch.float32, device=x.device)
        I = torch.empty((n, k), dtype=torch.int64, device=x.device)
        self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
        L.check(L.lib().dph_index_search(self._h, x.data_ptr(), n, k, D.data_ptr(), I.data_ptr(), L.MEM_DEVICE))
        return D, I

    def search_partial(self, x, k, filter=None):
        """torch cuda [n,d] -> per-shard (D, I, G) torch cuda; G = canonical scan position (tie-break).  filter: as in search."""
        with self._filtered(filter):
            return self._search_partial(x, k)

    def _search_partial(self, x, k):
        import torch
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        n = x.shape[0]
        D = torch.empty((n, k), dtype=torch.float32, device=x.device)
        I = torch.empty((n, k), dtype=torch.int64, device=x.device)
        G = torch.empty((n, k), dtype=torch.int32, device=x.device)
        self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
        L.check(L.lib().dph_index_search_partial(self._h, x.data_ptr(), n, k, D.data_ptr(), I.data_ptr(), G.data_ptr()))
        return D, I, G

    def coarse_local(self, x):
        """torch cuda [n,d] -> int64 [n,nprobe] keys of this shard's best lists (score key << 32 | ~global list id)."""
        import torch
        n = x.shape[0]
        keys = torch.empty((n, self.nprobe), dtype=torch.int64, device=x.device)
        self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
        L.check(L.lib().dph_index_coarse_local(self._h, x.data_ptr(), n, keys.data_ptr()))
        return keys

    def search_preassigned(self, keys_gathered, k, filter=None):
        """all-gathered keys [nshards,n,nprobe] -> this shard's partial (D, I, G) for the batch passed to coarse_local.  filter: as in
        search, this shard's own."""
        with self._filtered(filter):
            return self._search_preassigned(keys_gathered, k)

    def _search_preassigned(self, keys_gathered, k):
        import torch
        W, n, _ = keys_gathered.shape
        D = torch.empty((n, k), dtype=torch.float32, device=keys_gathered.device)
        I = torch.empty((n, k), dtype=torch.int64, device=keys_gathered.device)
        G = torch.empty((n, k), dtype=torch.int32, device=keys_gathered.device)
        self.set_stream(torch.cuda.current_stream(keys_gathered.device).cuda_stream)
        L.check(L.lib().dph_index_search_preassigned(self._h, keys_gathered.data_ptr(), W, n, k, D.data_ptr(), I.data_ptr(), G.data_ptr()))
        return D, I, G

    def coarse_split(self, x_local):
        """torch cuda [n_local,d] (this rank's slice of the batch) -> records [n_local, 768 + 2 nprobe] f32: rotated query, probed
        lists (int32 bits) and coarse scores over ALL lists (dph_index_coarse_split)."""
        import torch
        n = x_local.shape[0]
        rec = torch.empty((n, L.lib().dph_index_record_floats(self._h)), dtype=torch.float32, device=x_local.device)
        self.set_stream(torch.cuda.current_stream(x_local.device).cuda_stream)
        L.check(L.lib().dph_index_coarse_split(self._h, x_local.data_ptr(), n, rec.data_ptr()))
        return rec

    def search_assigned(self, rec, k, filter=None):
        """all-gathered records [n, 768 + 2 nprobe] (batch order) -> this shard's partial (D, I, G).  filter: as in search, this
        shard's own."""
        with self._filtered(filter):
            return self._search_assigned(rec, k)

    def _search_assigned(self, rec, k):
        import torch
        assert rec.is_cuda and rec.dtype == torch.float32 and rec.is_contiguous()
        n = rec.shape[0]
        D = torch.empty((n, k), dtype=torch.float32, device=rec.device)
        I = torch.empty((n, k), dtype=torch.int64, device=rec.device)
        G = torch.empty((n, k), dtype=torch.int32, device=rec.device)
        self.set_stream(torch.cuda.current_stream(rec.device).cuda_stream)
        L.check(L.lib().dph_index_search_assigned(self._h, rec.data_ptr(), n, k, D.data_ptr(), I.data_ptr(), G.data_ptr()))
        return D, I, G

    def _last(self, which, shape, dtype):
        out = np.empty(shape, dtype=dtype)
        L.check(L.lib().dph_index_copy_last(self._h, which, _np_ptr(out), out.nbytes))
        return out

    def last_flags(self, n):
        return self._last(0, (n,), np.int32)

    def last_probes(self, n):
        return self._last(1, (n, self.nprobe), np.int32)

    def last_coarse(self, n):
        return self._last(2, (n, self.nprobe), np.float32)

    def last_xr(self, n):
        return self._last(3, (n, self.d), np.float32)

    # ---- reconstruct ----------------------------------------------------------------------------
    def reconstruct_batch(self, ids):
        """labels [m] -> (vec [m,d] f32 in ROTATED space, found [m] u8); missing label -> zeros (index.py:287-288)."""
        if isinstance(ids, np.ndarray) or isinstance(ids, (list, tuple)):
            ids = np.ascontiguousarray(ids, dtype=np.int64)
            out = np.empty((len(ids), self.d), dtype=np.float32)
            found = np.empty(len(ids), dtype=np.uint8)
            L.check(L.lib().dph_index_reconstruct_batch(self._h, _np_ptr(ids), len(ids), _np_ptr(out), _np_ptr(found), L.MEM_HOST))
            return out, found
        import torch
        assert ids.is_cuda and ids.dtype == torch.int64
        out = torch.empty((ids.numel(), self.d), dtype=torch.float32, device=ids.device)
        found = torch.empty(ids.numel(), dtype=torch.uint8, device=ids.device)
        self.set_stream(torch.cuda.current_stream(ids.device).cuda_stream)
        L.check(L.lib().dph_index_reconstruct_batch(self._h, ids.data_ptr(), ids.numel(), out.data_ptr(), found.data_ptr(), L.MEM_DEVICE))
        return out, found


class IndexFilter:
    """A row filter of one IvfPqIndex (make_filter): a device mask of one bit per row of the index's shard."""

    def __init__(self, index, h):
        self.index = index          # the mask belongs to this handle; keeping it alive keeps the handle alive
        self._h = h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        index = getattr(self, "index", None)
        if h and getattr(index, "_h", None) and L is not None and getattr(L, "_lib", None) is not None:   # the handle outlives the filter
            L._lib.dph_filter_free(h)

    @property
    def rows(self):
        """Selected rows of the shard."""
        return int(L.lib().dph_filter_rows(self._h))

    @property
    def nbytes(self):
        """Device bytes of the mask (4 per 32-row code block of the shard)."""
        return int(L.lib().dph_filter_bytes(self._h))

    def mask(self):
        """-> uint32 [code blocks of the shard]: bit l of word b = row l of block b is selected (blocks in the shard's list order)."""
        out = np.empty(self.nbytes // 4, dtype=np.uint32)
        L.check(L.lib().dph_filter_copy_mask(self._h, _np_ptr(out)))
        return out


class QueryFilters:
    """Per-query filters of one IvfPqIndex for one batch of n queries (make_query_filters): nsel selectors, each the shard's blocks that
    hold a selected row with their mask words, and the selector of every query."""

    def __init__(self, index, h, nsel, n):
        self.index = index          # the filter belongs to this handle; keeping it alive keeps the handle alive
        self._h = h
        self.nsel, self.n = nsel, n

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        index = getattr(self, "index", None)
        if h and getattr(index, "_h", None) and L is not None and getattr(L, "_lib", None) is not None:   # the handle outlives the filter
            L._lib.dph_query_filter_free(h)

    def rows(self, i):
        """Selected rows of the shard by selector i."""
        if not 0 <= i < self.nsel:
            raise IndexError(i)
        return int(L.lib().dph_query_filter_rows(self._h, i))

    @property
    def nbytes(self):
        """Device bytes of the filter: 8 per selected block, 4 per list of the shard per selector, the assignment and the bases."""
        return int(L.lib().dph_query_filter_bytes(self._h))

    def csr(self, i):
        """Selector i -> (off [lists of the shard + 1] u32, blk [m] u32, word [m] u32): list lo + j's blocks are blk[off[j]:off[j+1]]
        (ascending block numbers of the list) with their mask words (bit l = lane l's row is selected)."""
        if not 0 <= i < self.nsel:
            raise IndexError(i)
        m = int(L.lib().dph_query_filter_blocks(self._h, i))
        lo, hi = self.index.shard
        off = np.empty(hi - lo + 1, dtype=np.uint32)
        blk, word = np.empty(m, dtype=np.uint32), np.empty(m, dtype=np.uint32)
        L.check(L.lib().dph_query_filter_copy_selector(self._h, i, _np_ptr(off), _np_ptr(blk), _np_ptr(word)))
        return off, blk, word

    def for_rows(self, a, b):
        """The filter of queries a..b-1 of this batch (a new QueryFilters of the same index, holding only the selectors they use)."""
        sels, assign = self._spec
        used, sub = np.unique(assign[a:b], return_inverse=True)
        keep = used >= 0
        remap = np.full(len(used), -1, dtype=np.int64)
        remap[keep] = np.arange(int(keep.sum()))
        return self.index.make_query_filters([sels[i] for i in used[keep]], remap[sub.ravel()])

    def mask(self, i):
        """Selector i expanded to the row mask of make_filter (uint32 per code block of the shard)."""
        off, blk, word = self.csr(i)
        lo, hi = self.index.shard
        nb = (self.index.list_len()[lo:hi] + 31) // 32
        first = np.concatenate([[0], np.cumsum(nb)])[:-1]
        out = np.zeros(int(nb.sum()), dtype=np.uint32)
        lists = np.repeat(np.arange(hi - lo), np.diff(off.astype(np.int64)))
        out[first[lists] + blk] = word
        return out


def _window_scores(self, q, first_ids, L):
    """q [m,768] f32, first_ids [m] int64 (numpy) -> scores [m,L] f32: <q[i], un-rotated reconstruct(first_ids[i] + l)>;
    labels that are not in the index score 0 (the reference's zero vector, index.py:287-288)."""
    q = np.ascontiguousarray(q, dtype=np.float32)
    first_ids = np.ascontiguousarray(first_ids, dtype=np.int64)
    out = np.empty((len(first_ids), L), dtype=np.float32)
    L_.check(L_.lib().dph_index_window_scores(self._h, _np_ptr(q), _np_ptr(first_ids), len(first_ids), L, _np_ptr(out), L_.MEM_HOST))
    return out


L_ = L
IvfPqIndex.window_scores = _window_scores


def merge_shards(Dg, Ig, Gg, k):
    """all-gathered [nshards,n,k] torch cuda tensors -> (D, I) [n,k]; order score desc, scan position asc."""
    import torch
    nsh, n, kk = Dg.shape
    assert kk == k and Dg.is_contiguous() and Ig.is_contiguous() and Gg.is_contiguous()
    D = torch.empty((n, k), dtype=torch.float32, device=Dg.device)
    I = torch.empty((n, k), dtype=torch.int64, device=Dg.device)
    st = torch.cuda.current_stream(Dg.device).cuda_stream
    L.check(L.lib().dph_merge_shards(Dg.data_ptr(), Ig.data_ptr(), Gg.data_ptr(), nsh, n, k, D.data_ptr(), I.data_ptr(), C.c_void_p(st)))
    return D, I


def pack_topk(D, I, G):
    """(D f32, I i64, G i32) [n,k] cuda -> P int64 [n,k,2] for a single all-gather."""
    import torch
    n, k = D.shape
    P = torch.empty((n, k, 2), dtype=torch.int64, device=D.device)
    st = torch.cuda.current_stream(D.device).cuda_stream
    L.check(L.lib().dph_pack_topk(D.data_ptr(), I.data_ptr(), G.data_ptr(), n, k, P.data_ptr(), C.c_void_p(st)))
    return P


def merge_shards_packed(Pg, k):
    """all-gathered P [nshards,n,k,2] -> (D, I) [n,k]."""
    import torch
    nsh, n = Pg.shape[0], Pg.shape[1]
    D = torch.empty((n, k), dtype=torch.float32, device=Pg.device)
    I = torch.empty((n, k), dtype=torch.int64, device=Pg.device)
    st = torch.cuda.current_stream(Pg.device).cuda_stream
    L.check(L.lib().dph_merge_shards_packed(Pg.data_ptr(), nsh, n, k, D.data_ptr(), I.data_ptr(), C.c_void_p(st)))
    return D, I
