"""ShardedIvfPq: the phrase index sharded by inverted-list range over the ranks of one torch.distributed job
(SURVEY.md 8e): every rank holds lists [lo, hi), replicated coarse quantizer / OPQ / PQ codebooks; a search is
  coarse step (exchange 1: query-split records or list-split candidate keys, see sharded_search_qsplit / sharded_search)
  ->  per-rank partial top-k over the global probe set  ->  exchange 2: ONE all-gather of the packed (candidate key, label) pairs
  ->  identical k-way merge on every rank.
With world_size 1 it degenerates to IvfPqIndex.  This is the call a user (MIPS.search_dense) makes."""
import numpy as np
import torch

from .ivfpq import IvfPqIndex, QueryFilters, default_stream_bytes, merge_shards, merge_shards_packed, pack_topk


def shard_ranges(list_len, world):
    """Contiguous list ranges cut by cumulative code bytes (not by list count), SURVEY.md 8e."""
    list_len = np.asarray(list_len, dtype=np.int64)
    cum = np.concatenate([[0], np.cumsum(list_len)])
    total = cum[-1]
    cuts = [0]
    for r in range(1, world):
        t = total * r / world
        i = int(np.searchsorted(cum, t, side="left"))
        if i > 0 and abs(cum[i - 1] - t) <= abs(cum[min(i, len(cum) - 1)] - t):
            i -= 1
        cuts.append(i)
    cuts.append(len(list_len))
    cuts = np.maximum.accumulate(np.array(cuts))
    return [(int(cuts[r]), int(cuts[r + 1])) for r in range(world)]


def gather_and_merge(D, I, G, k, world, group=None, merge_fn=merge_shards):
    """The single exchange step of the sharded search: all-gather every shard's [n,k] partial top-k
    (score f32, label i64, canonical scan position i32) and merge identically on every rank.
    Backend-agnostic (nccl on GPUs; the gloo CPU test passes a numpy merge_fn)."""
    import torch.distributed as dist
    n = D.shape[0]
    Dg = torch.empty((world * n, k), dtype=D.dtype, device=D.device)      # concatenated along dim 0 (gloo and nccl both accept it)
    Ig = torch.empty((world * n, k), dtype=I.dtype, device=I.device)
    Gg = torch.empty((world * n, k), dtype=G.dtype, device=G.device)
    dist.all_gather_into_tensor(Dg, D.contiguous(), group=group)
    dist.all_gather_into_tensor(Ig, I.contiguous(), group=group)
    dist.all_gather_into_tensor(Gg, G.contiguous(), group=group)
    return merge_fn(Dg.view(world, n, k), Ig.view(world, n, k), Gg.view(world, n, k), k)


def sharded_search(x, k, world, group, coarse_local, search_preassigned, pack, merge_packed):
    """The two-exchange protocol of one sharded search, independent of where the local work runs (CUDA in the product, the CPU
    oracle in tests/test_sharded_cpu.py over gloo):
        keys   = coarse_local(x)                      [n, nprobe] int64   this shard's best lists (score key << 32 | ~list id)
        keys_g = all_gather(keys)                     [W, n, nprobe]      exchange 1
        D,I,G  = search_preassigned(keys_g, k)        per-shard partial top-k over the GLOBAL probe set
        P_g    = all_gather(pack(D, I, G))            [W, n, k, 2]        exchange 2
        return merge_packed(P_g, k)                   identical on every rank"""
    import torch.distributed as dist
    n = x.shape[0]
    keys = coarse_local(x)
    keys_g = torch.empty((world * n, keys.shape[1]), dtype=torch.int64, device=keys.device)
    dist.all_gather_into_tensor(keys_g, keys.contiguous(), group=group)
    D, I, G = search_preassigned(keys_g.view(world, n, -1), k)
    P = pack(D, I, G)
    Pg = torch.empty((world * n, k, 2), dtype=torch.int64, device=P.device)
    dist.all_gather_into_tensor(Pg, P.contiguous(), group=group)
    return merge_packed(Pg.view(world, n, k, 2), k)


def query_slice(x, rank, world):
    """Rows [r P, (r+1) P) of the batch, P = ceil(n / W), zero rows padding the last slice (x: torch tensor on any device)."""
    n = x.shape[0]
    per = (n + world - 1) // world
    lo, hi = min(rank * per, n), min((rank + 1) * per, n)
    xl = x[lo:hi]
    if hi - lo < per:
        xl = torch.cat([xl, torch.zeros((per - (hi - lo), x.shape[1]), dtype=x.dtype, device=x.device)])
    return xl.contiguous()


def sharded_search_qsplit(x, k, world, rank, group, coarse_split, search_assigned, pack, merge_packed, x_local=None, n=None):
    """The query-split protocol (large batches): the coarse quantizer is replicated, so rank r rotates and assigns queries
    [r P, (r+1) P) of the batch (P = ceil(n / W), zero rows pad the last slice) over ALL lists and the ranks exchange the results:
        rec    = coarse_split(x[r P : (r+1) P])      [P, 768 + 2 nprobe]  rotated query | probed lists | coarse scores
        rec_g  = all_gather(rec)[:n]                 [n, ...]             exchange 1 (batch order: slices are contiguous)
        D,I,G  = search_assigned(rec_g, k)           per-shard partial top-k over the global probe set
        P_g    = all_gather(pack(D, I, G))           [W, n, k, 2]         exchange 2
        return merge_packed(P_g, k)
    Same probes, same scores as sharded_search; the per-query work before the scan is done once instead of once per rank.
    A caller that holds the batch on the host passes only its slice (x_local = query_slice(x_host, rank, world) on the device, n =
    the batch size): then a rank's host-to-device copy is n / W rows instead of n."""
    import torch.distributed as dist
    if x_local is None:
        n = x.shape[0]
        x_local = query_slice(x, rank, world)
    rec = coarse_split(x_local)
    rec_g = torch.empty((world * x_local.shape[0], rec.shape[1]), dtype=rec.dtype, device=rec.device)
    dist.all_gather_into_tensor(rec_g, rec.contiguous(), group=group)
    D, I, G = search_assigned(rec_g[:n], k)
    P = pack(D, I, G)
    Pg = torch.empty((world * n, k, 2), dtype=torch.int64, device=P.device)
    dist.all_gather_into_tensor(Pg, P.contiguous(), group=group)
    return merge_packed(Pg.view(world, n, k, 2), k)


def use_query_split(n, world, nlist, d=768):
    """Query-split pays when every rank's slice still fills tensor-core tiles and streaming the WHOLE centroid table (fp32 hi/lo planes)
    per batch is cheap next to the scan: C4 (1024 queries, IVF65536: 400 MB of planes) yes; C5 (128 vectors, IVF1048576: 6.4 GB) no."""
    return world > 1 and n >= 32 * world and nlist * d * 8 <= (1 << 30)


class ShardedIvfPq:
    def __init__(self, nlist, rank=0, world=1, device=0, group=None, local=None):
        self.rank, self.world, self.device, self.group = rank, world, device, group
        self.local = local if local is not None else IvfPqIndex(nlist, device=device)      # `local`: any object with the IvfPqIndex API (tests)
        self._pinned_in = None
        self._pinned_out = None
        self.query_split = None          # None: use_query_split() decides per batch; True / False force one protocol (tests, measurements)

    def _residency(self, list_len, codes_on_host, stream_bytes, host_capacity_bytes):
        if host_capacity_bytes is not None and not codes_on_host:
            raise ValueError("host_capacity_bytes needs codes_on_host=True")
        if codes_on_host:
            self.local.set_code_residency(True, default_stream_bytes(list_len, *self.range) if stream_bytes is None else stream_bytes)
            if host_capacity_bytes is not None:
                self.local.reserve_host_codes(host_capacity_bytes)

    def build_synthetic(self, A, list_len, seed, centroid_sigma=0.5, pq_sigma=0.25, codes_on_host=False, stream_bytes=None,
                        host_capacity_bytes=None):
        lo, hi = shard_ranges(list_len, self.world)[self.rank]
        self.range = (lo, hi)
        ix = self.local
        ix.set_opq(A)
        ix.gen_centroids(seed, centroid_sigma)
        ix.gen_pq(seed, pq_sigma)
        if self.world > 1:
            ix.set_shard(lo, hi)
        self._residency(list_len, codes_on_host, stream_bytes, host_capacity_bytes)
        ix.set_lists_synthetic(list_len, seed)
        return self

    @classmethod
    def from_arrays(cls, A, centroids, pq, list_len, codes, ids=None, rank=0, world=1, device=0, group=None, codes_on_host=False,
                    stream_bytes=None, host_capacity_bytes=None):
        """The arrays of a faiss IndexPreTransform(OPQ) -> IndexIVFPQ file (index.py:30), list-major rows of ALL lists; this rank
        uploads only the rows of its own list range.  codes_on_host / stream_bytes / host_capacity_bytes: IvfPqIndex.from_arrays, per
        rank (host_capacity_bytes is this rank's capacity)."""
        list_len = np.asarray(list_len, dtype=np.int64)
        self = cls(len(list_len), rank=rank, world=world, device=device, group=group)
        lo, hi = shard_ranges(list_len, world)[rank]
        self.range = (lo, hi)
        off = np.concatenate([[0], np.cumsum(list_len)])
        ix = self.local
        ix.set_opq(A)
        ix.set_centroids(centroids)
        ix.set_pq(pq)
        if world > 1:
            ix.set_shard(lo, hi)
        self._residency(list_len, codes_on_host, stream_bytes, host_capacity_bytes)
        ix.set_lists(list_len, codes[off[lo]:off[hi]], None if ids is None else ids[off[lo]:off[hi]])
        return self

    def add_with_ids(self, x, ids=None):
        """== faiss index.add_with_ids (build_phrase_index.py:145-150); a collective by convention like search: every rank passes the
        same batch.  No exchange is needed: assignment is deterministic and the coarse quantizer is replicated, so every rank derives
        the same global list lengths and labels (ids None -> ntotal + arange(n)) and stores the rows of its own lists."""
        self.local.add_with_ids(x, ids)

    def add_int8(self, q, ids, offset, scale):
        """add_with_ids of int8 rows dequantised in fp32 on the device (IvfPqIndex.add_int8); a collective like add_with_ids."""
        self.local.add_int8(q, ids, offset, scale)

    def remove_ids(self, sel):
        """== faiss index.remove_ids (IvfPqIndex.remove_ids selectors); a collective: every rank passes the same selector.  Each rank
        removes the rows of its own lists; the per-list counts are all-reduced so that every rank sets the same global list lengths
        (and list starts, which order ties in the merge).  Returns the number of rows removed from the whole index."""
        if self.world == 1:
            return self.local.remove_ids(sel)
        before = self.local.list_len()
        removed = self._sum_over_shards(self.local.remove_ids_per_list(sel))
        self.local.sync_list_len(before - removed)
        return int(removed.sum())

    def merge_from(self, sources, add_id=0):
        """== faiss index.merge_from (IvfPqIndex.merge_from) for one ShardedIvfPq or a list of them; a collective by convention: every
        rank passes the same sources.  Each rank merges its own shard of each source, which must hold the same list range.  No
        exchange is needed: every handle holds the global list lengths, so every rank reaches the same global lengths and list
        starts.  A rejection that depends only on the handles' shapes and tables is the same on every rank; one that depends on this
        rank's rows (a label + add_id out of range) or on its device memory leaves only that rank unchanged."""
        sources = [sources] if isinstance(sources, ShardedIvfPq) else list(sources)
        for s in sources:
            if not isinstance(s, ShardedIvfPq):
                raise TypeError(f"merge_from: sources must be ShardedIvfPq, got {type(s)!r}")
            if (s.rank, s.world) != (self.rank, self.world) or getattr(s, "range", None) != getattr(self, "range", None):
                raise RuntimeError("merge_from: a source is sharded differently (rank, world size or list range); the index is unchanged")
        self.local.merge_from([s.local for s in sources], add_id)

    def reserve_host_codes(self, nbytes):
        """Host mode: every rank reserves a host capacity of nbytes for its own shard (IvfPqIndex.reserve_host_codes), which makes
        add_with_ids, remove_ids and merge_from run in place on its page-locked array."""
        self.local.reserve_host_codes(nbytes)

    def make_filter(self, sel, exclude=False):
        """A row filter for search / search_device (IvfPqIndex.make_filter): every rank builds the mask of its own shard from the same
        selector, with no exchange (labels are looked up where the rows live).  A collective by convention: every rank passes the same
        selector."""
        return self.local.make_filter(sel, exclude)

    def make_query_filters(self, sels, assign=None):
        """Per-query filters for search / search_device (IvfPqIndex.make_query_filters): every rank builds the filter of its own shard
        from the same selectors, with no exchange.  A collective by convention: every rank passes the same selectors and assignment."""
        return self.local.make_query_filters(sels, assign)

    def set_resident_lists(self, lists):
        """Host mode: every rank keeps in device memory the given lists that fall in its own range (IvfPqIndex.set_resident_lists)."""
        lists = np.asarray(lists, dtype=np.int64).ravel()
        lo, hi = self.range
        self.local.set_resident_lists(lists[(lists >= lo) & (lists < hi)])

    # ---- the slice of the faiss index API that MIPS uses (index.py:30-33,200,286,296) ----
    @property
    def ntotal(self):
        return self.local.ntotal

    @property
    def d(self):
        return self.local.d

    @property
    def nlist(self):
        return self.local.nlist

    def opq_matrix(self):
        return self.local.opq_matrix()

    def _sum_over_shards(self, arr, op=None):
        """Every label lives on exactly one shard and the others return zeros: the all-reduce sum IS the gather."""
        if self.world == 1:
            return arr
        import torch.distributed as dist
        dev = torch.device("cuda", self.device) if dist.get_backend(self.group) == "nccl" else torch.device("cpu")    # gloo: CPU tests
        t = torch.from_numpy(np.ascontiguousarray(arr)).to(dev)
        dist.all_reduce(t, op=op or dist.ReduceOp.SUM, group=self.group)
        return t.cpu().numpy()

    def reconstruct_batch(self, ids):
        """labels [m] (numpy) -> (vec [m,d] f32 rotated space, found [m] u8), collective over the shards."""
        import torch.distributed as dist
        vec, found = self.local.reconstruct_batch(np.ascontiguousarray(ids, dtype=np.int64))
        if self.world == 1:
            return vec, found
        return self._sum_over_shards(vec), self._sum_over_shards(found.astype(np.int32), dist.ReduceOp.MAX).astype(np.uint8)

    def window_scores(self, q, first_ids, L):
        """q [m,768], first_ids [m] -> [m,L] phrase-window scores (dph_index_window_scores), collective over the shards."""
        return self._sum_over_shards(self.local.window_scores(q, first_ids, L))

    @property
    def nprobe(self):
        return self.local.nprobe

    @nprobe.setter
    def nprobe(self, v):
        self.local.nprobe = v

    def _qsplit(self, n):
        return self.world > 1 and (self.query_split is True or (self.query_split is None and use_query_split(n, self.world, self.local.nlist)))

    def _local_steps(self, filter):
        """This rank's search steps of both protocols, with `filter` (make_filter or make_query_filters) applied to each."""
        if filter is None:
            return self.local.search_assigned, self.local.search_preassigned
        return (lambda rec, k: self.local.search_assigned(rec, k, filter=filter),
                lambda keys, k: self.local.search_preassigned(keys, k, filter=filter))

    def search_device(self, x, k, filter=None):
        """x torch cuda [n,d] (same on every rank) -> (D, I) torch cuda [n,k] (same on every rank).  filter (make_filter, or
        make_query_filters for these n queries): only selected rows can be results (IvfPqIndex.search)."""
        if self.world == 1:
            return self.local.search(x, k, filter=filter)
        n = x.shape[0]
        if n > 4096:        # one chunk per collective round; a per-query filter is cut to each chunk's rows
            per = (lambda i: filter.for_rows(i, i + 4096)) if isinstance(filter, QueryFilters) else (lambda i: filter)
            parts = [self.search_device(x[i:i + 4096], k, per(i)) for i in range(0, n, 4096)]
            return torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
        assigned, preassigned = self._local_steps(filter)
        if self._qsplit(n):
            return sharded_search_qsplit(x, k, self.world, self.rank, self.group, self.local.coarse_split, assigned, pack_topk, merge_shards_packed)
        return sharded_search(x, k, self.world, self.group, self.local.coarse_local, preassigned, pack_topk, merge_shards_packed)

    def search(self, x, k, filter=None):
        """Host API == faiss index.search (index.py:200): numpy / pinned CPU tensor [n,d] -> numpy (D, I).  filter: as in
        search_device."""
        if self.world == 1 and isinstance(x, np.ndarray):
            return self.local.search(x, k, filter=filter)
        xt = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)) if isinstance(x, np.ndarray) else x
        n = xt.shape[0]
        dev = torch.device("cuda", self.device)
        if n <= 4096 and self._qsplit(n):        # query-split: only this rank's slice of the batch crosses PCIe
            xl = query_slice(xt, self.rank, self.world).to(dev, non_blocking=True)
            D, I = sharded_search_qsplit(None, k, self.world, self.rank, self.group, self.local.coarse_split, self._local_steps(filter)[0],
                                         pack_topk, merge_shards_packed, x_local=xl, n=n)
        else:
            D, I = self.search_device(xt.to(dev, non_blocking=True), k, filter)
        if self._pinned_out is None or self._pinned_out[0].shape != (n, k):
            self._pinned_out = (torch.empty((n, k), dtype=torch.float32).pin_memory(), torch.empty((n, k), dtype=torch.int64).pin_memory())
        Dh, Ih = self._pinned_out
        Dh.copy_(D, non_blocking=True)
        Ih.copy_(I, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        return Dh.numpy().copy(), Ih.numpy().copy()       # fresh arrays like faiss index.search; the pinned pair is staging only
