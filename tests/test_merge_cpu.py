"""CPU: the definition of merging indexes (tests/merge_ref.py, DESIGN.md 3.4) on hand examples, and a sharded merge over gloo with
oracle-backed shards that equals the unsharded oracle of the merged arrays."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.helpers import assert_topk_equal
from tests.merge_ref import np_merge


def rows(*tags):
    return np.array(tags, np.uint8)[:, None].repeat(96, 1)


def test_hand_example_ragged_lists():
    dest = (np.array([2, 0, 1, 0]), rows(1, 2, 3), np.array([10, 11, 12]))
    seq = (np.array([1, 2, 0, 0]), rows(4, 5, 6), None)                          # sequential labels 0, 1, 2
    expl = (np.array([0, 0, 3, 0]), rows(7, 8, 9), np.array([7, 8, 9]))
    lens, codes, ids = np_merge(dest, [seq, expl], add_id=100)
    assert list(lens) == [3, 2, 4, 0]
    assert list(ids) == [10, 11, 100, 101, 102, 12, 107, 108, 109]
    assert list(codes[:, 0]) == [1, 2, 4, 5, 6, 3, 7, 8, 9] and (codes == codes[:, :1]).all()
    # argument order decides the order inside a list; add_id shifts only the sources
    lens2, codes2, ids2 = np_merge(dest, [expl, seq])
    assert list(ids2) == [10, 11, 0, 1, 2, 12, 7, 8, 9] and list(codes2[:, 0]) == [1, 2, 4, 5, 6, 3, 7, 8, 9]


def test_sequential_destination_and_empty_sources():
    dest = (np.array([0, 3, 1]), rows(1, 2, 3, 4), None)                        # labels 0 .. 3
    empty = (np.zeros(3, np.int64), np.zeros((0, 96), np.uint8), None)
    lens, codes, ids = np_merge(dest, [empty, empty], add_id=5)
    assert list(lens) == [0, 3, 1] and list(ids) == [0, 1, 2, 3] and np.array_equal(codes, dest[1])
    src = (np.array([2, 0, 0]), rows(5, 6), np.array([3, 3]))                   # a label already present, twice
    lens, codes, ids = np_merge(dest, [src, empty])
    assert list(lens) == [2, 3, 1] and list(ids) == [3, 3, 0, 1, 2, 3] and list(codes[:, 0]) == [5, 6, 1, 2, 3, 4]


def test_equals_per_list_concatenation_on_random_arrays():
    rng = np.random.default_rng(0)
    nlist = 37
    parts = []
    for k in range(4):
        ln = rng.integers(0, 70, nlist) * (rng.random(nlist) < 0.7)
        n = int(ln.sum())
        parts.append((ln, rng.integers(0, 256, (n, 96), dtype=np.uint8), None if k == 2 else rng.permutation(n).astype(np.int64) * 3))
    lens, codes, ids = np_merge(parts[0], parts[1:], add_id=1000)
    off = [np.concatenate([[0], np.cumsum(p[0])]) for p in parts]
    o = 0
    for l in range(nlist):
        for k, (ln, c, i) in enumerate(parts):
            lab = np.arange(int(ln.sum())) if i is None else i
            seg = slice(off[k][l], off[k][l + 1])
            m = int(ln[l])
            assert np.array_equal(codes[o:o + m], c[seg]) and np.array_equal(ids[o:o + m], lab[seg] + (1000 if k else 0))
            o += m
    assert o == len(ids) == int(lens.sum())


# ---- sharded merge over gloo: every rank merges its shard of the same sources into an oracle-backed list-range shard ----
def _shard_class():
    from tests.merge_ref import arrays
    from tests.test_add_cpu import _OracleAddShard

    class OracleMergeShard(_OracleAddShard):
        """_OracleAddShard that can also merge the same shard of other indexes, like dph_index_merge_from on a shard: its own lists
        get the sources' rows, the other lists only their lengths."""

        def merge_from(self, sources, add_id):
            assert all((s.lo, s.hi) == (self.lo, self.hi) for s in sources)
            lens, codes, ids = np_merge(arrays(self.local), [arrays(s.local) for s in sources], add_id)
            assert not lens[:self.lo].any() and not lens[self.hi:].any()
            self.local.__init__(self.local.A, self.local.pq, lens, centroids=self.local.C, codes=codes, ids=ids)
            self.lens = self.lens + sum(s.lens for s in sources)
            self.ntotal = int(self.lens.sum())

    return OracleMergeShard


def _worker_merge(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from densephrases_b200.sharded import ShardedIvfPq, sharded_search
    from oracle import encode_ref as E
    from oracle import ivfpq_ref as R
    from tests.test_add_cpu import _merge_packed, _model, _near, _pack
    nlist, nprobe, k = 20, 6, 10
    A, Cm, pq = _model(R, nlist, 11)
    lo, hi = (0, 9) if rank == 0 else (9, nlist)
    Shard = _shard_class()
    rng = np.random.default_rng(12)
    batches = [(_near(A, Cm, rng.integers(0, nlist, n), 13 + i, 0.2), ids) for i, (n, ids) in
               enumerate([(120, None), (60, 5000 + np.arange(60)), (0, np.zeros(0, np.int64)), (50, 6000 + np.arange(50))])]
    shards = []
    for x, ids in batches:
        sh = ShardedIvfPq(nlist, rank=rank, world=world, local=Shard(R, A, Cm, pq, nlist, lo, hi, nprobe))
        if len(x):
            sh.add_with_ids(torch.from_numpy(x), ids)
        shards.append(sh)
    main = shards[0]
    main.merge_from(shards[1:], add_id=7)
    q = _near(A, Cm, rng.integers(0, nlist, 7), 15, 0.3)
    D, I = sharded_search(torch.from_numpy(q), k, world, None, main.local.coarse_local, main.local.search_preassigned, _pack, _merge_packed)
    if rank == 0:
        parts = []
        for x, ids in batches:                               # each unsharded index from its own batch, then the merge definition
            full = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
            if len(x):
                full.add_with_ids(x, ids)
            parts.append((full.list_len, full.codes if full.codes is not None else np.zeros((0, 96), np.uint8), full.ids))
        lens, codes, ids = np_merge(parts[0], parts[1:], add_id=7)
        ref = E.GrowableRefIndex(A, pq, lens, centroids=Cm, codes=codes, ids=ids)
        Dr, Ir = ref.search(q, k, nprobe)
        np.savez(out, D=D.numpy(), I=I.numpy(), Dr=Dr, Ir=Ir, lens=main.local.lens, lens_r=lens, ntotal=main.ntotal,
                 local_ids=main.local.local.ids, ids_r=ids)
    dist.destroy_process_group()


def test_gloo_world2_sharded_merge_equals_unsharded(tmp_path, oracle):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "merge2.npz")
    mp.spawn(_worker_merge, args=(2, port, out), nprocs=2, join=True)
    g = np.load(out)
    assert np.array_equal(g["lens"], g["lens_r"]) and int(g["ntotal"]) == 230
    assert np.array_equal(g["local_ids"], g["ids_r"][:int(g["lens_r"][:9].sum())])      # rank 0 holds exactly its lists' merged rows
    assert_topk_equal(g["D"], g["I"], g["Dr"], g["Ir"], "sharded merge vs the unsharded merge definition")
