"""CPU: the definition of removing vectors (oracle/remove_ref, DESIGN.md 3.2): the literal faiss IndexIVF::remove_ids loop equals its
closed form, hand examples, and a sharded remove over gloo with oracle-backed shards equals the unsharded oracle."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import remove_ref as RR
from tests.helpers import assert_topk_equal

RAGGED = [0, 1, 31, 32, 33, 64, 65, 1000]


def ragged_arrays(seed, lens=RAGGED):
    rng = np.random.default_rng(seed)
    lens = np.asarray(lens, np.int64)
    n = int(lens.sum())
    return lens, rng.integers(0, 256, (n, 96), dtype=np.uint8), rng.permutation(n).astype(np.int64) * 2 + 5


@pytest.mark.parametrize("frac", [0.0, 0.01, 0.3, 0.7, 1.0])
def test_literal_loop_equals_closed_form_label_sets(frac):
    for seed in range(4):
        lens, codes, ids = ragged_arrays(seed)
        rng = np.random.default_rng(100 + seed)
        sel = rng.choice(ids, int(frac * len(ids)), replace=False)
        sel = np.concatenate([sel, sel[:5], [-1, -7, 10**12, 4]])          # duplicates, negative and absent labels
        rng.shuffle(sel)
        a, b = RR.ref_remove(lens, codes, ids, sel), RR.np_remove(lens, codes, ids, sel)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
        assert a[3].sum() == int(np.isin(ids, sel).sum())
        assert not np.isin(a[2], sel).any()
        assert sorted(a[2]) == sorted(ids[~np.isin(ids, sel)])


def test_literal_loop_equals_closed_form_label_ranges():
    lens, codes, _ = ragged_arrays(3)
    ids = np.arange(int(lens.sum()), dtype=np.int64)                            # list-major labels: a range is a run of lists
    perm = np.random.default_rng(1).permutation(len(ids)).astype(np.int64)      # labels scattered over the lists
    for labels in (ids, perm):
        for lo, hi in [(0, 0), (5, 3), (0, 40), (40, 97), (100, 1200), (-10, 5), (0, 10**9), (1200, 1226)]:
            a, b = RR.ref_remove(lens, codes, labels, range(lo, hi)), RR.np_remove(lens, codes, labels, range(lo, hi))
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
            assert a[3].sum() == int(((labels >= lo) & (labels < hi)).sum())


def test_hand_examples():
    lens = np.array([4], np.int64)
    codes = np.arange(4, dtype=np.uint8)[:, None].repeat(96, 1)
    ids = np.array([10, 11, 12, 13], np.int64)                                  # [a, b, c, d]
    for fn in (RR.ref_remove, RR.np_remove):
        l, c, i, per = fn(lens, codes, ids, np.array([12, 10]))                 # [a*, b, c*, d] -> [d, b]
        assert list(l) == [2] and list(i) == [13, 11] and list(c[:, 0]) == [3, 1] and list(per) == [2]
        l, c, i, per = fn(lens, codes, ids, range(10, 14))                      # the whole list
        assert list(l) == [0] and len(i) == 0 and c.shape == (0, 96)
        l, c, i, per = fn(lens, codes, ids, np.array([99, -1]))                 # nothing
        assert list(l) == [4] and list(i) == list(ids) and np.array_equal(c, codes) and list(per) == [0]
        l, c, i, per = fn(lens, codes, ids, np.array([10]))                     # the last row fills the hole
        assert list(i) == [13, 11, 12]


def test_ref_index_remove_makes_labels_explicit(oracle):
    from tests.helpers import opq_matrix
    nlist = 6
    lens = np.array([3, 0, 5, 1, 40, 2], np.int64)
    ref = RR.RemovableRefIndex(opq_matrix(1), oracle.gen_pq(1), lens, seed=1)    # synthetic codes, sequential labels
    codes = np.concatenate([ref.list_codes(l) for l in range(nlist)])
    n, per = ref.remove_ids(range(5, 5))                                         # empty selector: nothing changes
    assert n == 0 and not per.any() and ref.ids is None
    n, per = ref.remove_ids(range(100, 200))                                     # selects nothing, still explicit afterwards
    assert n == 0 and ref.ids is not None and np.array_equal(ref.ids, np.arange(51))
    n, per = ref.remove_ids(range(3, 10))
    assert n == 7 and list(per) == [0, 0, 5, 1, 1, 0]
    assert list(ref.list_ids(4)[:3]) == [48, 10, 11] and ref.ntotal == 44
    assert np.array_equal(ref.list_codes(4)[0], codes[48])


# ---- sharded remove over gloo: every rank removes the same selector from an oracle-backed list-range shard ----
def _shard_class():
    from tests.test_add_cpu import _OracleAddShard

    class OracleRemoveShard(_OracleAddShard):
        """_OracleAddShard that can also remove (its own lists' rows) and take the other shards' list lengths, like
        dph_index_remove_ids / dph_index_sync_list_len on a shard."""

        def __init__(self, R, A, Cm, pq, nlist, lo, hi, nprobe):
            super().__init__(R, A, Cm, pq, nlist, lo, hi, nprobe)
            self.local = RR.RemovableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)

        def list_len(self):
            return self.lens.copy()

        def remove_ids_per_list(self, sel):
            _, per = self.local.remove_ids(sel)
            assert not per[:self.lo].any() and not per[self.hi:].any()
            self.lens -= per
            self.ntotal = int(self.lens.sum())
            return per

        def sync_list_len(self, list_len):
            assert np.array_equal(list_len[self.lo:self.hi], self.lens[self.lo:self.hi])
            self.lens = np.array(list_len, np.int64)
            self.ntotal = int(self.lens.sum())

    return OracleRemoveShard


def _worker_remove(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from densephrases_b200.sharded import ShardedIvfPq, sharded_search
    from oracle import ivfpq_ref as R
    from tests.test_add_cpu import _merge_packed, _model, _near, _pack
    nlist, nprobe, k = 20, 6, 10
    A, Cm, pq = _model(R, nlist, 11)
    lo, hi = (0, 9) if rank == 0 else (9, nlist)
    shard = _shard_class()(R, A, Cm, pq, nlist, lo, hi, nprobe)
    sh = ShardedIvfPq(nlist, rank=rank, world=world, local=shard)
    full = RR.RemovableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    rng = np.random.default_rng(12)
    x1 = _near(A, Cm, rng.integers(0, nlist, 150), 13, 0.2)
    x2 = _near(A, Cm, rng.integers(0, 9, 40), 14, 0.2)                       # only shard 0's lists
    ids2 = 5000 + np.arange(40)
    for g in (sh, full):
        g.add_with_ids(x1, None) if g is full else g.add_with_ids(torch.from_numpy(x1))
        g.add_with_ids(x2, ids2)
    counts = []
    for sel in (range(30, 70), np.array([5003, 5010, 5010, 5039, -2, 77777]), rng.choice(150, 25, replace=False).astype(np.int64),
                range(0, 0)):
        n = sh.remove_ids(sel)
        nr, _ = full.remove_ids(sel)
        counts.append((n, nr))
    q = _near(A, Cm, rng.integers(0, nlist, 7), 15, 0.3)
    D, I = sharded_search(torch.from_numpy(q), k, world, None, shard.coarse_local, shard.search_preassigned, _pack, _merge_packed)
    if rank == 0:
        Dr, Ir = full.search(q, k, nprobe)
        np.savez(out, D=D.numpy(), I=I.numpy(), Dr=Dr, Ir=Ir, lens=shard.lens, lens_r=full.list_len, ntotal=shard.ntotal,
                 ntotal_r=full.ntotal, counts=np.array(counts))
    dist.destroy_process_group()


def test_gloo_world2_sharded_remove_equals_unsharded(tmp_path, oracle):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "remove2.npz")
    mp.spawn(_worker_remove, args=(2, port, out), nprocs=2, join=True)
    g = np.load(out)
    assert np.array_equal(g["lens"], g["lens_r"]) and int(g["ntotal"]) == int(g["ntotal_r"]) == 190 - int(g["counts"][:, 1].sum())
    c = g["counts"]
    assert np.array_equal(c[:, 0], c[:, 1]) and c[0, 0] == 40 and c[1, 0] == 3 and c[3, 0] == 0
    assert_topk_equal(g["D"], g["I"], g["Dr"], g["Ir"], "sharded removes vs the unsharded oracle")
