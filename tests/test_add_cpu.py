"""CPU: the floating-point definition of encoding added vectors (oracle/encode_ref ref_encode, DESIGN.md 3 "Growing the index") and the
oracle's add_with_ids, plus the sharded add over gloo with an oracle-backed shard."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import encode_ref as E
from tests.helpers import assert_topk_equal, opq_matrix


def _model(R, nlist, seed):
    return opq_matrix(seed), R.gen_centroids(seed, 0, nlist), R.gen_pq(seed)


def _near(A, Cm, lists, seed, noise):
    rng = np.random.default_rng(seed)
    return ((Cm[np.asarray(lists)] + noise * rng.standard_normal((len(lists), A.shape[0]))) @ A).astype(np.float32)


def test_c_encode_equals_numpy_and_coarse_top1(oracle):
    nlist = 24
    A, Cm, pq = _model(oracle, nlist, 3)
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    x = np.concatenate([_near(A, Cm, np.arange(12) * 2, 1, 0.3), 0.4 * np.random.default_rng(2).standard_normal((5, 768)).astype(np.float32)])
    l, c = ref.encode(x)
    ln, cn = E.np_encode(x, A, Cm, pq)
    assert np.array_equal(l, ln) and np.array_equal(c, cn)
    assert np.array_equal(l, ref.coarse(ref.rotate(x), 1)[1][:, 0])


def test_codes_equal_fp64_argmin_outside_rounding_gaps(oracle):
    """Where the fp64 gap between the best two codewords exceeds a bound on the fp32 chain's error, the fp32 argmin is the fp64 one.
    Bound: the 8-term squared distance of residual entries |r| and |c| <= 2 carries a relative error < 20 * 2^-24 per term, so
    |dist32 - dist64| <= 20 * 2^-24 * 8 * 16 < 2e-4 (plus the residual's own rounding, covered by recomputing from the fp32 residual)."""
    nlist = 40
    A, Cm, pq = _model(oracle, nlist, 4)
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    x = _near(A, Cm, np.random.default_rng(0).integers(0, nlist, 300), 5, 0.25)
    l, c = ref.encode(x)
    r = (ref.rotate(x) - Cm[l]).astype(np.float64).reshape(len(x), 96, 1, 8)
    d64 = ((r - pq.astype(np.float64)[None]) ** 2).sum(-1)                   # [n, 96, 256]
    part = np.sort(d64, axis=-1)
    decided = part[..., 1] - part[..., 0] > 2e-4
    assert decided.mean() > 0.99
    assert np.array_equal(c[decided], d64.argmin(-1)[decided])


def test_planted_ties_lowest_list_and_codeword(oracle):
    nlist = 16
    A, Cm, pq = _model(oracle, nlist, 6)
    Cm = Cm.copy(); pq = pq.copy()
    Cm[11] = Cm[4]
    pq[:, 250] = pq[:, 30]
    xr = Cm[11] + pq[np.arange(96), np.full(96, 250)].reshape(768)
    x = np.stack([xr @ A, xr @ A]).astype(np.float32)
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    l, c = ref.encode(x)
    ln, cn = E.np_encode(x, A, Cm, pq)
    assert np.array_equal(l, ln) and np.array_equal(c, cn)
    assert (l == 4).all() and not (c == 250).any() and (c == 30).sum() > 48


def test_ref_add_with_ids_order_and_default_labels(oracle):
    nlist = 8
    A, Cm, pq = _model(oracle, nlist, 7)
    lens = np.array([2, 0, 1, 0, 0, 3, 0, 1], np.int64)
    ref = E.GrowableRefIndex(A, pq, lens, centroids=Cm, seed=7)              # synthetic codes, sequential labels
    old_codes = np.concatenate([ref.list_codes(l) for l in range(nlist)])
    x = _near(A, Cm, [5, 1, 5, 2, 5, 1], 8, 0.05)
    l, c = ref.add_with_ids(x)
    assert list(l) == [5, 1, 5, 2, 5, 1]
    assert np.array_equal(ref.list_len, lens + np.bincount(l, minlength=nlist))
    assert list(ref.list_ids(5)) == [3, 4, 5, 7, 9, 11] and list(ref.list_ids(1)) == [8, 12]
    assert list(ref.list_ids(2)) == [2, 10] and ref.ntotal == 13
    assert np.array_equal(ref.list_codes(5)[3:], c[[0, 2, 4]]) and np.array_equal(ref.list_codes(5)[:3], old_codes[3:6])
    l2, c2 = ref.add_with_ids(x[:2], ids=np.array([100, 3]))
    assert list(ref.list_ids(5))[-1] == 100 and list(ref.list_ids(1))[-1] == 3 and ref.ntotal == 15


# ---- sharded add over gloo: every rank adds the same batch to an oracle-backed list-range shard ----
def _fkey(f):
    b = np.asarray(f, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return np.where(b & 0x80000000, (~b) & 0xFFFFFFFF, b | 0x80000000)


def _fkey_inv(k):
    k = np.asarray(k, dtype=np.uint64)
    return np.where(k & 0x80000000, k & 0x7FFFFFFF, (~k) & 0xFFFFFFFF).astype(np.uint32).view(np.float32)


class _OracleAddShard:
    """IvfPqIndex-shaped list-range shard backed by the oracle: it stores only the rows of lists [lo, hi) and counts the others,
    like dph_index_add_with_ids on a shard."""

    def __init__(self, R, A, Cm, pq, nlist, lo, hi, nprobe):
        self.R, self.lo, self.hi, self.nprobe = R, lo, hi, nprobe
        self.lens = np.zeros(nlist, np.int64)                               # ALL lists
        self.local = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
        self.ntotal = 0

    def add_with_ids(self, x, ids):
        l, c = self.local.encode(x.numpy() if hasattr(x, "numpy") else x)
        ids = self.ntotal + np.arange(len(l)) if ids is None else np.asarray(ids, np.int64)
        mine = (l >= self.lo) & (l < self.hi)
        self.local.append(l[mine], c[mine], ids[mine])
        self.lens += np.bincount(l, minlength=len(self.lens))
        self.ntotal += len(l)

    def coarse_local(self, x):
        xr = self.local.rotate(x.numpy())
        S = self.R.np_matmul_nt_seq(xr, self.local.centroids()[self.lo:self.hi])
        keys = np.zeros((len(xr), self.nprobe), dtype=np.uint64)
        for q in range(len(xr)):
            for r, j in enumerate(sorted(range(self.hi - self.lo), key=lambda j: (-float(S[q, j]), j))[:self.nprobe]):
                keys[q, r] = (_fkey(S[q, j]) << np.uint64(32)) | np.uint64(0xFFFFFFFF - (j + self.lo))
        self._xr = xr
        return torch.from_numpy(keys.view(np.int64))

    def search_preassigned(self, keys_g, k):
        kg = keys_g.numpy().view(np.uint64)
        n = kg.shape[1]
        key = np.full((n, self.nprobe), -1, dtype=np.int64)
        for q in range(n):
            allk = sorted((int(v) for v in kg[:, q, :].ravel() if v != 0), reverse=True)[:self.nprobe]
            key[q, :len(allk)] = [0xFFFFFFFF - (v & 0xFFFFFFFF) for v in allk]
        D, I = self.local.search_preassigned(self._xr, np.where((key >= self.lo) & (key < self.hi), key, -1), k)
        G = np.zeros_like(I)
        for q in range(n):
            starts = np.concatenate([[0], np.cumsum([self.lens[l] if l >= 0 else 0 for l in key[q]])])     # global list lengths
            for r in range(k):
                if I[q, r] >= 0:
                    l, off = self.local.locate(np.array([I[q, r]]))
                    G[q, r] = starts[list(key[q]).index(int(l[0]))] + int(off[0])
        return torch.from_numpy(D), torch.from_numpy(I), torch.from_numpy(G.astype(np.int32))


def _pack(D, I, G):
    ck = (_fkey(D.numpy()) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - (G.numpy().astype(np.int64) & 0xFFFFFFFF).astype(np.uint64))
    return torch.from_numpy(np.ascontiguousarray(np.stack([np.where(I.numpy() >= 0, ck, 0).view(np.int64), I.numpy()], axis=-1)))


def _merge_packed(Pg, k):
    Pn = Pg.numpy()
    n = Pn.shape[1]
    D = np.full((n, k), np.float32(-3.4028234663852886e38), dtype=np.float32)
    I = np.full((n, k), -1, dtype=np.int64)
    for q in range(n):
        ent = sorted(((int(np.uint64(Pn[s, q, r, 0])), int(Pn[s, q, r, 1])) for s in range(Pn.shape[0]) for r in range(k) if Pn[s, q, r, 0] != 0),
                     reverse=True)[:k]
        for i, (ckey, lab) in enumerate(ent):
            D[q, i], I[q, i] = _fkey_inv(ckey >> 32), lab
    return torch.from_numpy(D), torch.from_numpy(I)


def _worker_add(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from densephrases_b200.sharded import ShardedIvfPq, sharded_search
    from oracle import ivfpq_ref as R
    nlist, nprobe, k = 20, 6, 10
    A, Cm, pq = _model(R, nlist, 11)
    lo, hi = (0, 9) if rank == 0 else (9, nlist)
    shard = _OracleAddShard(R, A, Cm, pq, nlist, lo, hi, nprobe)
    sh = ShardedIvfPq(nlist, rank=rank, world=world, local=shard)
    rng = np.random.default_rng(12)
    x1 = _near(A, Cm, rng.integers(0, nlist, 120), 13, 0.2)
    x2 = _near(A, Cm, rng.integers(0, nlist, 80), 14, 0.2)
    ids2 = 5000 + rng.permutation(80)
    sh.add_with_ids(torch.from_numpy(x1))
    sh.add_with_ids(torch.from_numpy(x2), ids2)
    q = _near(A, Cm, rng.integers(0, nlist, 7), 15, 0.3)
    D, I = sharded_search(torch.from_numpy(q), k, world, None, shard.coarse_local, shard.search_preassigned, _pack, _merge_packed)
    if rank == 0:
        # the unsharded oracle index built from the concatenated arrays
        l1, c1 = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm).encode(x1)
        l2, c2 = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm).encode(x2)
        l, c, ids = np.concatenate([l1, l2]), np.concatenate([c1, c2]), np.concatenate([np.arange(120), ids2])
        order = np.argsort(l, kind="stable")
        full = E.GrowableRefIndex(A, pq, np.bincount(l, minlength=nlist), centroids=Cm, codes=c[order], ids=ids[order])
        Dr, Ir = full.search(q, k, nprobe)
        np.savez(out, D=D.numpy(), I=I.numpy(), Dr=Dr, Ir=Ir, lens=shard.lens, lens_r=full.list_len, ntotal=shard.ntotal)
    dist.destroy_process_group()


def test_gloo_world2_sharded_add_equals_unsharded(tmp_path, oracle):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "add2.npz")
    mp.spawn(_worker_add, args=(2, port, out), nprocs=2, join=True)
    g = np.load(out)
    assert np.array_equal(g["lens"], g["lens_r"]) and int(g["ntotal"]) == 200
    assert_topk_equal(g["D"], g["I"], g["Dr"], g["Ir"], "sharded adds vs unsharded oracle of the concatenated arrays")
