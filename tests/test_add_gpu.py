"""GPU: growing a resident index (dph_index_encode / dph_index_add_with_ids / dph_index_copy_lists) against the CPU oracle.
Encoding is bit-exact (list numbers and codes); after any sequence of adds the device state equals set_lists of the concatenated
list-major arrays, so lists(), reconstruct and search all match the oracle index built from those arrays."""
import numpy as np
import pytest

from oracle import encode_ref as E
from tests.helpers import assert_topk_equal, near_queries, opq_matrix

pytestmark = pytest.mark.gpu
SEED = 77


def model(oracle, nlist, seed=SEED):
    return opq_matrix(seed), oracle.gen_centroids(seed, 0, nlist), oracle.gen_pq(seed)


def gpu_index(A, Cm, pq, lens, codes=None, ids=None, shard=None):
    from densephrases_b200 import IvfPqIndex
    ix = IvfPqIndex(len(lens))
    ix.set_opq(A); ix.set_centroids(Cm); ix.set_pq(pq)
    if shard is not None:
        ix.set_shard(*shard)
    ix.set_lists(lens, np.zeros((0, 96), np.uint8) if codes is None else codes, ids)
    return ix


def vectors_near(A, Cm, lists, seed, noise=0.05):
    """x whose rotated image is centroid[l] + noise: each lands in (or next to) list l."""
    rng = np.random.default_rng(seed)
    xr = Cm[np.asarray(lists)] + noise * rng.standard_normal((len(lists), 768))
    return (xr @ A).astype(np.float32)


def assert_lists_equal(ix, ref, what=""):
    lens, codes, ids = ix.lists()
    assert np.array_equal(lens, ref.list_len), what
    assert np.array_equal(codes, ref.codes if ref.codes is not None else np.zeros((0, 96), np.uint8)), what
    assert np.array_equal(ids, ref.ids if ref.ids is not None else np.arange(ref.ntotal)), what


@pytest.mark.parametrize("nlist", [1, 16, 512, 4096])       # 512, 4096: tensor-core coarse candidates + exact re-rank + proof
def test_encode_matches_oracle(oracle, nlist):
    import torch
    A, Cm, pq = model(oracle, nlist)
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    ix = gpu_index(A, Cm, pq, np.zeros(nlist, np.int64))
    rng = np.random.default_rng(nlist)
    for n in (1, 31, 32, 33, 1000):
        x = np.concatenate([vectors_near(A, Cm, rng.integers(0, nlist, n - n // 4), n, noise=0.3),
                            0.5 * rng.standard_normal((n // 4, 768)).astype(np.float32)])
        lr, cr = ref.encode(x)
        lh, ch = ix.encode(x)
        assert np.array_equal(lh, lr) and np.array_equal(ch, cr), f"host n={n}"
        ld, cd = ix.encode(torch.from_numpy(x).cuda())
        assert np.array_equal(ld.cpu().numpy(), lr) and np.array_equal(cd.cpu().numpy(), cr), f"device n={n}"
    assert ix.ntotal == 0


def test_encode_and_add_across_staging_chunks(oracle, monkeypatch):
    import torch
    nlist, n = 64, 1000
    A, Cm, pq = model(oracle, nlist)
    x = vectors_near(A, Cm, np.random.default_rng(0).integers(0, nlist, n), 1, noise=0.3)
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    lr, cr = ref.encode(x)
    monkeypatch.setenv("DPH_UPLOAD_CHUNK_ROWS", "97")          # 11 encode chunks, 1 staging chunk per few lists in lists()
    ix = gpu_index(A, Cm, pq, np.zeros(nlist, np.int64))
    for xx in (x, torch.from_numpy(x).cuda()):
        l, c = ix.encode(xx)
        assert np.array_equal(np.asarray(l.cpu() if hasattr(l, "cpu") else l), lr)
        assert np.array_equal(np.asarray(c.cpu() if hasattr(c, "cpu") else c), cr)
    ix.add(x)
    ix.add(torch.from_numpy(x).cuda())
    ref.add_with_ids(x)
    ref.add_with_ids(x)
    assert_lists_equal(ix, ref, "chunked adds")


def test_planted_ties_pick_lowest_list_and_code(oracle):
    nlist = 32
    A, Cm, pq = model(oracle, nlist)
    Cm = Cm.copy(); pq = pq.copy()
    Cm[9] = Cm[3]                                             # duplicate centroids: every score ties exactly
    pq[:, 200] = pq[:, 17]                                    # duplicate codewords in every sub-quantizer
    code = np.full(96, 200)
    xr = Cm[9] + pq[np.arange(96), code].reshape(768)         # residual == the duplicated codeword (lands on list 3 or 9)
    x = np.stack([xr @ A, (Cm[20] + pq[np.arange(96), code].reshape(768)) @ A]).astype(np.float32)
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    ix = gpu_index(A, Cm, pq, np.zeros(nlist, np.int64))
    lr, cr = ref.encode(x)
    l, c = ix.encode(x)
    assert np.array_equal(l, lr) and np.array_equal(c, cr)
    assert l[0] == 3, "tie between duplicate centroids 3 and 9 must go to the lower list"
    assert (cr == 200).sum() == 0 and (cr == 17).sum() > 0, "duplicate codewords: the lower index must win"


def ragged_model(oracle):
    nlist = 48
    rng = np.random.default_rng(5)
    lens = rng.integers(0, 400, nlist).astype(np.int64)
    lens[[0, 7, 47]] = 0; lens[3] = 1; lens[4] = 32; lens[5] = 33             # stay as they are: nothing is added to them
    lens[[10, 11, 12, 13, 14]] = [0, 1, 31, 32, 33]                          # grow across block boundaries
    A, Cm, pq = model(oracle, nlist)
    codes = np.concatenate([oracle.gen_codes(SEED + 7, l, 0, int(lens[l])) for l in range(nlist)])
    ids = rng.permutation(int(lens.sum())).astype(np.int64) * 3 + 2 * 10**9       # no collision with the labels the tests add
    targets = np.setdiff1d(np.arange(nlist), [0, 7, 47, 3, 4, 5])
    return nlist, lens, A, Cm, pq, codes, ids, targets


@pytest.mark.parametrize("mode", [1, 3, 2, 4, 0])
def test_set_lists_then_two_adds_equals_oracle(oracle, mode):
    import torch
    nlist, lens, A, Cm, pq, codes, ids, targets = ragged_model(oracle)
    ref = E.GrowableRefIndex(A, pq, lens, centroids=Cm, codes=codes, ids=ids)
    ix = gpu_index(A, Cm, pq, lens, codes, ids)
    rng = np.random.default_rng(8)
    x2 = vectors_near(A, Cm, np.concatenate([[10, 11, 12, 13, 14] * 3, rng.choice(targets, 300)]), 2)
    ids2 = 10**9 + rng.permutation(len(x2)).astype(np.int64)
    x3 = vectors_near(A, Cm, rng.choice(targets, 500), 3)
    ix.add_with_ids(x2, ids2)
    ix.add(torch.from_numpy(x3).cuda())                       # device buffers, default labels ntotal + i
    ref.add_with_ids(x2, ids2)
    ref.add_with_ids(x3)
    assert ix.ntotal == ref.ntotal == int(lens.sum()) + len(x2) + len(x3)
    assert (ref.list_len[[0, 7, 47, 3, 4, 5]] == [0, 0, 0, 1, 32, 33]).all()
    assert_lists_equal(ix, ref, "set_lists + add + add")
    v, f = ix.reconstruct_batch(ref.ids)
    vr, fr = ref.reconstruct(ref.ids)
    assert f.all() and np.array_equal(v.view(np.int32), vr.view(np.int32))
    ix.nprobe = 12
    ix.set_scan_mode(mode)
    q = np.concatenate([near_queries(ref, 15, 99), x3[:4]])
    D, I = ix.search(q, 10)
    Dr, Ir = ref.search(q, 10, 12)
    assert_topk_equal(D, I, Dr, Ir, f"mode={mode}")


def test_empty_index_grown_by_adds_equals_from_arrays(oracle):
    import torch
    from densephrases_b200 import IvfPqIndex
    nlist = 128
    A, Cm, pq = model(oracle, nlist)
    zeros = np.zeros(nlist, np.int64)
    ix = IvfPqIndex.from_arrays(A, Cm, pq, zeros, np.zeros((0, 96), np.uint8))
    ref = E.GrowableRefIndex(A, pq, zeros, centroids=Cm)
    rng = np.random.default_rng(3)
    for i, n in enumerate((700, 1, 333)):
        x = vectors_near(A, Cm, rng.integers(0, nlist, n), 10 + i, noise=0.2)
        ix.add(x if i != 1 else torch.from_numpy(x).cuda())
        ref.add_with_ids(x)
    full = IvfPqIndex.from_arrays(A, Cm, pq, ref.list_len, ref.codes, ref.ids)
    assert_lists_equal(ix, ref)
    assert np.array_equal(np.concatenate([a.ravel().view(np.uint8) for a in ix.lists()]),
                          np.concatenate([a.ravel().view(np.uint8) for a in full.lists()]))
    assert ix.device_bytes > 0
    q = near_queries(ref, 20, 4)
    for g in (ix, full):
        g.nprobe = 8
    D, I = ix.search(q, 10)
    Df, If = full.search(q, 10)
    Dr, Ir = ref.search(q, 10, 8)
    assert np.array_equal(D.view(np.int32), Df.view(np.int32)) and np.array_equal(I, If)
    assert_topk_equal(D, I, Dr, Ir, "grown from empty")


def test_synthetic_labels_survive_an_add(oracle):
    from densephrases_b200 import IvfPqIndex
    nlist = 24
    lens = np.random.default_rng(1).integers(0, 90, nlist).astype(np.int64)
    A = opq_matrix(SEED)
    ref = E.GrowableRefIndex(A, oracle.gen_pq(SEED), lens, centroids=oracle.gen_centroids(SEED, 0, nlist), seed=SEED)
    ix = IvfPqIndex(nlist)
    ix.set_opq(A); ix.gen_pq(SEED); ix.gen_centroids(SEED); ix.set_lists_synthetic(lens, SEED)
    old = np.arange(ref.ntotal, dtype=np.int64)
    v0, f0 = ix.reconstruct_batch(old)
    x = vectors_near(A, ref.centroids(), np.random.default_rng(2).integers(0, nlist, 200), 5)
    ix.add(x)
    ref.add_with_ids(x)
    v1, f1 = ix.reconstruct_batch(old)
    assert f0.all() and f1.all() and np.array_equal(v0.view(np.int32), v1.view(np.int32))
    new = np.arange(len(old), len(old) + len(x), dtype=np.int64)
    vn, fn = ix.reconstruct_batch(new)
    vr, fr = ref.reconstruct(new)
    assert fn.all() and np.array_equal(vn.view(np.int32), vr.view(np.int32))
    assert_lists_equal(ix, ref)
    ix.nprobe = 6
    D, I = ix.search(x[:12], 10)
    Dr, Ir = ref.search(x[:12], 10, 6)
    assert_topk_equal(D, I, Dr, Ir, "synthetic + add")


def test_shard_halves_add_the_same_batch(oracle):
    import torch
    from densephrases_b200.ivfpq import merge_shards
    nlist, lens, A, Cm, pq, codes, ids, targets = ragged_model(oracle)
    off = np.concatenate([[0], np.cumsum(lens)])
    h = 20
    full = gpu_index(A, Cm, pq, lens, codes, ids)
    halves = [gpu_index(A, Cm, pq, lens, codes[off[a]:off[b]], ids[off[a]:off[b]], shard=(a, b)) for a, b in ((0, h), (h, nlist))]
    x = vectors_near(A, Cm, np.random.default_rng(4).integers(0, nlist, 400), 6, noise=0.2)
    for g in [full] + halves:
        g.add(x)
        g.nprobe = 16
    lf, cf, idf = full.lists()
    parts = [g.lists() for g in halves]
    assert all(np.array_equal(p[0], lf) for p in parts) and all(g.ntotal == full.ntotal for g in halves)
    assert np.array_equal(np.concatenate([p[1] for p in parts]), cf) and np.array_equal(np.concatenate([p[2] for p in parts]), idf)
    q = torch.from_numpy(x[:40]).cuda()
    D, I = full.search(q, 10)
    res = [g.search_partial(q, 10) for g in halves]
    Dm, Im = merge_shards(*(torch.stack([r[i] for r in res]).contiguous() for i in range(3)), 10)
    assert torch.equal(Dm.view(torch.int32), D.view(torch.int32)) and torch.equal(Im, I)


def test_search_probes_equal_encode_lists(oracle):
    nlist = 64
    A, Cm, pq = model(oracle, nlist)
    ix = gpu_index(A, Cm, pq, np.zeros(nlist, np.int64))
    x = vectors_near(A, Cm, np.random.default_rng(9).integers(0, nlist, 50), 9, noise=0.4)
    ix.add(x)
    ix.nprobe = 4
    ix.search(x, 5)
    assert np.array_equal(ix.last_probes(len(x))[:, 0], ix.encode(x)[0])


def test_repeated_label_reconstructs_to_last_row(oracle):
    nlist = 16
    A, Cm, pq = model(oracle, nlist)
    ix = gpu_index(A, Cm, pq, np.zeros(nlist, np.int64))
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    xa = vectors_near(A, Cm, [2, 5, 5], 1)
    xb = vectors_near(A, Cm, [11], 2)
    ix.add_with_ids(xa, np.array([5, 6, 5]))
    ix.add_with_ids(xb, np.array([5]))
    ref.add_with_ids(xa, np.array([5, 6, 5]))
    lb, cb = ref.add_with_ids(xb, np.array([5]))
    assert_lists_equal(ix, ref)
    assert (ix.lists()[2] == 5).sum() == 3
    v, f = ix.reconstruct_batch(np.array([5]))
    want = (pq[np.arange(96), cb[0]].reshape(768) + Cm[lb[0]]).astype(np.float32)
    assert f.all() and np.array_equal(v[0].view(np.int32), want.view(np.int32))
    ix.nprobe = nlist
    D, I = ix.search(xa[1:2], 4)
    Dr, Ir = ref.search(xa[1:2], 4, nlist)
    assert_topk_equal(D, I, Dr, Ir, "repeated labels")


def test_rejected_adds_leave_the_index_unchanged(oracle):
    nlist, lens, A, Cm, pq, codes, ids, _ = ragged_model(oracle)
    ix = gpu_index(A, Cm, pq, lens, codes, ids)
    ix.nprobe = 8
    ref = E.GrowableRefIndex(A, pq, lens, centroids=Cm, codes=codes, ids=ids)
    q = near_queries(ref, 8, 1)
    D0, I0 = ix.search(q, 10)
    L0 = ix.lists()
    n0, b0 = ix.ntotal, ix.device_bytes
    x = vectors_near(A, Cm, np.arange(10), 3)
    bad_x = x.copy(); bad_x[4, 100] = np.nan
    inf_x = x.copy(); inf_x[0, 0] = np.inf
    with pytest.raises(RuntimeError):
        ix.add_with_ids(x, np.arange(10) - 1)                  # label -1
    with pytest.raises(RuntimeError):
        ix.add(bad_x)
    with pytest.raises(RuntimeError):
        ix.add(inf_x)
    with pytest.raises(RuntimeError):
        ix.add_with_ids(x, np.arange(9))                       # ids / n mismatch
    with pytest.raises(RuntimeError):
        ix.add(x[:, :700])                                     # wrong dimension
    assert ix.ntotal == n0 and ix.device_bytes == b0
    D1, I1 = ix.search(q, 10)
    assert np.array_equal(D0.view(np.int32), D1.view(np.int32)) and np.array_equal(I0, I1)
    assert all(np.array_equal(a, b) for a, b in zip(L0, ix.lists()))
    ix.add(np.zeros((0, 768), np.float32))                    # n = 0: no-op
    assert ix.ntotal == n0
