"""GPU: replacing the resident lists of a handle (dph_index_set_lists / _synthetic).  A re-set handle equals a fresh one given the same
call: a call without labels leaves sequential labels, device_bytes() counts every array once, and a rejected call changes nothing."""
import numpy as np
import pytest

from oracle import encode_ref as E
from tests.helpers import assert_topk_equal, near_queries, opq_matrix

pytestmark = pytest.mark.gpu
SEED = 31


def lists_model(oracle, nlist=40):
    rng = np.random.default_rng(SEED)
    lens = rng.integers(0, 200, nlist).astype(np.int64)
    lens[[0, 9]] = 0; lens[5] = 32; lens[6] = 33
    A, Cm, pq = opq_matrix(SEED), oracle.gen_centroids(SEED, 0, nlist), oracle.gen_pq(SEED)
    codes = np.concatenate([oracle.gen_codes(SEED + 1, l, 0, int(lens[l])) for l in range(nlist)])
    perm_ids = rng.permutation(int(lens.sum())).astype(np.int64) * 5 + 10**6
    return lens, A, Cm, pq, codes, perm_ids


def new_index(A, Cm, pq):
    from densephrases_b200 import IvfPqIndex
    ix = IvfPqIndex(len(Cm))
    ix.set_opq(A); ix.set_centroids(Cm); ix.set_pq(pq)
    return ix


def vectors_near(A, Cm, n, seed):
    rng = np.random.default_rng(seed)
    return ((Cm[rng.integers(0, len(Cm), n)] + 0.05 * rng.standard_normal((n, 768))) @ A).astype(np.float32)


def assert_sequential(ix, fresh, ref, what):
    """ix holds what `fresh` (the same set call on a new handle) holds, with labels 0..ntotal-1, and matches the oracle."""
    got = ix.lists()
    assert np.array_equal(got[2], np.arange(ref.ntotal)), what
    assert all(np.array_equal(a, b) for a, b in zip(got, fresh.lists())), what
    labels = np.arange(ref.ntotal, dtype=np.int64)
    v, f = ix.reconstruct_batch(labels)
    vr, _ = ref.reconstruct(labels)
    assert f.all() and np.array_equal(v.view(np.int32), vr.view(np.int32)), what
    ix.nprobe = 8
    q = near_queries(ref, 16, 5)
    assert_topk_equal(*ix.search(q, 10), *ref.search(q, 10, 8), what)


def test_reset_without_labels_gives_sequential_labels(oracle):
    lens, A, Cm, pq, codes, perm_ids = lists_model(oracle)
    ix = new_index(A, Cm, pq)
    ix.set_lists(lens, codes, perm_ids)
    ix.set_lists(lens, codes)                                  # same lengths: old and new label arrays have the same size
    fresh = new_index(A, Cm, pq)
    fresh.set_lists(lens, codes)
    assert_sequential(ix, fresh, E.GrowableRefIndex(A, pq, lens, centroids=Cm, codes=codes), "set_lists with labels, then without")

    ix.add(vectors_near(A, Cm, 300, 1))                         # the add makes the labels explicit
    lens2 = ix.list_len()
    ix.set_lists_synthetic(lens2, SEED)
    fresh = new_index(A, Cm, pq)
    fresh.set_lists_synthetic(lens2, SEED)
    assert_sequential(ix, fresh, E.GrowableRefIndex(A, pq, lens2, centroids=Cm, seed=SEED), "add, then set_lists_synthetic")


@pytest.mark.parametrize("labels", [False, True])
def test_reset_counts_device_bytes_once(oracle, labels):
    from densephrases_b200 import IvfPqIndex
    lens, A, Cm, pq, codes, perm_ids = lists_model(oracle)
    ids = perm_ids if labels else None

    def build(times):
        ix = IvfPqIndex(len(lens))
        for _ in range(times):
            ix.set_opq(A); ix.set_centroids(Cm); ix.set_pq(pq); ix.gen_centroids(SEED); ix.gen_pq(SEED)
            ix.set_lists(lens, codes, ids)
        return ix

    nlist, nb, rows = len(lens), int(((lens + 31) // 32).sum()), int(lens.sum())
    want = 4 * (768 * 768 + nlist * 768 + 96 * 256 * 8) + nlist * 4 + (nlist + 1) * 8 + nlist * 8 + nb * 3072
    if labels:
        want += nb * 32 * 8 + 2 * rows * 8
    assert build(1).device_bytes == want
    assert build(2).device_bytes == want
    ix = build(1)
    ix.add(vectors_near(A, Cm, 200, 2))
    ix.set_lists(lens, codes, ids)
    assert ix.device_bytes == want


def test_rejected_set_lists_leaves_the_index_unchanged(oracle):
    lens, A, Cm, pq, codes, perm_ids = lists_model(oracle)
    ix = new_index(A, Cm, pq)
    ix.set_lists(lens, codes, perm_ids)
    ix.nprobe = 8
    q = near_queries(E.GrowableRefIndex(A, pq, lens, centroids=Cm, codes=codes, ids=perm_ids), 16, 2)
    D0, I0 = ix.search(q, 10)
    L0, n0, b0 = ix.lists(), ix.ntotal, ix.device_bytes
    for bad in (-1, 2**31):
        bad_lens = lens.copy()
        bad_lens[7] = bad
        with pytest.raises(RuntimeError, match="bad list length"):
            ix.set_lists(bad_lens, codes)
        with pytest.raises(RuntimeError, match="bad list length"):
            ix.set_lists_synthetic(bad_lens, SEED)
        assert np.array_equal(ix.list_len(), lens)
        assert ix.ntotal == n0 and ix.device_bytes == b0
        assert all(np.array_equal(a, b) for a, b in zip(L0, ix.lists()))
        D, I = ix.search(q, 10)
        assert np.array_equal(D.view(np.int32), D0.view(np.int32)) and np.array_equal(I, I0)
