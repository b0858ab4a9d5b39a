"""GPU: removing vectors from a resident index (dph_index_remove_ids / dph_index_sync_list_len) against the CPU oracle.  After any
sequence of adds and removes the device state equals set_lists of the oracle's list-major arrays (faiss' IndexIVF::remove_ids loop
without a direct map, DESIGN.md 3.2), so lists(), reconstruct and search all match the oracle index built from those arrays."""
import ctypes as C

import numpy as np
import pytest

from oracle import remove_ref as RR
from tests.helpers import assert_topk_equal, near_queries, opq_matrix
from tests.test_add_gpu import SEED, assert_lists_equal, gpu_index, model, ragged_model, vectors_near

pytestmark = pytest.mark.gpu
NEG = np.float32(-3.4028234663852886e38)


def ragged_pair(oracle, shard=None):
    nlist, lens, A, Cm, pq, codes, ids, targets = ragged_model(oracle)
    ref = RR.RemovableRefIndex(A, pq, lens, centroids=Cm, codes=codes, ids=ids)
    return gpu_index(A, Cm, pq, lens, codes, ids, shard=shard), ref


def synthetic_pair(oracle, lens, seed=SEED):
    from densephrases_b200 import IvfPqIndex
    A = opq_matrix(seed)
    ref = RR.RemovableRefIndex(A, oracle.gen_pq(seed), lens, centroids=oracle.gen_centroids(seed, 0, len(lens)), seed=seed)
    ix = IvfPqIndex(len(lens))
    ix.set_opq(A); ix.gen_pq(seed); ix.gen_centroids(seed); ix.set_lists_synthetic(lens, seed)
    return ix, ref


def remove_both(ix, ref, sel):
    n = ix.remove_ids(sel)
    nr, _ = ref.remove_ids(sel.cpu().numpy() if hasattr(sel, "cpu") else sel)
    assert n == nr
    return n


def assert_not_found(ix, labels):
    v, f = ix.reconstruct_batch(np.asarray(labels, np.int64))
    assert not f.any() and not v.any()


@pytest.mark.parametrize("mode", [1, 3, 2, 4, 0])
def test_range_and_set_remove_after_set_lists(oracle, mode):
    import torch
    ix, ref = ragged_pair(oracle)
    ids0 = ref.ids.copy()
    rng = np.random.default_rng(mode)
    lo = int(np.sort(ids0)[len(ids0) // 3])
    rng_sel = range(lo, lo + 3 * 900)                                        # labels are 2e9 + 3 k: ~900 rows over every list
    assert remove_both(ix, ref, rng_sel) > 800
    assert_lists_equal(ix, ref, "range remove")
    sel = rng.choice(ref.ids, 400, replace=False)
    sel = np.concatenate([sel, sel[:20], [-1, -5, 7, 2 * 10**9 + 1]])       # duplicates, negative and absent labels
    rng.shuffle(sel)
    assert remove_both(ix, ref, torch.from_numpy(sel).cuda() if mode == 0 else sel) == 400
    assert_lists_equal(ix, ref, "set remove")
    gone = ids0[~np.isin(ids0, ref.ids)]
    assert_not_found(ix, gone)
    v, f = ix.reconstruct_batch(ref.ids)
    vr, _ = ref.reconstruct(ref.ids)
    assert f.all() and np.array_equal(v.view(np.int32), vr.view(np.int32))
    ix.nprobe = 12
    ix.set_scan_mode(mode)
    q = near_queries(ref, 24, 99)
    D, I = ix.search(q, 10)
    Dr, Ir = ref.search(q, 10, 12)
    assert_topk_equal(D, I, Dr, Ir, f"mode={mode}")
    assert not np.isin(I, gone).any()


def test_synthetic_index_middle_range_makes_labels_explicit(oracle):
    lens = np.random.default_rng(2).integers(0, 300, 40).astype(np.int64)
    ix, ref = synthetic_pair(oracle, lens)
    b0 = ix.device_bytes
    n = ref.ntotal
    assert remove_both(ix, ref, range(n // 3, n // 2)) == n // 2 - n // 3
    assert_lists_equal(ix, ref, "synthetic, middle range")
    assert ix.device_bytes > b0                                               # the index gained labels and a direct map
    assert_not_found(ix, np.arange(n // 3, n // 2))
    v, f = ix.reconstruct_batch(ref.ids)
    assert f.all() and np.array_equal(v.view(np.int32), ref.reconstruct(ref.ids)[0].view(np.int32))
    ix.nprobe = 8
    q = near_queries(ref, 16, 3)
    assert_topk_equal(*ix.search(q, 10), *ref.search(q, 10, 8), "synthetic after remove")


def test_remove_everything_and_empty_selectors(oracle):
    lens = np.array([5, 0, 70, 33, 1], np.int64)
    ix, ref = synthetic_pair(oracle, lens)
    L0, b0 = ix.lists(), ix.device_bytes
    for sel in (range(10, 10), range(9, 3), np.zeros(0, np.int64)):
        assert ix.remove_ids(sel) == 0
    assert ix.device_bytes == b0 and all(np.array_equal(a, b) for a, b in zip(L0, ix.lists()))     # labels still implicit
    assert remove_both(ix, ref, np.array([-3, 10**6], np.int64)) == 0                 # not empty: labels become explicit
    assert ix.device_bytes > b0 and all(np.array_equal(a, b) for a, b in zip(L0, ix.lists()))
    assert ix.remove_ids(range(-2**70, 2**70)) == ref.remove_ids(range(-100, 10**12))[0] == 109     # bounds past int64 are clamped
    assert ix.last_remove_tmp_bytes() > 0
    assert ix.remove_ids(range(5, 5)) == 0 and ix.last_remove_tmp_bytes() == 0                      # the hooks describe the last call
    assert ix.ntotal == ix.ntotal_local == 0 and not ix.list_len().any()
    assert_lists_equal(ix, ref, "everything removed")
    ix.nprobe = len(lens)
    D, I = ix.search(np.random.default_rng(1).standard_normal((3, 768)).astype(np.float32), 5)
    assert (I == -1).all() and (D.view(np.int32) == NEG.view(np.int32)).all()
    x = vectors_near(ref.A, ref.centroids(), [2, 2, 4], 1)                            # and it can grow again
    ix.add_with_ids(x, np.array([7, 8, 9]))
    ref.add_with_ids(x, np.array([7, 8, 9]))
    assert_lists_equal(ix, ref, "re-grown")


def test_label_added_twice_and_update(oracle):
    nlist = 16
    A, Cm, pq = model(oracle, nlist)
    ix = gpu_index(A, Cm, pq, np.zeros(nlist, np.int64))
    ref = RR.RemovableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    xa = vectors_near(A, Cm, [2, 5, 5, 9, 5], 1)
    for g in (ix, ref):
        g.add_with_ids(xa, np.array([5, 6, 5, 40, 41]))
    assert remove_both(ix, ref, np.array([5])) == 2                            # both rows of label 5
    assert_lists_equal(ix, ref)
    assert_not_found(ix, [5])
    xb = vectors_near(A, Cm, [11, 3], 2)                                       # update 40 and 41: remove, then add
    assert remove_both(ix, ref, range(40, 42)) == 2
    ix.add_with_ids(xb, np.array([40, 41]))
    lb, cb = ref.add_with_ids(xb, np.array([40, 41]))
    assert_lists_equal(ix, ref, "update")
    v, f = ix.reconstruct_batch(np.array([40, 41]))
    want = np.stack([pq[np.arange(96), cb[i]].reshape(768) + Cm[lb[i]] for i in range(2)]).astype(np.float32)
    assert f.all() and np.array_equal(v.view(np.int32), want.view(np.int32))
    ix.nprobe = nlist
    assert_topk_equal(*ix.search(xb, 4), *ref.search(xb, 4, nlist), "update")


def test_interleaved_adds_and_removes(oracle):
    import torch
    ix, ref = ragged_pair(oracle)
    A, Cm = ref.A, ref.C
    rng = np.random.default_rng(21)
    next_label = 10**9
    for step in range(10):
        if step % 3 == 0:
            n = int(rng.integers(1, 400))
            x = vectors_near(A, Cm, rng.integers(0, ref.nlist, n), step)
            ids = next_label + np.arange(n)
            next_label += n
            ix.add_with_ids(x, ids)
            ref.add_with_ids(x, ids)
        elif step % 3 == 1:
            sel = rng.choice(ref.ids, int(rng.integers(1, ref.ntotal // 4)), replace=False)
            remove_both(ix, ref, sel if step % 2 else torch.from_numpy(sel))
        else:
            a = int(rng.choice(ref.ids))
            remove_both(ix, ref, range(a, a + int(rng.integers(1, 3000))))
        assert_lists_equal(ix, ref, f"step {step}")
    ix.nprobe = 16
    q = near_queries(ref, 16, 5)
    assert_topk_equal(*ix.search(q, 10), *ref.search(q, 10, 16), "interleaved")


def test_block_shift_through_small_staging_chunks(oracle, monkeypatch):
    lens = np.array([33, 64, 5, 0, 97, 31, 160, 2, 65, 40], np.int64)
    off = np.concatenate([[0], np.cumsum(lens)])
    monkeypatch.setenv("DPH_UPLOAD_CHUNK_ROWS", "40")                         # one block per staging chunk
    ix, ref = synthetic_pair(oracle, lens)
    labels = np.arange(int(lens.sum()), dtype=np.int64)

    def assert_map_equal(what):                 # the direct map, compacted through many staging chunks: every label's row
        assert_lists_equal(ix, ref, what)
        v, f = ix.reconstruct_batch(labels)
        vr, fr = ref.reconstruct(labels)
        assert np.array_equal(f, fr) and np.array_equal(f.astype(bool), np.isin(labels, ref.ids)), what
        assert np.array_equal(v.view(np.int32), vr.view(np.int32)), what

    # no list loses a block: one row from lists whose block count stays (64 -> 63, 5 -> 4, 160 -> 159, 40 -> 39): no block moves
    assert remove_both(ix, ref, np.array([off[1] + 3, off[2] + 4, off[6], off[9] + 39])) == 4
    assert_map_equal("no block moves")
    # list 0 loses a block (33 -> 32): every later block moves down, one chunk at a time
    assert remove_both(ix, ref, np.array([0], np.int64)) == 1
    assert_map_equal("every block moves")
    assert remove_both(ix, ref, np.concatenate([ref.list_ids(4)[:50], ref.list_ids(8)[::3], ref.list_ids(1)])) > 50
    assert_map_equal("several lists lose blocks")
    ix.nprobe = 10
    q = near_queries(ref, 8, 2)
    assert_topk_equal(*ix.search(q, 10), *ref.search(q, 10, 10), "after block shifts")


def test_two_shards_remove_then_sync(oracle):
    import torch
    from densephrases_b200.ivfpq import merge_shards
    nlist, lens, A, Cm, pq, codes, ids, targets = ragged_model(oracle)
    off = np.concatenate([[0], np.cumsum(lens)])
    h = 20
    full = gpu_index(A, Cm, pq, lens, codes, ids)
    halves = [gpu_index(A, Cm, pq, lens, codes[off[a]:off[b]], ids[off[a]:off[b]], shard=(a, b)) for a, b in ((0, h), (h, nlist))]
    ref = RR.RemovableRefIndex(A, pq, lens, centroids=Cm, codes=codes, ids=ids)
    rng = np.random.default_rng(4)
    for sel in (rng.choice(ids, 700, replace=False), ids[off[h] + 5:off[h] + 40],       # the second touches only the second shard
                range(int(np.sort(ids)[100]), int(np.sort(ids)[900]))):
        before = halves[0].list_len()
        per = sum(g.remove_ids_per_list(sel) for g in halves)
        for g in halves:
            g.sync_list_len(before - per)
        full.remove_ids(sel)
        ref.remove_ids(sel)
    lf, cf, idf = full.lists()
    assert np.array_equal(lf, ref.list_len)
    parts = [g.lists() for g in halves]
    assert all(np.array_equal(p[0], lf) for p in parts) and all(g.ntotal == full.ntotal == ref.ntotal for g in halves)
    assert np.array_equal(np.concatenate([p[1] for p in parts]), ref.codes) and np.array_equal(np.concatenate([p[2] for p in parts]), ref.ids)
    with pytest.raises(RuntimeError):
        bad = ref.list_len.copy(); bad[3] += 1
        halves[0].sync_list_len(bad)                                             # an in-shard length that is not the shard's own
    for g in [full] + halves:
        g.nprobe = 16
    q = torch.from_numpy(near_queries(ref, 40, 8)).cuda()
    D, I = full.search(q, 10)
    res = [g.search_partial(q, 10) for g in halves]
    Dm, Im = merge_shards(*(torch.stack([r[i] for r in res]).contiguous() for i in range(3)), 10)
    assert torch.equal(Dm.view(torch.int32), D.view(torch.int32)) and torch.equal(Im, I)
    assert_topk_equal(D.cpu().numpy(), I.cpu().numpy(), *ref.search(q.cpu().numpy(), 10, 16), "shards after removes")


def test_temporary_memory_bound_on_a_large_index(oracle):
    nlist = 1024
    lens = np.full(nlist, 3_200_000 // nlist, np.int64)                       # 3.2 M rows: 307 MB of codes
    ix, ref = synthetic_pair(oracle, lens)
    ix.remove_ids(np.array([-1], np.int64))                                    # first remove: the labels become explicit
    ref.remove_ids(np.array([-1], np.int64))
    b0 = ix.device_bytes
    stage = 256 << 20
    for sel in (range(100_000, 250_000), np.random.default_rng(1).choice(3_200_000, 20_000, replace=False).astype(np.int64)):
        n = remove_both(ix, ref, sel)
        n_ids = len(sel) if isinstance(sel, np.ndarray) else 0
        assert ix.last_remove_tmp_bytes() <= stage + 64 * nlist + 32 * n_ids + 32 * n + 4096
        assert ix.device_bytes == b0
    assert_lists_equal(ix, ref, "large index")


def test_rejected_calls_leave_the_index_unchanged(oracle):
    from densephrases_b200 import _lib as L
    ix, ref = ragged_pair(oracle)
    L0, n0, b0 = ix.lists(), ix.ntotal, ix.device_bytes
    ids = np.ascontiguousarray(ref.ids[:10])
    p = ids.ctypes.data_as(C.c_void_p)
    n = C.c_int64(0)
    lib = L.lib()
    assert lib.dph_index_remove_ids(ix._h, p, 10, 5, 9, L.MEM_HOST, C.byref(n), None) != 0          # both selector forms
    assert lib.dph_index_remove_ids(ix._h, p, -1, 0, 0, L.MEM_HOST, C.byref(n), None) != 0          # n_ids < 0
    assert lib.dph_index_remove_ids(ix._h, None, 10, 0, 5, L.MEM_HOST, C.byref(n), None) != 0       # neither: a count, no labels
    for sel in (ids.astype(np.float64), ids.astype(np.int32), list(ids), range(0, 10, 2), 7):
        with pytest.raises((TypeError, ValueError)):
            ix.remove_ids(sel)
    assert ix.ntotal == n0 and ix.device_bytes == b0
    assert all(np.array_equal(a, b) for a, b in zip(L0, ix.lists()))
