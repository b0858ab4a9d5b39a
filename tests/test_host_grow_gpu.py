"""GPU: mutable host indexes (DESIGN.md 3.5, "Mutable host indexes").  A host-mode index with a reserved host capacity is grown,
shrunk and merged in place, and after every step equals a device-resident twin that took the same calls: lists() byte for byte and
search bits (D and I) in every scan mode, nprobe and k; the twin is checked against the oracles.  The in-place mover runs through many
staging chunks, at the first and the last list; the capacity, the resident set and the rejected calls keep their contracts; the
sharded handle forwards it all with world 1."""
import numpy as np
import pytest

from oracle import remove_ref as RR
from tests.merge_ref import np_merge
from tests.test_add_gpu import assert_lists_equal, gpu_index, model, vectors_near
from tests.test_host_codes_gpu import EXACT, PAIR, QUAD, SINGLE, assert_bits
from tests.test_host_grow_cpu import first_changed_block, layout
from tests.test_merge_gpu import arrays

pytestmark = pytest.mark.gpu
MB = 1 << 20
ADD_ID = 3 * 10**8


def host_index(A, Cm, pq, lens, codes=None, ids=None, capacity=64 * MB, stream_bytes=64 * MB, shard=None):
    from densephrases_b200 import IvfPqIndex
    return IvfPqIndex.from_arrays(A, Cm, pq, lens, np.zeros((0, 96), np.uint8) if codes is None else codes, ids, shard=shard,
                                  codes_on_host=True, stream_bytes=stream_bytes, host_capacity_bytes=capacity)


def assert_same_lists(ix, twin, what=""):
    for a, b in zip(ix.lists(), twin.lists()):
        assert np.array_equal(a, b), what
    assert ix.ntotal == twin.ntotal and ix.ntotal_local == twin.ntotal_local, what


def assert_same_search(ix, twin, q, nprobes, what=""):
    for nprobe in nprobes:
        for mode in (QUAD, PAIR, SINGLE, EXACT):
            for g in (ix, twin):
                g.nprobe = nprobe
                g.set_scan_mode(mode)
            for k in (1, 10, 100):
                assert_bits(ix.search(q, k), twin.search(q, k), f"{what} nprobe={nprobe} mode={mode} k={k}")


def state(g, q):
    g.nprobe = 8
    g.set_scan_mode(QUAD)
    return [a.copy() for a in g.lists()], g.ntotal, g.device_bytes, g.host_bytes, g.search(q, 10)


def assert_unchanged(before, g, q, what=""):
    after = state(g, q)
    assert all(np.array_equal(a, b) for a, b in zip(before[0], after[0])), what
    assert before[1:4] == after[1:4], what
    assert_bits(after[4], before[4], what)


@pytest.mark.parametrize("nlist", [64, 512])
def test_adds_removes_and_a_merge_equal_the_device_twin(oracle, nlist):
    import torch
    A, Cm, pq = model(oracle, nlist)
    rng = np.random.default_rng(nlist)
    ix = host_index(A, Cm, pq, np.zeros(nlist, np.int64))
    twin = gpu_index(A, Cm, pq, np.zeros(nlist, np.int64))
    ref = RR.RemovableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    host0 = ix.host_bytes
    assert host0 == 64 * MB // 3072 * 3072
    q = vectors_near(A, Cm, rng.integers(0, nlist, 24), 1, noise=0.3)
    nprobes = (1, 32, nlist)

    def step(what, call, on_ref=None):
        for g in (ix, twin):
            call(g)
        if on_ref is not None:
            on_ref(ref)
        assert_same_lists(ix, twin, what)
        assert_same_search(ix, twin, q, nprobes, what)
        assert ix.host_bytes == host0, what                       # within the capacity nothing is reallocated

    x1 = vectors_near(A, Cm, rng.integers(0, nlist, 900), 2, noise=0.3)
    x2 = vectors_near(A, Cm, rng.integers(0, nlist, 700), 3, noise=0.3)
    x3 = vectors_near(A, Cm, rng.integers(0, nlist, 800), 4, noise=0.3)
    x4 = vectors_near(A, Cm, rng.integers(0, nlist, 600), 5, noise=0.3)
    ids3 = 10**9 + rng.permutation(800).astype(np.int64)
    ids4 = 2 * 10**9 + rng.permutation(600).astype(np.int64)
    step("add host implicit", lambda g: g.add(x1), lambda r: r.add_with_ids(x1))
    step("add device implicit", lambda g: g.add(torch.from_numpy(x2).cuda()), lambda r: r.add_with_ids(x2))
    step("add host explicit", lambda g: g.add_with_ids(x3, ids3), lambda r: r.add_with_ids(x3, ids3))
    step("add device explicit", lambda g: g.add_with_ids(torch.from_numpy(x4).cuda(), torch.from_numpy(ids4).cuda()),
         lambda r: r.add_with_ids(x4, ids4))
    assert_lists_equal(twin, ref, "the twin against the add oracle")
    sel = rng.choice(twin.lists()[2], 300, replace=False)
    sel = np.concatenate([sel, sel[:10], [-1, 7 * 10**9]])
    step("remove label set", lambda g: g.remove_ids(sel), lambda r: r.remove_ids(sel))
    step("remove range", lambda g: g.remove_ids(range(10**9 + 100, 10**9 + 500)), lambda r: r.remove_ids(range(10**9 + 100, 10**9 + 500)))
    assert_lists_equal(twin, ref, "the twin against the remove oracle")
    srcs = [arrays(nlist, 1500, 10, True, 10**7), arrays(nlist, 900, 11, False)]
    six = [gpu_index(A, Cm, pq, *a) for a in srcs]
    before = twin.lists()
    step("merge two device sources", lambda g: g.merge_from(six, add_id=ADD_ID))
    want = np_merge(before, srcs, ADD_ID)
    for a, b in zip(twin.lists(), want):
        assert np.array_equal(a, b), "the twin against the merge definition"
    x5 = vectors_near(A, Cm, rng.integers(0, nlist, 500), 6, noise=0.3)
    step("add after the merge", lambda g: g.add(x5))
    mv = ix.last_host_move()
    assert mv["blocks_written"] > 0 and mv["chunks"] >= 1


@pytest.mark.parametrize("chunk_rows", ["32", "100"])            # staging chunks of 1 and 3 blocks
def test_mover_through_many_chunks_at_the_first_and_the_last_list(oracle, monkeypatch, chunk_rows):
    monkeypatch.setenv("DPH_UPLOAD_CHUNK_ROWS", chunk_rows)
    cb = max(1, int(chunk_rows) * 96 // 3072)
    nlist = 32
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 4000, 21, True)
    lens[0] = max(lens[0], 70)
    lens[-1] = 0
    codes, ids = np.random.default_rng(3).integers(0, 256, (int(lens.sum()), 96), dtype=np.uint8), np.arange(int(lens.sum())) * 5
    ix = host_index(A, Cm, pq, lens, codes, ids, capacity=4 * MB)
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    q = vectors_near(A, Cm, np.random.default_rng(4).integers(0, nlist, 16), 1, noise=0.3)
    for what, target, n in (("first list", 0, 100), ("last list", nlist - 1, 45), ("first list again", 0, 1)):
        x = vectors_near(A, Cm, [target] * n, 7 + n)
        old = twin.list_len()
        for g in (ix, twin):
            g.add_with_ids(x, 10**8 + n + np.arange(n))
        new = twin.list_len()
        mv = ix.last_host_move()
        d_first, nb = first_changed_block(old, new), layout(new)[1]
        assert mv["blocks_written"] == nb - d_first and mv["chunks"] == -(-(nb - d_first) // cb), what
        if target == 0 and new[0] - old[0] >= 32:
            assert d_first == old[0] // 32 and mv["chunks"] > 10, what    # from list 0's old tail block on, everything moves
        if target == nlist - 1:
            assert d_first >= layout(old)[0][-1], what                  # nothing before the last list moves
        assert_same_lists(ix, twin, what)
        assert_same_search(ix, twin, q, (4, nlist), what)
    for sel in (ids[:300:3].copy(), range(10**8, 10**8 + 150)):        # the block shift, ascending, through the same chunks
        for g in (ix, twin):
            g.remove_ids(sel)
        assert_same_lists(ix, twin, f"remove {type(sel).__name__}")
        assert ix.last_host_move()["chunks"] > 1
    assert_same_search(ix, twin, q, (4, nlist), "after the removes")


def test_capacity_bounds_adds_and_reserve_grows_it(oracle):
    nlist = 16
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 3000, 2, True)
    nb = layout(lens)[1]
    ix = host_index(A, Cm, pq, lens, codes, ids, capacity=(nb + 4) * 3072 + 100)     # rounded down to whole blocks
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    assert ix.host_bytes == (nb + 4) * 3072
    q = vectors_near(A, Cm, np.random.default_rng(1).integers(0, nlist, 16), 2, noise=0.3)
    x = vectors_near(A, Cm, np.random.default_rng(2).integers(0, nlist, 400), 3)
    s = state(ix, q)
    with pytest.raises(RuntimeError, match="bytes of host codes; the reserved host capacity is"):
        ix.add_with_ids(x, 10**8 + np.arange(400))
    assert_unchanged(s, ix, q, "an add past the capacity")
    ix.reserve_host_codes(nb * 3072)                                  # at or below the allocation: nothing changes
    assert ix.host_bytes == (nb + 4) * 3072
    ix.reserve_host_codes(64 * MB)                                    # the growth copy
    assert ix.host_bytes == 64 * MB // 3072 * 3072
    assert_same_lists(ix, twin, "after the growth copy")
    for g in (ix, twin):
        g.add_with_ids(x, 10**8 + np.arange(400))
        g.remove_ids(ids[:500].copy())
    assert ix.host_bytes == 64 * MB // 3072 * 3072
    assert_same_lists(ix, twin, "add + remove after the reservation")
    assert_same_search(ix, twin, q, (4, nlist), "add + remove after the reservation")
    # reserved after set_lists without a capacity: the index becomes mutable, the array stays as it is until a larger capacity
    from densephrases_b200 import IvfPqIndex
    ro = IvfPqIndex.from_arrays(A, Cm, pq, lens, codes, ids, codes_on_host=True, stream_bytes=16 * MB)
    ro.reserve_host_codes(0)
    assert ro.host_bytes == nb * 3072
    t2 = gpu_index(A, Cm, pq, lens, codes, ids)
    for g in (ro, t2):
        g.remove_ids(range(0, 3000))
    assert ro.host_bytes == nb * 3072
    assert_same_lists(ro, t2, "remove after reserve_host_codes(0)")
    # a capacity smaller than the lists before set_lists: set_lists allocates what they need
    small = host_index(A, Cm, pq, lens, codes, ids, capacity=3072)
    assert small.host_bytes == nb * 3072


def test_resident_set_empties_on_a_mutation(oracle):
    nlist = 16
    A, Cm, pq = model(oracle, nlist)
    rng = np.random.default_rng(9)
    lens = rng.integers(10, 60, nlist).astype(np.int64)
    lens[3] = 90                                                      # 3 blocks; every other list <= 2
    lens[7] = 20
    codes = rng.integers(0, 256, (int(lens.sum()), 96), dtype=np.uint8)
    ids = 1000 + np.arange(int(lens.sum()))
    ix = host_index(A, Cm, pq, lens, codes, ids, capacity=8 * MB, stream_bytes=2 * 3072)
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    q = vectors_near(A, Cm, rng.integers(0, nlist, 16), 2, noise=0.3)
    ix.set_resident_lists([3])                                        # region: 3 resident + 2 stream blocks
    assert_same_search(ix, twin, q, (nlist,), "resident list 3")
    assert ix.last_fetch()["resident_lists_scanned"] > 0
    x = vectors_near(A, Cm, [7] * 20, 3)
    for g in (ix, twin):
        g.add_with_ids(x, 10**7 + np.arange(20))
    assert twin.list_len()[7] <= 64
    assert_same_search(ix, twin, q, (nlist,), "after a small add")      # list 3 (3 blocks) now streams: the 5-block region is kept
    assert ix.last_fetch()["resident_lists_scanned"] == 0
    big = vectors_near(A, Cm, [5] * 200, 4)
    for g in (ix, twin):
        g.add_with_ids(big, 2 * 10**7 + np.arange(200))
    assert twin.list_len()[5] > 5 * 32
    with pytest.raises(RuntimeError, match="stream region"):
        ix.search(q, 10)
    ix.set_resident_lists([3, 5])
    assert_same_search(ix, twin, q, (1, nlist), "list 5 resident")
    assert_same_lists(ix, twin)


def test_rejections_leave_a_mutable_host_index_unchanged(oracle):
    nlist = 16
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 3000, 5, True)
    ix = host_index(A, Cm, pq, lens, codes, ids)
    q = vectors_near(A, Cm, np.random.default_rng(1).integers(0, nlist, 16), 2, noise=0.3)
    x = vectors_near(A, Cm, [1, 2, 3], 0)
    bad = x.copy()
    bad[1, 5] = np.nan
    other_pq = pq.copy()
    other_pq[3, 7, 1] = np.nextafter(other_pq[3, 7, 1], np.float32(2))
    differing = gpu_index(A, Cm, other_pq, lens, codes, ids + 10**6)
    host_src = host_index(A, Cm, pq, lens, codes, ids + 10**6)
    s = state(ix, q)
    for what, call, match in (("negative label", lambda: ix.add_with_ids(x, np.array([7, -3, 9])), "negative label"),
                              ("non-finite input", lambda: ix.add_with_ids(bad, np.array([7, 8, 9])), "non-finite"),
                              ("differing tables", lambda: ix.merge_from(differing), "PQ codebooks"),
                              ("host-mode source", lambda: ix.merge_from(host_src), "host memory")):
        with pytest.raises(RuntimeError, match=match):
            call()
        assert_unchanged(s, ix, q, what)


def test_sharded_world_one_host_mode_add_then_remove(oracle):
    import torch
    from densephrases_b200.sharded import ShardedIvfPq
    nlist = 64
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 5000, 8, True)
    sh = ShardedIvfPq.from_arrays(A, Cm, pq, lens, codes, ids, codes_on_host=True, stream_bytes=32 * MB, host_capacity_bytes=32 * MB)
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    assert sh.local.host_bytes == 32 * MB // 3072 * 3072
    x = vectors_near(A, Cm, np.random.default_rng(2).integers(0, nlist, 1000), 3, noise=0.3)
    for g in (sh, twin):
        g.add_with_ids(x, 10**8 + np.arange(1000))
    assert sh.remove_ids(ids[::7].copy()) == twin.remove_ids(ids[::7].copy())
    assert sh.remove_ids(range(10**8, 10**8 + 300)) == twin.remove_ids(range(10**8, 10**8 + 300)) == 300
    assert_same_lists(sh.local, twin, "sharded world 1")
    q = vectors_near(A, Cm, np.random.default_rng(4).integers(0, nlist, 32), 5, noise=0.3)
    for g in (sh, twin):
        g.nprobe = 16
    assert_bits(sh.search(q, 10), twin.search(q, 10))
    D, I = sh.search_device(torch.from_numpy(q).cuda(), 10)
    assert_bits((D.cpu().numpy(), I.cpu().numpy()), twin.search(q, 10))
