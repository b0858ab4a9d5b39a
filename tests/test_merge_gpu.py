"""GPU: merging indexes (dph_index_merge_from) against the merge definition (tests/merge_ref.py, DESIGN.md 3.4).  After a merge the
device state equals set_lists of the concatenated list-major arrays: lists(), device_bytes(), search bits in every scan mode, and the
adds and removes that follow all match a twin built that way; the sources do not change; a rejected call changes nothing."""
import numpy as np
import pytest

from oracle import encode_ref as E
from tests.helpers import near_queries
from tests.merge_ref import np_merge
from tests.test_add_gpu import gpu_index, model, vectors_near

pytestmark = pytest.mark.gpu
ADD_ID = 1_000_000


def arrays(nlist, n, seed, labels, label0=0):
    """Ragged list-major arrays: about a third of the lists empty; labels None (sequential) or a permutation from label0."""
    rng = np.random.default_rng(seed)
    w = rng.random(nlist) * (rng.random(nlist) < 0.67)
    w[0] += 1e-3
    lens = rng.multinomial(n, w / w.sum()).astype(np.int64) if n else np.zeros(nlist, np.int64)
    codes = rng.integers(0, 256, (n, 96), dtype=np.uint8)
    ids = label0 + rng.permutation(n).astype(np.int64) * 3 if labels else None
    return lens, codes, ids


def assert_arrays_equal(got, want, what=""):
    lens, codes, ids = want
    assert np.array_equal(got[0], lens), what
    assert np.array_equal(got[1], codes), what
    assert np.array_equal(got[2], ids if ids is not None else np.arange(int(lens.sum()))), what


def case(oracle, nlist, labels, n_src, shard=None):
    """-> (model, dest arrays, source arrays, dest index, source indexes); labels: 'explicit' everywhere or 'seq' (sequential dest, one
    sequential source, the others explicit)."""
    A, Cm, pq = model(oracle, nlist)
    dest = arrays(nlist, 3000, 1, labels == "explicit", 5 * 10**6)
    sizes = [700, 0, 1500][:n_src] if n_src > 1 else [700]
    srcs = [arrays(nlist, n, 10 + s, labels == "explicit" or s > 0, 10**7 * (s + 1)) for s, n in enumerate(sizes)]
    mk = lambda a: gpu_index(A, Cm, pq, *a, shard=shard)
    return (A, Cm, pq), dest, srcs, mk(dest), [mk(s) for s in srcs]


@pytest.mark.parametrize("labels", ["seq", "explicit"])
@pytest.mark.parametrize("nlist", [1, 16, 512, 4096])
def test_merge_equals_set_lists_of_concatenation(oracle, nlist, labels):
    for n_src in (1, 3):
        (A, Cm, pq), dest, srcs, ix, six = case(oracle, nlist, labels, n_src)
        want = np_merge(dest, srcs, ADD_ID)
        ix.merge_from(six if n_src > 1 else six[0], add_id=ADD_ID)
        assert_arrays_equal(ix.lists(), want, f"n_src={n_src}")
        assert ix.ntotal == ix.ntotal_local == int(want[0].sum())
        twin = gpu_index(A, Cm, pq, *want)
        assert ix.device_bytes == twin.device_bytes
        for s, a in zip(six, srcs):                                      # the sources are not modified
            assert_arrays_equal(s.lists(), a, "source")


def test_search_bits_equal_twin_in_every_scan_mode(oracle):
    (A, Cm, pq), dest, srcs, ix, six = case(oracle, 512, "seq", 3)
    ix.merge_from(six, add_id=ADD_ID)
    want = np_merge(dest, srcs, ADD_ID)
    twin = gpu_index(A, Cm, pq, *want)
    ref = E.GrowableRefIndex(A, pq, want[0], centroids=Cm, codes=want[1], ids=want[2])
    q = near_queries(ref, 64, 3)
    for mode in (4, 2, 3):                                                  # quad, pair, single
        for g in (ix, twin):
            g.nprobe = 16
            g.set_scan_mode(mode)
        D, I = ix.search(q, 10)
        Dt, It = twin.search(q, 10)
        assert np.array_equal(D.view(np.int32), Dt.view(np.int32)) and np.array_equal(I, It), f"mode {mode}"
        assert (I >= 0).all()


def test_duplicated_label_reconstructs_the_latest_source(oracle):
    nlist = 16
    A, Cm, pq = model(oracle, nlist)
    dup = 424242
    parts = []
    for s in range(3):
        lens, codes, ids = arrays(nlist, 200, 30 + s, True, 10**6 * (s + 1))
        ids[[7, 150][s % 2]] = dup
        parts.append((lens, codes, ids))
    ix, a, b = (gpu_index(A, Cm, pq, *p) for p in parts)
    ix.merge_from([a, b])
    assert_arrays_equal(ix.lists(), np_merge(parts[0], parts[1:]))
    v, f = ix.reconstruct_batch(np.array([dup], np.int64))
    latest = E.GrowableRefIndex(A, pq, parts[2][0], centroids=Cm, codes=parts[2][1], ids=parts[2][2])
    vr, _ = latest.reconstruct(np.array([dup], np.int64))
    assert f.all() and np.array_equal(v.view(np.int32), vr.view(np.int32))
    ix.nprobe = nlist
    D, I = ix.search(vectors_near(A, Cm, [0], 1), 700)
    assert (I == dup).sum() == 3                                            # search finds every row carrying it


def test_add_and_remove_after_merge_match_twin(oracle):
    (A, Cm, pq), dest, srcs, ix, six = case(oracle, 64, "seq", 3)
    ix.merge_from(six, add_id=ADD_ID)
    want = np_merge(dest, srcs, ADD_ID)
    twin = gpu_index(A, Cm, pq, *want)
    x = vectors_near(A, Cm, np.random.default_rng(5).integers(0, 64, 500), 6)
    ids = 9 * 10**8 + np.arange(500)
    for g in (ix, twin):
        g.add_with_ids(x, ids)
    assert_arrays_equal(ix.lists(), twin.lists(), "add")
    sel = np.random.default_rng(7).choice(want[2], 900, replace=False)
    for g in (ix, twin):
        assert g.remove_ids(sel) == 900
        assert g.remove_ids(range(int(ids[100]), int(ids[300]))) == 200
    assert_arrays_equal(ix.lists(), twin.lists(), "remove")
    assert ix.device_bytes == twin.device_bytes


def test_empty_sources_are_a_no_op(oracle):
    (A, Cm, pq), dest, _, ix, _ = case(oracle, 16, "seq", 1)
    empty = gpu_index(A, Cm, pq, np.zeros(16, np.int64))
    L0, b0 = ix.lists(), ix.device_bytes
    ix.merge_from([empty, empty], add_id=-5)
    ix.merge_from([])
    assert ix.device_bytes == b0                                            # the labels stay sequential
    assert_arrays_equal(ix.lists(), L0)


def test_rejections_leave_the_index_unchanged(oracle):
    from densephrases_b200 import IvfPqIndex
    nlist = 16
    (A, Cm, pq), dest, srcs, ix, six = case(oracle, nlist, "explicit", 1)
    L0, n0, b0 = ix.lists(), ix.ntotal, ix.device_bytes
    bad = []
    for which in range(3):                                                  # one bit of one table differs
        t = [A.copy(), Cm.copy(), pq.copy()]
        t[which].reshape(-1).view(np.uint32)[37] ^= 1
        bad.append(gpu_index(*t, *srcs[0]))
    bad.append(gpu_index(*model(oracle, nlist + 1), np.zeros(nlist + 1, np.int64)))          # another nlist
    bad.append(gpu_index(A, Cm, pq, np.zeros(nlist, np.int64), shard=(0, 8)))                 # another shard range
    for b in bad:
        with pytest.raises(RuntimeError):
            ix.merge_from([six[0], b])
    with pytest.raises(RuntimeError, match="own source"):
        ix.merge_from([six[0], ix])
    with pytest.raises(RuntimeError, match="add_id"):
        ix.merge_from(six[0], add_id=2**63 - 10)                            # overflow
    with pytest.raises(RuntimeError, match="add_id"):
        ix.merge_from(six[0], add_id=-10**7 - 1)                            # the source's smallest label is 10^7
    seq = gpu_index(A, Cm, pq, arrays(nlist, 50, 3, False)[0], arrays(nlist, 50, 3, False)[1])
    with pytest.raises(RuntimeError, match="add_id"):
        ix.merge_from(seq, add_id=-1)                                       # sequential labels start at 0
    with pytest.raises(TypeError):
        ix.merge_from([six[0], "not an index"])
    unset = IvfPqIndex(nlist)
    with pytest.raises(RuntimeError):
        ix.merge_from(unset)
    assert ix.ntotal == n0 and ix.device_bytes == b0
    assert_arrays_equal(ix.lists(), L0)
    ix.merge_from(six[0], add_id=-10**7)                                    # the smallest label becomes 0: accepted
    assert ix.ntotal == n0 + 700


def test_two_shards_match_the_unsharded_merge(oracle):
    import torch
    from densephrases_b200.ivfpq import merge_shards
    nlist, h = 64, 27
    (A, Cm, pq), dest, srcs, full, sfull = case(oracle, nlist, "seq", 3)
    full.set_profile(True)
    full.merge_from(sfull, add_id=ADD_ID)
    assert len(full.last_merge_ms()) == 4 and (full.last_merge_ms() >= 0).all()
    off = lambda a: np.concatenate([[0], np.cumsum(a[0])])

    def part(a, lo, hi):
        o = off(a)
        codes = a[1][o[lo]:o[hi]]
        return a[0], codes, a[2][o[lo]:o[hi]] if a[2] is not None else None      # no labels: a shard's are the global list-major rows

    halves = []
    for lo, hi in ((0, h), (h, nlist)):
        ix = gpu_index(A, Cm, pq, *part(dest, lo, hi), shard=(lo, hi))
        ix.merge_from([gpu_index(A, Cm, pq, *part(s, lo, hi), shard=(lo, hi)) for s in srcs], add_id=ADD_ID)
        halves.append(ix)
    lf, cf, idf = full.lists()
    parts = [g.lists() for g in halves]
    assert all(np.array_equal(p[0], lf) for p in parts) and all(g.ntotal == full.ntotal for g in halves)
    assert np.array_equal(np.concatenate([p[1] for p in parts]), cf) and np.array_equal(np.concatenate([p[2] for p in parts]), idf)
    with pytest.raises(RuntimeError, match="shard range"):
        halves[0].merge_from(gpu_index(A, Cm, pq, *part(srcs[0], h, nlist), shard=(h, nlist)))
    for g in [full] + halves:
        g.nprobe = 16
    ref = E.GrowableRefIndex(A, pq, lf, centroids=Cm, codes=cf, ids=idf)
    q = torch.from_numpy(near_queries(ref, 40, 8)).cuda()
    D, I = full.search(q, 10)
    res = [g.search_partial(q, 10) for g in halves]
    Dm, Im = merge_shards(*(torch.stack([r[i] for r in res]).contiguous() for i in range(3)), 10)
    assert torch.equal(Dm.view(torch.int32), D.view(torch.int32)) and torch.equal(Im, I)
