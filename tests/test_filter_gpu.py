"""GPU: the filtered search (DESIGN.md 3.6) against the CPU oracle (oracle/filter_ref.c): D bits and I in every scan mode, nprobe, k and
selector form; the filter's mask against tests/filter_ref.py; selecting everything against the unfiltered search (G included); no side
effects; host mode and two shards against the device-resident unsharded index; and the filter's lifetime."""
import numpy as np
import pytest

from oracle import filter_ref as FR
from tests.filter_ref import np_mask
from tests.helpers import assert_topk_equal
from tests.host_codes_ref import blocks
from tests.test_add_gpu import gpu_index, model, vectors_near
from tests.test_host_codes_gpu import host_index, queries
from tests.test_merge_gpu import arrays

pytestmark = pytest.mark.gpu
FAST, EXACT, PAIR, SINGLE, QUAD = 0, 1, 2, 3, 4


def case(oracle, nlist, labels, n=20000, seed=3):
    """Ragged lists (about a third empty); labels sequential, or explicit with one label on two rows."""
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, n, seed, labels == "explicit")
    if ids is not None:
        ids[-1] = ids[0]
    ref = oracle.RefIndex(A, pq, lens, centroids=Cm, codes=codes, ids=ids)
    return (A, Cm, pq, lens, codes, ids), ref


def selectors(ref):
    """name -> (selector, exclude)."""
    lab = FR.labels(ref)
    rng = np.random.default_rng(7)
    s = np.sort(np.unique(lab))
    off = np.concatenate([[0], np.cumsum(ref.list_len)])
    whole = np.concatenate([lab[off[l]:off[l + 1]][(np.arange(ref.list_len[l]) // 32) % 2 == 0] for l in range(ref.nlist)]
                           + [np.zeros(0, np.int64)])
    out = {}
    for pct in (50, 10, 1):
        out[f"set{pct}"] = (rng.choice(lab, max(len(lab) * pct // 100, 1), replace=False), False)
    out["set1_dups_absent"] = (np.concatenate([out["set1"][0], out["set1"][0][:5], [-1, -9, 10**15]]), False)
    out["range"] = (range(int(s[len(s) // 3]), int(s[len(s) // 3 + len(s) // 5])), False)
    for name in ("set50", "set10", "set1", "range"):
        out[name + "_exclude"] = (out[name][0], True)
    out["whole_blocks"] = (whole, False)                                  # even blocks of every list: odd blocks empty
    out["nothing"] = (np.zeros(0, np.int64), False)
    out["nothing_range"] = (range(3, 3), False)
    out["few"] = (rng.choice(lab, 3, replace=False), False)             # fewer than k selected rows probed
    out["everything"] = (np.zeros(0, np.int64), True)
    return out


def assert_mask(f, ref, selected, lo=0, hi=None):
    want = np_mask(ref.list_len, selected, lo, hi)
    assert np.array_equal(f.mask(), want)
    assert f.rows == int(np.unpackbits(want.view(np.uint8)).sum()) and f.nbytes == 4 * len(want)


@pytest.mark.parametrize("labels", ["seq", "explicit"])
@pytest.mark.parametrize("nlist", [1, 64, 4096])
def test_filtered_search_equals_the_oracle(oracle, nlist, labels):
    arrs, ref = case(oracle, nlist, labels)
    A, Cm, pq, lens, codes, ids = arrs
    ix = gpu_index(A, Cm, pq, lens, codes, ids)
    q = queries(A, Cm, lens, 40, nlist)
    for name, (sel, exclude) in selectors(ref).items():
        selected = FR.selected_rows(ref, sel, exclude)
        f = ix.make_filter(sel, exclude=exclude)
        assert_mask(f, ref, selected)
        for nprobe in sorted({1, min(32, nlist), min(nlist, 1024)}):          # every list, up to the nprobe limit
            ix.nprobe = nprobe
            for k in (1, 10, 100, 1024):
                Dr, Ir, _ = FR.search(ref, q, k, nprobe, selected)
                for mode in (FAST, QUAD, PAIR, SINGLE, EXACT):
                    ix.set_scan_mode(mode)
                    D, I = ix.search(q, k, filter=f)
                    assert_topk_equal(D, I, Dr, Ir, f"{name} nprobe={nprobe} k={k} mode={mode}")
    ix.set_scan_mode(FAST)


@pytest.mark.parametrize("labels", ["seq", "explicit"])
def test_everything_selected_equals_unfiltered_and_filters_change_nothing(oracle, labels):
    import torch
    arrs, ref = case(oracle, 512, labels, n=60000)
    A, Cm, pq, lens, codes, ids = arrs
    ix = gpu_index(A, Cm, pq, lens, codes, ids)
    lists0, bytes0 = ix.lists(), ix.device_bytes
    xt = torch.from_numpy(queries(A, Cm, lens, 64, 1)).cuda()
    everything = ix.make_filter(np.zeros(0, np.int64), exclude=True)
    assert everything.rows == ix.ntotal
    some = ix.make_filter(FR.labels(ref)[::7])
    for a, b in zip(ix.lists(), lists0):                  # building filters changes nothing; sequential labels stay sequential
        assert np.array_equal(a, b)
    assert ix.device_bytes == bytes0
    for nprobe in (8, 256):
        ix.nprobe = nprobe
        for mode in (FAST, QUAD, PAIR, SINGLE, EXACT):
            ix.set_scan_mode(mode)
            for k in (10, 100):
                before = [t.cpu().numpy() for t in ix.search_partial(xt, k)]
                with_all = [t.cpu().numpy() for t in ix.search_partial(xt, k, filter=everything)]
                ix.search_partial(xt, k, filter=some)
                after = [t.cpu().numpy() for t in ix.search_partial(xt, k)]
                for a, b, c in zip(before, with_all, after):
                    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"nprobe={nprobe} mode={mode} k={k}"
                    assert np.array_equal(a.view(np.uint8), c.view(np.uint8)), f"nprobe={nprobe} mode={mode} k={k}"
    for a, b in zip(ix.lists(), lists0):
        assert np.array_equal(a, b)
    assert ix.device_bytes == bytes0


@pytest.mark.parametrize("resident", ["none", "some"])
def test_host_mode_equals_the_resident_twin(oracle, resident):
    nlist = 256
    arrs, ref = case(oracle, nlist, "explicit", n=40000, seed=5)
    A, Cm, pq, lens, codes, ids = arrs
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    ix = host_index(A, Cm, pq, lens, codes, ids, (int(blocks(lens).max()) + 3) * 3072)
    if resident == "some":
        ix.set_resident_lists(np.arange(0, nlist, 3))
    q = queries(A, Cm, lens, 48, 2)
    for name, (sel, exclude) in selectors(ref).items():
        ft, fh = twin.make_filter(sel, exclude=exclude), ix.make_filter(sel, exclude=exclude)
        assert np.array_equal(ft.mask(), fh.mask())
        for nprobe in (16, 256):
            twin.nprobe = ix.nprobe = nprobe
            for mode in (FAST, QUAD, SINGLE, EXACT):
                twin.set_scan_mode(mode); ix.set_scan_mode(mode)
                D, I = ix.search(q, 10, filter=fh)
                Dt, It = twin.search(q, 10, filter=ft)
                assert np.array_equal(D.view(np.int32), Dt.view(np.int32)) and np.array_equal(I, It), f"{name} nprobe={nprobe} mode={mode}"
                assert ix.last_fetch()["slices"] > (1 if nprobe == 256 else 0)


def test_two_shards_equal_the_unsharded_index(oracle):
    import torch
    from densephrases_b200 import merge_shards
    from densephrases_b200.sharded import ShardedIvfPq, shard_ranges
    nlist, nprobe = 96, 24
    arrs, ref = case(oracle, nlist, "explicit", n=30000, seed=9)
    A, Cm, pq, lens, codes, ids = arrs
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    twin.nprobe = nprobe
    off = np.concatenate([[0], np.cumsum(lens)])
    shards = []
    for lo, hi in shard_ranges(lens, 2):
        sh = gpu_index(A, Cm, pq, lens, codes[off[lo]:off[hi]], ids[off[lo]:off[hi]], shard=(lo, hi))
        sh.nprobe = nprobe
        shards.append((sh, lo, hi))
    q = queries(A, Cm, lens, 40, 9)
    xt = torch.from_numpy(q).cuda()
    per = (len(q) + 1) // 2
    for name, (sel, exclude) in selectors(ref).items():
        selected = FR.selected_rows(ref, sel, exclude)
        fs = [sh.make_filter(sel, exclude=exclude) for sh, _, _ in shards]
        for f, (_, lo, hi) in zip(fs, shards):
            assert_mask(f, ref, selected, lo, hi)
        for k in (10, 100):
            Dw, Iw = twin.search(q, k, filter=twin.make_filter(sel, exclude=exclude))
            keys_g = torch.stack([sh.coarse_local(xt) for sh, _, _ in shards]).contiguous()
            parts = [sh.search_preassigned(keys_g, k, filter=f) for (sh, _, _), f in zip(shards, fs)]
            rec = torch.cat([sh.coarse_split(xt[r * per:(r + 1) * per].contiguous()) for r, (sh, _, _) in enumerate(shards)]).contiguous()
            parts2 = [sh.search_assigned(rec, k, filter=f) for (sh, _, _), f in zip(shards, fs)]
            for ps in (parts, parts2):
                D, I = merge_shards(*(torch.stack([p[i] for p in ps]).contiguous() for i in range(3)), k)
                D, I = D.cpu().numpy(), I.cpu().numpy()
                assert np.array_equal(D.view(np.int32), Dw.view(np.int32)) and np.array_equal(I, Iw), f"{name} k={k}"
    # ShardedIvfPq with one rank: the same filter through its own keywords
    s1 = ShardedIvfPq.from_arrays(A, Cm, pq, lens, codes, ids)
    s1.nprobe = nprobe
    sel = FR.labels(ref)[::5]
    f1 = s1.make_filter(sel)
    Dw, Iw = twin.search(q, 10, filter=twin.make_filter(sel))
    for D, I in (s1.search(q, 10, filter=f1), [t.cpu().numpy() for t in s1.search_device(xt, 10, filter=f1)]):
        assert np.array_equal(D.view(np.int32), Dw.view(np.int32)) and np.array_equal(I, Iw)


def test_a_stale_or_foreign_filter_is_rejected(oracle):
    arrs, _ = case(oracle, 64, "explicit", n=8000, seed=4)
    A, Cm, pq, lens, codes, ids = arrs
    ix = gpu_index(A, Cm, pq, lens, codes, ids)
    other = gpu_index(A, Cm, pq, lens, codes, ids)
    ix.nprobe = other.nprobe = 16
    q = queries(A, Cm, lens, 16, 4)
    sel = np.asarray(ids[::4])

    def state(g):
        return [a.copy() for a in g.lists()] + [g.device_bytes]

    def same(a, b):
        return all(np.array_equal(x, y) for x, y in zip(a, b))

    with pytest.raises(RuntimeError, match="another index"):
        ix.search(q, 10, filter=other.make_filter(sel))
    rng = np.random.default_rng(0)
    steps = [
        ("add", lambda g: g.add_with_ids(vectors_near(A, Cm, rng.integers(0, 64, 300), 1), 10**9 + np.arange(300, dtype=np.int64))),
        ("remove", lambda g: g.remove_ids(np.asarray(ids[1::9]))),
        ("merge", lambda g: g.merge_from(gpu_index(A, Cm, pq, lens, codes, ids), add_id=5 * 10**8)),
        ("set_lists", lambda g: g.set_lists(lens, codes, ids)),
    ]
    for name, step in steps:
        f = ix.make_filter(sel)
        ix.search(q, 10, filter=f)
        step(ix)
        before = state(ix)
        with pytest.raises(RuntimeError, match="rebuild the filter"):
            ix.search(q, 10, filter=f)
        assert same(state(ix), before), name
        D0, I0 = ix.search(q, 10)                          # the stale filter was cleared from the handle
        lens2, codes2, ids2 = ix.lists()
        ref = oracle.RefIndex(A, pq, lens2, centroids=Cm, codes=codes2, ids=ids2)
        f2 = ix.make_filter(sel)
        D, I = ix.search(q, 10, filter=f2)
        Dr, Ir, _ = FR.search(ref, q, 10, 16, FR.selected_rows(ref, sel))
        assert_topk_equal(D, I, Dr, Ir, name)
        Du, Iu = ref.search(q, 10, 16)
        assert_topk_equal(D0, I0, Du, Iu, name)
    # set_resident_lists / stream_bytes do not change the layout: a host index's filter survives them
    hx = host_index(A, Cm, pq, lens, codes, ids, None)
    hx.nprobe = 16
    hf = hx.make_filter(sel)
    want = hx.search(q, 10, filter=hf)
    hx.set_resident_lists([0, 5, 9])
    hx.set_code_residency(True, 2 << 20)
    got = hx.search(q, 10, filter=hf)
    assert np.array_equal(got[0].view(np.int32), want[0].view(np.int32)) and np.array_equal(got[1], want[1])
