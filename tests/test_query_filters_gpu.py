"""GPU: per-query filters (DESIGN.md 3.7).  The device-built CSR of every selector against make_filter's mask; a batch with per-query
filters against each row searched alone with its make_filter and against the oracle (D bits and I) over nprobe, k, flagged queries, -1
rows, shared selectors, chunked batches, host and device buffers and host mode; the other search paths and two shards; the rejections;
MIPS per-question document filters."""
import numpy as np
import pytest

from oracle import filter_ref as FR
from tests.helpers import assert_topk_equal
from tests.host_codes_ref import blocks
from tests.query_filter_ref import csr_mask, np_csr, query_filtered_search
from tests.test_add_gpu import gpu_index, model
from tests.test_filter_gpu import case
from tests.test_host_codes_gpu import host_index, queries
from tests.test_merge_gpu import arrays

pytestmark = pytest.mark.gpu
FAST, EXACT, PAIR, SINGLE, QUAD = 0, 1, 2, 3, 4


def sel_list(ref, rng):
    """Selectors of every form: label sets (small, with duplicates, absent and negative labels), ranges (empty, lo >= hi, crossing
    lists), nothing."""
    lab = FR.labels(ref)
    s = np.sort(np.unique(lab))
    few = rng.choice(lab, max(len(lab) // 200, 2), replace=False)
    return [few,
            np.concatenate([rng.choice(lab, len(lab) // 20, replace=False), few[:3], few[:3], [-1, -5, 10**15]]),
            range(int(s[len(s) // 3]), int(s[len(s) // 3 + len(s) // 50])),          # crosses lists
            rng.choice(lab, 7, replace=False),
            np.zeros(0, np.int64), range(3, 3), range(9, 2),
            np.array([lab[0], lab[-1]]),                                           # explicit case: lab[-1] == lab[0], a label on two rows
            rng.choice(lab, len(lab) // 100, replace=False)]


def assert_csr(qf, ix, ref, sels, lo=0, hi=None):
    for i, sel in enumerate(sels):
        selected = FR.selected_rows(ref, sel)
        off, blk, word = qf.csr(i)
        want = np_csr(ref.list_len, selected, lo, hi)
        assert all(np.array_equal(a, b) for a, b in zip((off, blk, word), want)), i
        mask = ix.make_filter(sel).mask()
        assert np.array_equal(csr_mask(ref.list_len, off, blk, word, lo, hi), mask), i
        assert qf.rows(i) == int(np.unpackbits(mask.view(np.uint8)).sum()), i


@pytest.mark.parametrize("labels", ["seq", "explicit"])
def test_csr_equals_make_filter_mask(oracle, labels):
    import torch
    arrs, ref = case(oracle, 256, labels, n=30000, seed=11)
    ix = gpu_index(*arrs)
    sels = sel_list(ref, np.random.default_rng(2))
    qf = ix.make_query_filters(sels, assign=np.arange(len(sels)))
    assert_csr(qf, ix, ref, sels)
    nl = ix.nlist
    assert qf.nbytes == sum(len(qf.csr(i)[1]) for i in range(len(sels))) * 8 + len(sels) * (nl + 1) * 4 + (len(sels) + 1) * 8 + 4 * len(sels)
    dev = [torch.from_numpy(s).cuda() if isinstance(s, np.ndarray) else s for s in sels]    # device labels
    assert_csr(ix.make_query_filters(dev), ix, ref, sels)


def check_batch(ix, ref, q, sels, selected, assign, k, what, x=None):
    """A per-query filtered batch == each row alone with its make_filter == the oracle."""
    qf = ix.make_query_filters(sels, assign)
    D, I = ix.search(q if x is None else x, k, filter=qf)
    if x is not None:
        D, I = D.cpu().numpy(), I.cpu().numpy()
    Dr, Ir = query_filtered_search(ref, q, k, ix.nprobe, selected, assign)
    assert_topk_equal(D, I, Dr, Ir, what)
    return D, I


@pytest.mark.parametrize("labels", ["seq", "explicit"])
def test_batch_equals_rows_alone_and_the_oracle(oracle, labels):
    import torch
    nlist = 512
    arrs, ref = case(oracle, nlist, labels, n=60000, seed=12)
    ix = gpu_index(*arrs)
    rng = np.random.default_rng(3)
    sels = sel_list(ref, rng)
    selected = [FR.selected_rows(ref, s) for s in sels]
    q = queries(arrs[0], arrs[1], arrs[3], 40, 12)
    assign = rng.integers(-1, len(sels), len(q))
    assign[:len(sels)] = np.arange(len(sels))                 # every selector, some shared, some -1 rows
    xt = torch.from_numpy(q).cuda()
    for nprobe in (1, 16, 256):
        ix.nprobe = nprobe
        for k in (1, 10, 100, 1024):
            for mode in (FAST, QUAD, EXACT):
                ix.set_scan_mode(mode)
                what = f"nprobe={nprobe} k={k} mode={mode}"
                D, I = check_batch(ix, ref, q, sels, selected, assign, k, what)
                if k == 10 and mode == FAST:
                    check_batch(ix, ref, q, sels, selected, assign, k, what + " device", x=xt)
                    for i in range(0, len(q), 7):     # row alone with its make_filter
                        f = None if assign[i] < 0 else ix.make_filter(sels[assign[i]])
                        Di, Ii = ix.search(q[i:i + 1], k, filter=f)
                        assert np.array_equal(Di.view(np.int32), D[i:i + 1].view(np.int32)) and np.array_equal(Ii, I[i:i + 1]), what
    ix.set_scan_mode(FAST)


def test_flagged_queries_take_the_exact_rerun(oracle):
    """Every row has the same code: equal scores in a list, so a query whose selection leaves more than keep of them in the scan has
    a dropped threshold equal to its k-th score, the proof fails and the exact pass re-runs it."""
    nlist = 32
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 20000, 14, True)
    codes[:] = codes[0]
    ref = oracle.RefIndex(A, pq, lens, centroids=Cm, codes=codes, ids=ids)
    ix = gpu_index(A, Cm, pq, lens, codes, ids)
    ix.nprobe = 4
    rng = np.random.default_rng(14)
    sels = [rng.choice(ids, len(ids) // 2, replace=False), rng.choice(ids, 20, replace=False)]
    selected = [FR.selected_rows(ref, s) for s in sels]
    q = queries(A, Cm, lens, 12, 14)
    assign = np.arange(12) % 3 - 1
    check_batch(ix, ref, q, sels, selected, assign, 10, "flagged")
    flags = ix.last_flags(len(q))
    assert flags[assign == 0].any()


def test_chunked_batch(oracle):
    # nlist 65536: the coarse-score bound cuts the batch into chunks of 4096 queries
    nlist = 65536
    arrs, ref = case(oracle, nlist, "explicit", n=200000, seed=13)
    ix = gpu_index(*arrs)
    ix.nprobe = 8
    rng = np.random.default_rng(4)
    sels = sel_list(ref, rng)[:4]
    selected = [FR.selected_rows(ref, s) for s in sels]
    q = queries(arrs[0], arrs[1], arrs[3], 4200, 13)
    assign = rng.integers(-1, len(sels), len(q))
    qf = ix.make_query_filters(sels, assign)
    D, I = ix.search(q, 10, filter=qf)
    pick = np.concatenate([np.arange(0, 20), np.arange(4090, 4110), np.arange(4180, 4200)])
    Dr, Ir = query_filtered_search(ref, q[pick], 10, 8, selected, assign[pick])
    assert_topk_equal(D[pick], I[pick], Dr, Ir, "chunked")


@pytest.mark.parametrize("resident", ["none", "some"])
def test_host_mode(oracle, resident):
    nlist = 256
    arrs, ref = case(oracle, nlist, "explicit", n=40000, seed=5)
    A, Cm, pq, lens, codes, ids = arrs
    twin = gpu_index(*arrs)
    ix = host_index(A, Cm, pq, lens, codes, ids, (int(blocks(lens).max()) + 3) * 3072)
    if resident == "some":
        ix.set_resident_lists(np.arange(0, nlist, 3))
    rng = np.random.default_rng(5)
    sels = sel_list(ref, rng)
    selected = [FR.selected_rows(ref, s) for s in sels]
    q = queries(A, Cm, lens, 48, 2)
    assign = rng.integers(-1, len(sels), len(q))
    for nprobe in (16, 256):
        twin.nprobe = ix.nprobe = nprobe
        D, I = ix.search(q, 10, filter=ix.make_query_filters(sels, assign))
        Dt, It = twin.search(q, 10, filter=twin.make_query_filters(sels, assign))
        assert np.array_equal(D.view(np.int32), Dt.view(np.int32)) and np.array_equal(I, It), nprobe
        Dr, Ir = query_filtered_search(ref, q, 10, nprobe, selected, assign)
        assert_topk_equal(D, I, Dr, Ir, f"host nprobe={nprobe}")
        assert ix.last_fetch()["slices"] > (1 if nprobe == 256 else 0)


def test_other_paths_and_two_shards(oracle):
    import torch
    from densephrases_b200 import merge_shards
    from densephrases_b200.sharded import shard_ranges
    nlist, nprobe = 96, 24
    arrs, ref = case(oracle, nlist, "explicit", n=30000, seed=9)
    A, Cm, pq, lens, codes, ids = arrs
    twin = gpu_index(*arrs)
    twin.nprobe = nprobe
    rng = np.random.default_rng(6)
    sels = sel_list(ref, rng)
    q = queries(A, Cm, lens, 40, 9)
    xt = torch.from_numpy(q).cuda()
    assign = rng.integers(-1, len(sels), len(q))
    Dw, Iw = twin.search(q, 10, filter=twin.make_query_filters(sels, assign))
    Dp, Ip, _ = twin.search_partial(xt, 10, filter=twin.make_query_filters(sels, assign))
    assert np.array_equal(Dp.cpu().numpy().view(np.int32), Dw.view(np.int32)) and np.array_equal(Ip.cpu().numpy(), Iw)
    off = np.concatenate([[0], np.cumsum(lens)])
    shards = []
    for lo, hi in shard_ranges(lens, 2):
        sh = gpu_index(A, Cm, pq, lens, codes[off[lo]:off[hi]], ids[off[lo]:off[hi]], shard=(lo, hi))
        sh.nprobe = nprobe
        qf = sh.make_query_filters(sels, assign)
        for i, sel in enumerate(sels):              # each shard holds its own lists' blocks
            o, b, w = qf.csr(i)
            want = np_csr(ref.list_len, FR.selected_rows(ref, sel), lo, hi)
            assert all(np.array_equal(a, c) for a, c in zip((o, b, w), want))
        shards.append((sh, qf))
    per = (len(q) + 1) // 2
    keys_g = torch.stack([sh.coarse_local(xt) for sh, _ in shards]).contiguous()
    parts = [sh.search_preassigned(keys_g, 10, filter=qf) for sh, qf in shards]
    rec = torch.cat([sh.coarse_split(xt[r * per:(r + 1) * per].contiguous()) for r, (sh, _) in enumerate(shards)]).contiguous()
    parts2 = [sh.search_assigned(rec, 10, filter=qf) for sh, qf in shards]
    for ps in (parts, parts2):
        D, I = merge_shards(*(torch.stack([p[i] for p in ps]).contiguous() for i in range(3)), 10)
        assert np.array_equal(D.cpu().numpy().view(np.int32), Dw.view(np.int32)) and np.array_equal(I.cpu().numpy(), Iw)


def test_rejections_change_nothing(oracle):
    arrs, ref = case(oracle, 64, "explicit", n=8000, seed=4)
    A, Cm, pq, lens, codes, ids = arrs
    ix = gpu_index(*arrs)
    other = gpu_index(*arrs)
    ix.nprobe = other.nprobe = 16
    q = queries(A, Cm, lens, 16, 4)
    sels = [np.asarray(ids[::4]), range(int(ids.min()), int(np.median(ids)))]
    assign = np.arange(16) % 3 - 1
    D0, I0 = ix.search(q, 10)

    def state(g):
        return [a.copy() for a in g.lists()] + [g.device_bytes]

    def same(a, b):
        return all(np.array_equal(x, y) for x, y in zip(a, b))

    def unchanged():
        assert same(state(ix), before)
        D, I = ix.search(q, 10)
        assert np.array_equal(D.view(np.int32), D0.view(np.int32)) and np.array_equal(I, I0)

    before = state(ix)
    with pytest.raises(ValueError):
        ix.make_query_filters(sels, np.array([0, 2]))
    with pytest.raises(RuntimeError, match="assigned selector"):     # the C check, past the Python one
        from densephrases_b200 import _lib as L
        import ctypes as C
        h = C.c_void_p()
        a = np.array([5], np.int32)
        r = np.zeros(2, np.int64)
        L.check(L.lib().dph_query_filter_create(C.byref(h), ix._h, None, None, r.ctypes.data, 1, a.ctypes.data, 1, L.MEM_HOST))
    with pytest.raises(RuntimeError, match="not both"):
        lab = np.asarray(ids[:3])
        lo_ = np.array([0, 3], np.int64)
        r = np.array([1, 5], np.int64)
        a = np.zeros(1, np.int32)
        L.check(L.lib().dph_query_filter_create(C.byref(h), ix._h, lab.ctypes.data, lo_.ctypes.data, r.ctypes.data, 1, a.ctypes.data, 1,
                                                L.MEM_HOST))
    unchanged()
    with pytest.raises(RuntimeError, match="another index"):
        ix.search(q, 10, filter=other.make_query_filters(sels, assign))
    unchanged()
    with pytest.raises(RuntimeError, match="queries"):
        ix.search(q[:5], 10, filter=ix.make_query_filters(sels, assign))
    unchanged()
    f = ix.make_query_filters(sels, assign)
    ix.remove_ids(np.asarray(ids[1::9]))
    after = state(ix)
    with pytest.raises(RuntimeError, match="rebuild the filter"):
        ix.search(q, 10, filter=f)
    assert same(state(ix), after)
    lens2, codes2, ids2 = ix.lists()
    ref2 = oracle.RefIndex(A, pq, lens2, centroids=Cm, codes=codes2, ids=ids2)
    Du, Iu = ix.search(q, 10)                                        # nothing stays set on the handle
    Dr, Ir = ref2.search(q, 10, 16)
    assert_topk_equal(Du, Iu, Dr, Ir, "unfiltered after the rejections")
    D, I = ix.search(q, 10, filter=ix.make_query_filters(sels, assign))
    Dq, Iq = query_filtered_search(ref2, q, 10, 16, [FR.selected_rows(ref2, s) for s in sels], assign)
    assert_topk_equal(D, I, Dq, Iq, "rebuilt")


def test_mips_doc_filters(oracle):
    from densephrases_b200.mips import MIPS
    nlist = 64
    A, Cm, pq = model(oracle, nlist)
    lens, codes, _ = arrays(nlist, 20000, 21, False)
    ix = gpu_index(A, Cm, pq, lens, codes, None)
    ix.nprobe = 32
    N = int(lens.sum())
    rng = np.random.default_rng(21)
    doc = np.sort(rng.integers(0, 300, N)).astype(np.int32)          # one run per document, as idx2id groups are built
    idx_f = {'0': {'doc': doc, 'word': np.zeros(N, np.int32)}}
    mips = MIPS.from_components(ix, idx_f, None, cuda=False, index_path='synthetic_PQ')
    B = 6
    query = np.concatenate([queries(A, Cm, lens, B, 3), queries(A, Cm, lens, B, 4)], 1)
    per_q = [rng.choice(300, 5, replace=False) for _ in range(B)]
    per_q[2] = None
    out = mips.search_dense(query, ['q'] * B, top_k=20, doc_filter=mips.doc_filters(per_q))
    for i, docs in enumerate(per_q):
        f = None if docs is None else mips.doc_filter(docs)
        one = mips.search_dense(query[i:i + 1], ['q'], top_k=20, doc_filter=f)
        for a, b in zip(out, one):
            assert np.array_equal(np.asarray(a)[i:i + 1], np.asarray(b)), i
        if docs is not None:
            for d, lab in ((out[0][i], out[2][i]), (out[3][i], out[5][i])):
                assert set(d[lab >= 0].tolist()) <= set(docs.tolist())
