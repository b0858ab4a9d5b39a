"""GPU: an index whose codes are in host memory (DESIGN.md 3.5) against its twin in device memory built from the same arrays: search
bits (D and I) in every scan mode, k, nprobe, stream-region size and resident set; the fetch counters against the slicing rule of
tests/host_codes_ref.py; reconstruct, window scores, lists(), both sharded protocols' local steps and MIPS; and the rejected calls."""
import numpy as np
import pytest

from tests.host_codes_ref import blocks, np_slices
from tests.test_add_gpu import gpu_index, model, vectors_near
from tests.test_merge_gpu import arrays

pytestmark = pytest.mark.gpu
QUAD, PAIR, SINGLE, EXACT = 4, 2, 3, 1


def host_index(A, Cm, pq, lens, codes, ids, stream_bytes, shard=None):
    from densephrases_b200 import IvfPqIndex
    return IvfPqIndex.from_arrays(A, Cm, pq, lens, codes, ids, shard=shard, codes_on_host=True, stream_bytes=stream_bytes)


def queries(A, Cm, lens, n, seed):
    rng = np.random.default_rng(seed)
    return vectors_near(A, Cm, rng.choice(np.flatnonzero(lens), n), seed, noise=0.3)


def assert_bits(got, want, what=""):
    assert np.array_equal(got[0].view(np.int32), want[0].view(np.int32)), what
    assert np.array_equal(got[1], want[1]), what


def fetch_counts(ix):
    f = ix.last_fetch()
    return [f["slices"], f["lists_fetched"], f["blocks_fetched"], f["resident_lists_scanned"]]


@pytest.mark.parametrize("labels", ["seq", "explicit"])
@pytest.mark.parametrize("nlist", [1, 16, 512, 4096])
def test_search_bits_equal_the_resident_twin(oracle, nlist, labels):
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 20000, 7, labels == "explicit")
    nb = blocks(lens)
    everything, tight = int(nb.sum()) * 3072, (int(nb.max()) + 1) * 3072       # one slice, or many (just above the largest list)
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    ix = host_index(A, Cm, pq, lens, codes, ids, everything)
    assert ix.host_bytes == int(nb.sum()) * 3072 and ix.ntotal == twin.ntotal
    q = queries(A, Cm, lens, 48, nlist)
    want = {}
    for nprobe in (1, 16, 256):
        twin.nprobe = nprobe
        for mode in (QUAD, PAIR, SINGLE, EXACT):
            twin.set_scan_mode(mode)
            for k in (1, 10, 100):
                want[nprobe, mode, k] = twin.search(q, k)
    half = np.random.default_rng(nlist).choice(nlist, nlist // 2, replace=False)
    for res in ([], half, np.arange(nlist)):
        ix.set_resident_lists(res)
        for region in (everything, tight):
            ix.set_code_residency(True, region)
            for (nprobe, mode, k), w in want.items():
                ix.nprobe = nprobe
                ix.set_scan_mode(mode)
                what = f"res={len(res)} region={region} nprobe={nprobe} mode={mode} k={k}"
                assert_bits(ix.search(q, k), w, what)
                _, counts = np_slices(ix.last_probes(len(q)), lens, res, region // 3072, 0, nlist)
                assert fetch_counts(ix) == counts, what
                if len(res) == nlist:
                    assert counts[0] == 1 and counts[2] == 0
    assert ix.ntotal == twin.ntotal and ix.host_bytes == int(nb.sum()) * 3072


@pytest.mark.parametrize("labels", ["seq", "explicit"])
def test_reconstruct_window_scores_and_lists_equal_the_twin(oracle, labels, monkeypatch):
    monkeypatch.setenv("DPH_UPLOAD_CHUNK_ROWS", "700")        # many staging chunks through the host copy
    nlist = 512
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 9000, 3, labels == "explicit")
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    ix = host_index(A, Cm, pq, lens, codes, ids, None)
    ix.set_resident_lists(np.arange(0, nlist, 3))
    for a, b in zip(ix.lists(), twin.lists()):
        assert np.array_equal(a, b)
    labs = np.concatenate([ids if ids is not None else np.arange(len(codes)), [-1, 10**12]]).astype(np.int64)
    v, f = ix.reconstruct_batch(labs)
    vt, ft = twin.reconstruct_batch(labs)
    assert np.array_equal(v.view(np.int32), vt.view(np.int32)) and np.array_equal(f, ft) and f[:-2].all()
    rng = np.random.default_rng(4)
    qv = rng.standard_normal((64, 768)).astype(np.float32)
    first = rng.choice(labs[:-2], 64)
    assert np.array_equal(ix.window_scores(qv, first, 5).view(np.int32), twin.window_scores(qv, first, 5).view(np.int32))


def test_synthetic_lists_in_host_mode_equal_resident_mode(monkeypatch):
    from densephrases_b200 import IvfPqIndex
    monkeypatch.setenv("DPH_UPLOAD_CHUNK_ROWS", "3000")
    nlist, seed = 64, 11
    lens = np.random.default_rng(seed).integers(0, 2000, nlist) * (np.arange(nlist) % 4 != 1)
    A = np.linalg.qr(np.random.default_rng(seed).standard_normal((768, 768)))[0].astype(np.float32)
    made = []
    for on_host in (False, True):
        ix = IvfPqIndex(nlist)
        ix.set_opq(A); ix.gen_centroids(seed); ix.gen_pq(seed)
        if on_host:
            ix.set_code_residency(True, 200 * 3072)
        ix.set_lists_synthetic(lens, seed)
        made.append(ix)
    twin, ix = made
    for a, b in zip(ix.lists(), twin.lists()):
        assert np.array_equal(a, b)
    q = queries(A, ix.centroids(), lens, 32, 2)
    for g in made:
        g.nprobe = 24
    assert_bits(ix.search(q, 10), twin.search(q, 10))
    assert ix.last_fetch()["slices"] > 1


def test_two_shards_in_host_mode_equal_the_unsharded_index(oracle):
    import torch
    from densephrases_b200 import merge_shards
    from densephrases_b200.sharded import shard_ranges
    nlist, k, nprobe = 96, 10, 24
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 30000, 5, True)
    twin = gpu_index(A, Cm, pq, lens, codes, ids)
    twin.nprobe = nprobe
    off = np.concatenate([[0], np.cumsum(lens)])
    shards = []
    for si, (lo, hi) in enumerate(shard_ranges(lens, 2)):
        nb = blocks(lens[lo:hi])
        sh = host_index(A, Cm, pq, lens, codes[off[lo]:off[hi]], ids[off[lo]:off[hi]], (int(nb.max()) + 2) * 3072, shard=(lo, hi))
        sh.set_resident_lists(np.arange(lo, hi, 2 + si))
        sh.nprobe = nprobe
        sh.set_scan_mode((QUAD, PAIR)[si])
        shards.append(sh)
    q = queries(A, Cm, lens, 40, 9)
    xt = torch.from_numpy(q).cuda()
    Dw, Iw = twin.search(q, k)
    keys_g = torch.stack([sh.coarse_local(xt) for sh in shards]).contiguous()       # list-split coarse quantizer
    parts = [sh.search_preassigned(keys_g, k) for sh in shards]
    per = (len(q) + 1) // 2                                                           # query-split coarse quantizer
    rec = torch.cat([sh.coarse_split(xt[r * per:(r + 1) * per].contiguous()) for r, sh in enumerate(shards)]).contiguous()
    parts2 = [sh.search_assigned(rec, k) for sh in shards]
    for ps in (parts, parts2):
        D, I = merge_shards(*(torch.stack([p[i] for p in ps]).contiguous() for i in range(3)), k)
        assert_bits((D.cpu().numpy(), I.cpu().numpy()), (Dw, Iw))
    assert all(sh.last_fetch()["slices"] >= 1 for sh in shards)


def _equal(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_equal(a[x], b[x]) for x in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return np.array_equal(np.asarray(a), np.asarray(b))
    return a == b or (a != a and b != b)


def test_mips_with_codes_on_host_equals_mips_in_device_memory(tmp_path, monkeypatch):
    from densephrases import Options
    from densephrases_b200 import runtime as R
    from densephrases_b200 import synthetic_dump as SD
    nlist = 32
    SD.write_synthetic_dump(str(tmp_path), f"start/{nlist}_flat_OPQ96", 128 * 300, nlist, 128, seed=1234)
    o = Options()
    o.add_model_options(); o.add_index_options(); o.add_retrieval_options(); o.add_data_options()
    args = o.parse(["--dump_dir", str(tmp_path), "--index_name", f"start/{nlist}_flat_OPQ96", "--cuda"])
    monkeypatch.delenv("DPH_CODES_ON_HOST", raising=False)
    dev = R.load_phrase_index(args, ignore_logging=True)
    monkeypatch.setenv("DPH_CODES_ON_HOST", "0.0002")           # ~210 KB: a few lists per slice
    host = R.load_phrase_index(args, ignore_logging=True)
    assert host.index.local.host_bytes > 0 and dev.index.local.host_bytes == 0
    qr = np.random.default_rng(5)
    query = qr.standard_normal((6, 1536))
    for idxs in (False, True):
        a = dev.search(query, q_texts=["q"] * 6, top_k=10, return_idxs=idxs)
        b = host.search(query, q_texts=["q"] * 6, top_k=10, return_idxs=idxs)
        assert _equal(a, b), f"return_idxs={idxs}"
    assert host.index.local.last_fetch()["slices"] > 1


def test_rejections_leave_the_index_unchanged(oracle):
    import torch
    nlist = 16
    A, Cm, pq = model(oracle, nlist)
    lens, codes, ids = arrays(nlist, 3000, 2, True)
    nb = blocks(lens)
    ix = host_index(A, Cm, pq, lens, codes, ids, int(nb.max()) * 3072)
    src = host_index(A, Cm, pq, lens, codes, ids + 10**6, None)
    dest = gpu_index(A, Cm, pq, lens, codes, ids)
    q = queries(A, Cm, lens, 16, 1)
    want = ix.search(q, 10)

    def state(g):
        return [a.copy() for a in g.lists()], g.ntotal, g.device_bytes, g.host_bytes

    def unchanged(before, g=ix):
        after = state(g)
        assert all(np.array_equal(a, b) for a, b in zip(before[0], after[0])) and before[1:] == after[1:]

    ix.set_code_residency(True, (int(nb.max()) - 1) * 3072)          # the region no longer holds the largest list
    s = state(ix)
    with pytest.raises(RuntimeError, match="stream region"):
        ix.search(q, 10)
    unchanged(s)
    ix.set_resident_lists([int(np.argmax(lens))])                    # ... unless that list is resident
    assert_bits(ix.search(q, 10), want)
    s = state(ix)
    for bad in ([nlist], [-1], [0, 3, 99]):
        with pytest.raises(RuntimeError, match="not in this shard"):
            ix.set_resident_lists(bad)
        unchanged(s)
    sh = host_index(A, Cm, pq, lens, codes[:int(lens[:8].sum())], ids[:int(lens[:8].sum())], None, shard=(0, 8))
    s8 = state(sh)
    with pytest.raises(RuntimeError, match="not in this shard"):
        sh.set_resident_lists([8])
    unchanged(s8, sh)
    x = vectors_near(A, Cm, [1, 2, 3], 0)
    for call in (lambda: ix.add_with_ids(x, np.array([7, 8, 9])), lambda: ix.add_with_ids(torch.from_numpy(x).cuda(), None),
                 lambda: ix.remove_ids(ids[:5].copy()), lambda: ix.remove_ids(range(0, 10**9)), lambda: ix.sync_list_len(lens),
                 lambda: ix.merge_from(src), lambda: ix.set_code_residency(False)):
        with pytest.raises(RuntimeError):
            call()
        unchanged(s)
    sd = state(dest)
    with pytest.raises(RuntimeError, match="host memory"):
        dest.merge_from(src)
    unchanged(sd, dest)
    assert_bits(ix.search(q, 10), want)
