"""CPU: building a phrase index from a phrase dump (build_index.run_index's host side, merge and write_meta) against the reference's
sample_data / add_to_index / merge_indexes / compress_metadata (tests/golden/index_vecs_reference.json.gz).  The device add is
replaced by a recorder of add_int8's calls here; test_index_vecs_gpu.py runs it."""
import ctypes
import gzip
import hashlib
import json
import os

import numpy as np
import pytest

from tests import index_vecs_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    with gzip.open(os.path.join(ROOT, "tests", "golden", "index_vecs_reference.json.gz")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def dump_dir(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("dump") / "dump")
    cases.write_dumps(d)
    return d


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def args_for(dump_dir, *extra):
    from densephrases_b200 import build_index
    return build_index.get_args(["--dump_dir", dump_dir, "--fine_quant", "OPQ96", "--num_clusters", "8", *extra])


def write_trained(path, nlist=8, seed=0):
    from densephrases_b200 import artifacts
    rng = np.random.default_rng(seed)
    A = np.linalg.qr(rng.standard_normal((768, 768)))[0].astype(np.float32)
    artifacts.write_faiss_index(path, A, rng.standard_normal((nlist, 768)).astype(np.float32),
                                rng.standard_normal((96, 256, 8)).astype(np.float32), np.zeros(nlist, np.int64),
                                np.zeros((0, 96), np.uint8), np.zeros(0, np.int64))


class _Recorder(object):
    """Stands in for the device index: records the rows add_int8 would add, dequantised by the fp32 chain."""

    def __init__(self, nlist):
        self.nlist, self.x, self.ids, self.calls = nlist, [], [], []

    def add_int8(self, q, ids, offset, scale):
        from densephrases_b200.build_index import int8_to_float
        assert q.dtype == np.int8
        self.x.append(int8_to_float(q, offset, scale))
        self.ids.append(np.array(ids))
        self.calls.append((len(q), offset, scale))

    def lists(self):
        return np.zeros(self.nlist, np.int64), np.zeros((0, 96), np.uint8), np.zeros(0, np.int64)


@pytest.fixture
def recorder(monkeypatch):
    from densephrases_b200 import artifacts, build_index
    made = []

    def fake(path, device=0):
        t = artifacts.read_faiss_index(path)
        made.append(_Recorder(len(t["list_len"])))
        return t, made[-1]
    monkeypatch.setattr(build_index, "_trained_index", fake)
    monkeypatch.setattr(build_index, "pinned_rows", lambda n: np.empty((n, 768), np.int8))
    return made


def test_int8_to_float_is_the_fp32_chain():
    from densephrases_b200.build_index import int8_to_float
    q = np.arange(-128, 128, dtype=np.int8)
    for off, scale in ((-2.0, 20.0), (-1.7, 17.3), (np.float64(-1.7), np.float64(17.3))):
        x = int8_to_float(q, off, scale)
        want = np.array([np.float32(np.float32(v) / np.float32(scale)) + np.float32(off) for v in q.tolist()], np.float32)
        assert x.dtype == np.float32 and np.array_equal(x.view(np.uint32), want.view(np.uint32))
    f64 = (q.astype(np.float64) / 20.0 - 2.0).astype(np.float32)
    assert int((int8_to_float(q, -2.0, 20.0) != f64).sum()) == 52        # numpy 2's float64 result differs in 52 of 256 values


def test_paths_follow_get_args(tmp_path):
    a = args_for("D")
    d = os.path.join("D", "start", "8_flat_OPQ96")
    assert (a.index_dir, a.trained_index_path, a.index_path, a.idx2id_path) == (
        d, os.path.join(d, "trained.faiss"), os.path.join(d, "index.faiss"), os.path.join(d, "idx2id.hdf5"))
    a = args_for("D", "--first_passage", "--dump_paths", "0-20.hdf5,20-40.hdf5", "--offset", "1000000000")
    d = os.path.join("D", "start", "8_flat_OPQ96_first")
    assert a.dump_paths == [os.path.join("D", "phrase", "0-20.hdf5"), os.path.join("D", "phrase", "20-40.hdf5")]
    assert (a.index_path, a.idx2id_path) == (os.path.join(d, "index", "1000000000.faiss"), os.path.join(d, "index", "1000000000.hdf5"))
    assert args_for("D", "--index_filter", "0.5").index_name == "8_flat_OPQ96_ft0"


@pytest.mark.parametrize("name,dr,vr,th", cases.SAMPLE_RUNS)
def test_sample_matches_reference(golden, dump_dir, name, dr, vr, th):
    from densephrases_b200.build_index import sample_data
    paths = [os.path.join(dump_dir, "phrase", f) for f in cases.FILES]
    x, avg, std = sample_data(paths, dr, vr, norm_th=th)
    g = golden["sample"][name]
    assert list(x.shape) == g["shape"] and str(x.dtype) == g["dtype"]
    assert (sha(x), sha(avg), sha(std)) == (g["x"], g["avg_vec"], g["std_vec"]), name


@pytest.mark.parametrize("run", cases.ADD_RUNS, ids=[r[0] for r in cases.ADD_RUNS])
def test_add_rows_labels_and_idx2id_match_reference(golden, dump_dir, recorder, tmp_path, run):
    from densephrases_b200 import artifacts, build_index
    name, files, offset, ndpa, first, filt = run
    trained = str(tmp_path / "trained.faiss")
    write_trained(trained)
    paths = [os.path.join(dump_dir, "phrase", cases.FILES[i]) for i in files]
    timings = {}
    build_index.add_dump_to_index(paths, trained, str(tmp_path / "index.faiss"), str(tmp_path / "idx2id.hdf5"), num_docs_per_add=ndpa,
                             offset=offset, first_passage=first, index_filter=filt, timings=timings)
    rec, g = recorder[-1], golden["add"][name]
    x = np.concatenate(rec.x)
    assert (sha(x), len(x)) == (g["x"], g["n"]), name
    assert np.concatenate(rec.ids).tolist() == g["ids"]
    assert timings["rows"] == g["n"] and timings["h2d_bytes"] == 768 * g["n"]
    idx = artifacts.read_idx2id(str(tmp_path / "idx2id.hdf5"))
    assert list(idx) == [str(offset)]
    assert idx[str(offset)]["doc"].dtype == np.int32 and idx[str(offset)]["word"].dtype == np.int32
    assert idx[str(offset)]["doc"].tolist() == g["doc"] and idx[str(offset)]["word"].tolist() == g["word"]
    tree = artifacts.open_hdf5(str(tmp_path / "idx2id.hdf5"))
    assert int(tree.attributes(tree.children(tree.root_addr)[str(offset)])["offset"]) == g["offset_attr"]


def test_mixed_offset_scale_documents_go_in_separate_calls(dump_dir, recorder, tmp_path):
    from densephrases_b200 import build_index
    trained = str(tmp_path / "trained.faiss")
    write_trained(trained)
    build_index.add_dump_to_index([os.path.join(dump_dir, "phrase", cases.FILES[1])], trained, str(tmp_path / "i.faiss"),
                             str(tmp_path / "i.hdf5"), num_docs_per_add=2000)
    calls = recorder[-1].calls              # documents 200 | 21 22 24, 25 (-2, 20), 30 39: the flush at i = 0, then three runs
    assert [c[1:] for c in calls] == [(-1.7, 17.3), (-1.7, 17.3), (-2.0, 20.0), (-1.7, 17.3)], calls


def test_merge_matches_reference_order_and_round_trips(golden, tmp_path):
    from densephrases_b200 import artifacts, build_index
    nlist = 8
    a = args_for(str(tmp_path / "d"), "--stage", "merge", "--inv_path", "merged.ivfdata")
    os.makedirs(a.subindex_dir)
    write_trained(a.trained_index_path, nlist)
    t = artifacts.read_faiss_index(a.trained_index_path)
    rng = np.random.default_rng(5)
    subs = {}
    for off, n in ((1000000000, 40), (0, 70)):
        lst = rng.integers(0, nlist, n)
        codes = rng.integers(0, 256, (n, 96)).astype(np.uint8)
        ids = off + np.arange(n, dtype=np.int64)
        lens, codes, ids = build_index.to_list_major(lst, codes, ids, nlist)
        artifacts.write_faiss_index(os.path.join(a.subindex_dir, f"{off}.faiss"), t["A"], t["centroids"], t["pq"], lens, codes, ids)
        g = golden["add"]["sub0" if off == 0 else "sub1"]
        artifacts.write_hdf5(os.path.join(a.subindex_dir, f"{off}.hdf5"),
                             {str(off): {"doc": np.array(g["doc"], np.int32), "word": np.array(g["word"], np.int32)}},
                             attrs={str(off): {"offset": off}})
        subs[off] = (lens, codes, ids)
    build_index.run_index(a)
    m = artifacts.read_faiss_index(a.index_path)
    assert os.path.exists(os.path.join(a.index_dir, "merged.ivfdata"))
    for key in ("A", "centroids", "pq"):
        assert np.array_equal(m[key], t[key])
    start = {o: np.concatenate([[0], np.cumsum(s[0])]) for o, s in subs.items()}
    want_codes, want_ids = [], []
    for l in range(nlist):                                         # each list: offset 0's entries, then 1e9's (ascending offsets)
        for o in (0, 1000000000):
            want_codes.append(subs[o][1][start[o][l]:start[o][l + 1]])
            want_ids.append(subs[o][2][start[o][l]:start[o][l + 1]])
    assert np.array_equal(m["list_len"], subs[0][0] + subs[1000000000][0])
    assert np.array_equal(m["codes"], np.concatenate(want_codes)) and np.array_equal(m["ids"], np.concatenate(want_ids))
    idx = artifacts.read_idx2id(a.idx2id_path)
    want = golden["merge"]["idx2id"]
    assert sorted(idx) == sorted(want)
    for k in want:
        assert idx[k]["doc"].tolist() == want[k]["doc"] and idx[k]["word"].tolist() == want[k]["word"]
    # a sub-index trained with other tables is rejected
    bad = dict(t)
    bad["pq"] = t["pq"].copy()
    bad["pq"].reshape(-1)[7] = np.nextafter(bad["pq"].reshape(-1)[7], np.float32(np.inf))
    artifacts.write_faiss_index(os.path.join(a.subindex_dir, "0.faiss"), bad["A"], bad["centroids"], bad["pq"], *subs[0])
    with pytest.raises(ValueError, match="bit-identical"):
        build_index.run_index(derive(a, replace=True))


def derive(a, **kw):
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_trained_and_index_files_round_trip(tmp_path):
    from densephrases_b200 import artifacts
    nlist = 8
    path = str(tmp_path / "trained.faiss")
    write_trained(path, nlist, seed=3)
    t = artifacts.read_faiss_index(path)
    assert t["ntotal"] == 0 and t["codes"].shape == (0, 96) and t["by_residual"] and t["metric"] == 0
    rng = np.random.default_rng(4)
    lens = rng.integers(0, 9, nlist)
    codes = rng.integers(0, 256, (int(lens.sum()), 96)).astype(np.uint8)
    ids = rng.permutation(int(lens.sum())).astype(np.int64) + 10 ** 9
    for payload in (None, "x.ivfdata"):
        p = str(tmp_path / f"index_{payload}.faiss")
        artifacts.write_faiss_index(p, t["A"], t["centroids"], t["pq"], lens, codes, ids, ondisk_payload=payload)
        r = artifacts.read_faiss_index(p)
        assert np.array_equal(r["list_len"], lens) and np.array_equal(r["codes"], codes) and np.array_equal(r["ids"], ids)


def test_meta_matches_reference(golden, dump_dir, tmp_path):
    from densephrases_b200 import artifacts
    from densephrases_b200.mips import MIPS
    out = artifacts.write_meta(os.path.join(dump_dir, "phrase"), str(tmp_path))
    assert out == os.path.join(str(tmp_path), "meta_compressed.pkl")
    meta = artifacts.read_meta(out)
    g = golden["meta"]
    assert list(meta) == g["order"]
    m = MIPS.__new__(MIPS)
    m.doc_groups = meta
    for key, want in g["records"].items():
        rec = meta[key]
        assert list(rec) == want["keys"]
        assert {k: str(v) for k, v in rec["dtypes"].items()} == want["dtypes"] and rec["title"] == want["title"]
        assert isinstance(rec["context"], bytes) and artifacts.decode_meta_field(rec["context"]).decode("utf-8") == want["context"]
        d = m.decompress_meta(key)
        assert d["context"] == want["context"] and d["title"] == want["title"]
        for t in ("word2char_start", "word2char_end", "f2o_start"):
            assert d[t].tolist() == want[t] and d[t].dtype == np.dtype(want["dtypes"][t]), (key, t)


def test_compress_metadata_cli(dump_dir, tmp_path):
    from densephrases_b200 import compress_metadata
    compress_metadata.main(["--input_dump_dir", os.path.join(dump_dir, "phrase"), "--output_dir", str(tmp_path)])
    assert os.path.getsize(tmp_path / "meta_compressed.pkl") > 0


@pytest.mark.parametrize("extra,match", [((), "SQ4"), (("--fine_quant", "none"), "none"), (("--hnsw",), "hnsw"),
                                         (("--stage", "move"), "move"), (("--first_passage", "--index_filter", "0.5"), "together")])
def test_refusals(tmp_path, extra, match):
    from densephrases_b200 import build_index
    argv = ["--dump_dir", str(tmp_path), "--stage", "all", "--num_clusters", "8"]
    if "--fine_quant" not in extra and extra != ():
        argv += ["--fine_quant", "OPQ96"]
    a = build_index.get_args(argv + list(extra))
    with pytest.raises(ValueError, match=match):
        build_index.run_index(a)


def test_small_sample_is_refused_before_training(tmp_path):
    from densephrases_b200 import build_index
    with pytest.raises(ValueError, match="at least"):
        build_index.train_phrase_index(np.zeros((255, 768), np.float32), 8, str(tmp_path / "t.faiss"))
    with pytest.raises(ValueError, match="at least"):
        build_index.train_phrase_index(np.zeros((300, 768), np.float32), 512, str(tmp_path / "t.faiss"))


def test_add_int8_is_exported():
    from densephrases_b200 import _lib
    assert "dph_index_add_int8" in _lib.EXPORTS
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "dph_index_add_int8")
