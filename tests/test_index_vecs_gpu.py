"""GPU: building a phrase index from an int8 phrase dump.  add_int8 against add_with_ids of the fp32-chain rows and the oracle's
encoding, from every kind of input buffer and on every kind of index; run_index over seeded dumps; merge of sub-indexes; and the
dump -> index -> meta -> MIPS path end to end."""
import os

import numpy as np
import pytest

from oracle import encode_ref as E
from tests.helpers import opq_matrix

pytestmark = pytest.mark.gpu
SEED = 91
OFFSET, SCALE = -1.7, 17.3           # neither is exact in fp32


def model(oracle, nlist):
    return opq_matrix(SEED), oracle.gen_centroids(SEED, 0, nlist), oracle.gen_pq(SEED)


def empty_index(A, Cm, pq, nlist, shard=None, host_capacity_bytes=None):
    from densephrases_b200 import IvfPqIndex
    return IvfPqIndex.from_arrays(A, Cm, pq, np.zeros(nlist, np.int64), np.zeros((0, 96), np.uint8), shard=shard,
                                  codes_on_host=host_capacity_bytes is not None, host_capacity_bytes=host_capacity_bytes)


def int8_rows(n, seed):
    q = np.random.default_rng(seed).integers(-128, 128, (n, 768)).astype(np.int8)
    q[0, :2] = (-128, 127)
    return q


def view(q, kind):
    """q's values in a buffer of the given kind, 16-byte aligned or at byte offset 1 ("_unaligned")."""
    import torch
    shift = 1 if kind.endswith("_unaligned") else 0
    kind = kind.replace("_unaligned", "")
    if kind == "pageable":
        buf = np.empty(q.size + 64, np.int8)
        base = (-buf.ctypes.data) % 16 + shift
        out = buf[base:base + q.size].reshape(q.shape)
        out[:] = q
        return out
    t = torch.empty(q.size + 64, dtype=torch.int8, pin_memory=(kind == "pinned"), device="cuda" if kind == "device" else "cpu")
    base = (-t.data_ptr()) % 16 + shift
    out = t[base:base + q.size].view(q.shape)
    out.copy_(torch.from_numpy(q))
    assert (out.data_ptr() % 16 == 0) == (shift == 0)
    return out.numpy() if kind == "pinned" else out           # a numpy view of page-locked memory: read in place


def assert_same_lists(a, b, what=""):
    la, ca, ia = a.lists()
    lb, cb, ib = b.lists()
    assert np.array_equal(la, lb) and np.array_equal(ca, cb) and np.array_equal(ia, ib), what


@pytest.mark.parametrize("kind", ["pageable", "pinned", "device", "pageable_unaligned", "pinned_unaligned", "device_unaligned"])
def test_add_int8_matches_add_with_ids_and_oracle(oracle, kind):
    from densephrases_b200.build_index import int8_to_float
    nlist, n = 64, 700
    A, Cm, pq = model(oracle, nlist)
    q = int8_rows(n, 1)
    x = int8_to_float(q, OFFSET, SCALE)
    ids = 5 + np.arange(n, dtype=np.int64) * 3
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    ref.add_with_ids(x, ids)
    ix8, ixf = empty_index(A, Cm, pq, nlist), empty_index(A, Cm, pq, nlist)
    import torch
    qv = view(q, kind)
    ix8.add_int8(qv, torch.from_numpy(ids).cuda() if kind.startswith("device") else ids, np.float64(OFFSET), np.float64(SCALE))
    ixf.add_with_ids(x, ids)
    assert_same_lists(ix8, ixf, kind)
    lens, codes, got_ids = ix8.lists()
    assert np.array_equal(lens, ref.list_len) and np.array_equal(codes, ref.codes) and np.array_equal(got_ids, ref.ids), kind


@pytest.mark.parametrize("kind", ["pageable", "pinned_unaligned", "device_unaligned"])
def test_add_int8_across_staging_chunks(oracle, monkeypatch, kind):
    from densephrases_b200.build_index import int8_to_float
    nlist, n = 32, 1000
    A, Cm, pq = model(oracle, nlist)
    q = int8_rows(n, 2)
    monkeypatch.setenv("DPH_UPLOAD_CHUNK_ROWS", "97")           # 11 chunks of dequantisation and encoding
    ix8, ixf = empty_index(A, Cm, pq, nlist), empty_index(A, Cm, pq, nlist)
    ix8.add_int8(view(q, kind), None, -2.0, 20.0)
    ix8.add_int8(view(q[:333], kind), None, OFFSET, SCALE)
    ixf.add_with_ids(int8_to_float(q, -2.0, 20.0), None)
    ixf.add_with_ids(int8_to_float(q[:333], OFFSET, SCALE), None)
    assert_same_lists(ix8, ixf, kind)


def test_add_int8_on_a_shard_and_a_host_index(oracle):
    from densephrases_b200.build_index import int8_to_float
    nlist, n = 64, 500
    A, Cm, pq = model(oracle, nlist)
    q = int8_rows(n, 3)
    x = int8_to_float(q, OFFSET, SCALE)
    ids = np.arange(n, dtype=np.int64) + 10 ** 9
    sh8, shf = empty_index(A, Cm, pq, nlist, shard=(16, 40)), empty_index(A, Cm, pq, nlist, shard=(16, 40))
    sh8.add_int8(q, ids, OFFSET, SCALE)
    shf.add_with_ids(x, ids)
    assert_same_lists(sh8, shf, "shard")
    assert sh8.ntotal == n
    ref = E.GrowableRefIndex(A, pq, np.zeros(nlist, np.int64), centroids=Cm)
    ref.add_with_ids(x, ids)
    ref.add_with_ids(x[:77], ids[:77] + n)
    host = empty_index(A, Cm, pq, nlist, host_capacity_bytes=64 << 20)
    host.add_int8(q, ids, OFFSET, SCALE)
    host.add_int8(view(q[:77], "pinned_unaligned"), ids[:77] + n, OFFSET, SCALE)
    lens, codes, got = host.lists()
    assert np.array_equal(lens, ref.list_len) and np.array_equal(codes, ref.codes) and np.array_equal(got, ref.ids)


def test_add_int8_rejections_leave_the_index_unchanged(oracle):
    from densephrases_b200 import IvfPqIndex
    nlist, n = 16, 64
    A, Cm, pq = model(oracle, nlist)
    q = int8_rows(n, 4)
    ix = empty_index(A, Cm, pq, nlist)
    ix.add_int8(q, None, OFFSET, SCALE)
    before = ix.lists()
    bad = [(q, None, OFFSET, 0.0), (q, None, OFFSET, np.inf), (q, None, OFFSET, np.nan), (q, None, np.nan, SCALE),
           (q, None, -np.inf, SCALE), (q, None, OFFSET, 1e40),           # 1e40 is inf in fp32
           (q, None, OFFSET, 1e-45),                                     # finite, but 127 / 1e-45 is not
           (q, np.arange(n, dtype=np.int64) - 1, OFFSET, SCALE)]        # a negative label
    for args in bad:
        with pytest.raises(RuntimeError):
            ix.add_int8(*args)
        after = ix.lists()
        assert all(np.array_equal(a, b) for a, b in zip(before, after)), args[2:]
    with pytest.raises(RuntimeError, match="read-only"):
        ro = IvfPqIndex.from_arrays(A, Cm, pq, np.zeros(nlist, np.int64), np.zeros((0, 96), np.uint8), codes_on_host=True)
        ro.add_int8(q, None, OFFSET, SCALE)
    small = empty_index(A, Cm, pq, nlist, host_capacity_bytes=3072)
    with pytest.raises(RuntimeError, match="capacity"):
        small.add_int8(q, None, OFFSET, SCALE)
    assert small.ntotal == 0


def golden_rows(paths):
    """The fp32-chain rows of the dumps in add order (file order, then h5py name order), documents with rows only."""
    from densephrases_b200 import dump
    from densephrases_b200.build_index import int8_to_float
    out = []
    for p in paths:
        groups = dump.read_dump(p)
        for name in sorted(groups, key=lambda k: k.encode()):
            ds, attrs = groups[name]
            if len(ds['start']):
                out.append(int8_to_float(ds['start'], attrs['offset'], attrs['scale']))
    return np.concatenate(out)


def test_run_index_matches_reference_and_oracle(oracle, tmp_path):
    import gzip
    import hashlib
    import json
    from densephrases_b200 import artifacts, build_index
    from tests import index_vecs_cases as cases
    with gzip.open(os.path.join(os.path.dirname(__file__), 'golden', 'index_vecs_reference.json.gz')) as f:
        g = json.load(f)
    d = str(tmp_path / 'dump')
    paths = cases.write_dumps(d)
    common = ['--dump_dir', d, '--fine_quant', 'OPQ96', '--num_clusters', '8', '--doc_sample_ratio', '1.0', '--vec_sample_ratio', '1.0']
    a = build_index.get_args(common + ['--stage', 'all'])
    timings = build_index.run_index(a)
    assert {'sample', 'train', 'read', 'gather', 'add', 'write'} <= set(timings)
    x = golden_rows(paths)
    assert hashlib.sha256(x.tobytes()).hexdigest() == g['add']['all_2000']['x']
    idx = artifacts.read_idx2id(a.idx2id_path)['0']
    assert idx['doc'].tolist() == g['add']['all_2000']['doc'] and idx['word'].tolist() == g['add']['all_2000']['word']
    t = artifacts.read_faiss_index(a.trained_index_path)
    assert t['ntotal'] == 0 and os.path.exists(os.path.join(a.index_dir, 'avg_vec.pkl'))
    ref = E.GrowableRefIndex(t['A'], t['pq'], np.zeros(8, np.int64), centroids=t['centroids'])
    ref.add_with_ids(x, np.array(g['add']['all_2000']['ids'], np.int64))
    got = artifacts.read_faiss_index(a.index_path)
    assert np.array_equal(got['list_len'], ref.list_len) and np.array_equal(got['codes'], ref.codes) and np.array_equal(got['ids'], ref.ids)
    # two sub-indexes and their merge == the single build, labels of the second file shifted to 1e9 + k
    for files, off in (('0-20.hdf5', 0), ('20-40.hdf5', 1000000000)):
        build_index.run_index(build_index.get_args(common + ['--stage', 'add', '--dump_paths', files, '--offset', str(off)]))
    m = build_index.get_args(common + ['--stage', 'merge', '--replace'])
    build_index.run_index(m)
    merged = artifacts.read_faiss_index(m.index_path)
    n0 = g['add']['sub0']['n']
    shifted = np.where(got['ids'] >= n0, got['ids'] - n0 + 1000000000, got['ids'])
    assert np.array_equal(merged['list_len'], got['list_len']) and np.array_equal(merged['codes'], got['codes'])
    assert np.array_equal(merged['ids'], shifted)
    assert sorted(artifacts.read_idx2id(m.idx2id_path)) == ['0', '1000000000']


def test_dump_to_index_to_mips_end_to_end(oracle, tmp_path):
    """dump_phrases (GPU encoder) -> run_index --stage all -> write_meta -> MIPS over index.faiss, idx2id.hdf5 and
    meta_compressed.pkl: a query built from a kept row finds the oracle's top hit of the same index, with the dump's text."""
    import argparse
    import json
    from densephrases_b200 import artifacts, build_index, dump
    from densephrases_b200.encoder import BertGeometry, Encoder, random_phrase_state_dict
    from densephrases_b200.mips import MIPS
    from oracle import ivfpq_ref
    from tests import dump_cases
    from tests.test_dump_cpu import G
    tok = dump_cases.tokenizer()
    geo = BertGeometry(vocab_size=max(tok.vocab.values()) + 1)
    enc = Encoder(geo, state_dict=random_phrase_state_dict(geo, 3), device=0, phrase_only=True)
    (tmp_path / 'data').mkdir()
    (tmp_path / 'data' / 'dev.json').write_text(json.dumps({'data': G['documents'] * 6}))
    dump_dir = str(tmp_path / 'out' / 'dump')
    args = argparse.Namespace(output_dir=str(tmp_path / 'out'), data_dir=str(tmp_path / 'data'), predict_file='dev.json', max_seq_length=64,
                              doc_stride=20, append_title=True, per_gpu_eval_batch_size=4, max_answer_length=10, do_lower_case=False,
                              filter_threshold=-1e8, dense_offset=-2.0, dense_scale=20.0, n_gpu=1)
    path = dump.dump_phrases(args, enc, tok)
    groups = dump.read_dump(path)
    assert sum(len(gr[0]['start']) for gr in groups.values()) >= 256
    a = build_index.get_args(['--dump_dir', dump_dir, '--stage', 'all', '--num_clusters', '32', '--fine_quant', 'OPQ96',
                              '--doc_sample_ratio', '1.0', '--vec_sample_ratio', '1.0'])
    build_index.run_index(a)
    artifacts.write_meta(os.path.join(dump_dir, 'phrase'), dump_dir)
    mips = MIPS(os.path.join(dump_dir, 'phrase'), a.index_path, a.idx2id_path, cuda=True)
    assert mips.doc_groups is not None and mips.is_pq
    idx = artifacts.read_idx2id(a.idx2id_path)['0']
    names = sorted((k for k in groups if len(groups[k][0]['start'])), key=lambda k: k.encode())
    rows = golden_rows([path])
    r = int(np.argmax((rows.astype(np.float64) ** 2).sum(1)))
    assert (str(idx['doc'][r]), idx['word'][r]) in {(k, w) for k in names for w in range(len(groups[k][0]['start']))}
    parts = artifacts.read_faiss_index(a.index_path)
    ref = ivfpq_ref.RefIndex(parts['A'], parts['pq'], parts['list_len'], centroids=parts['centroids'], codes=parts['codes'], ids=parts['ids'])
    _, I = ref.search(rows[r:r + 1], 1, nprobe=256)
    lab = int(I[0, 0])
    best = mips.search(np.concatenate([rows[r], rows[r]])[None], q_texts=['q'], top_k=5)[0][0]
    doc, word = int(idx['doc'][lab]), int(idx['word'][lab])
    assert (best['doc_idx'], best['start_idx']) == (doc, word)
    ds, attrs = groups[str(doc)]
    w2s, w2e, f2o = ds['word2char_start'], ds['word2char_end'], ds['f2o_start']
    c0, c1 = int(w2s[f2o[best['start_idx']]]), int(w2e[f2o[best['end_idx']]])
    assert c1 > c0 and best['answer'] == attrs['context'][c0:c1]
    assert best['context'] in attrs['context'] and best['context'][best['start_pos']:best['end_pos']] == best['answer']
    assert best['title'] == [attrs['title']]
