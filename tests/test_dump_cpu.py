"""CPU: the phrase dump's host side and its numpy oracle against the unmodified reference (tests/golden/dump_reference.json.gz):
context features, character offsets, the select / quantise / re-index restatement, the HDF5 file and the dump flags."""
import gzip
import hashlib
import json
import os

import numpy as np
import pytest

from densephrases_b200 import artifacts, dump
from densephrases_b200.phrase_dump import PhraseDump
from oracle import dump_ref
from tests import dump_cases

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'dump_reference.json.gz')


def golden():
    with gzip.open(GOLDEN, 'rb') as f:
        return json.loads(f.read())


G = golden()
CASES = {c[0]: c for c in dump_cases.CASES}
RUNS = [(c['name'], r['filter_threshold']) for c in G['cases'] for r in c['runs']]


def build(name):
    _, S, stride, title, L, thrs, off, scale, seed = CASES[name]
    tok = dump_cases.tokenizer()
    examples = dump.read_examples(G['documents'])
    features = dump.convert_examples_to_features(examples, tok, S, stride, title)
    toffs = dump.title_offsets(features, tok, title)
    start, logits = dump_cases.phrase_outputs(features, S, seed, [t + 1 for t in toffs])
    return tok, examples, features, toffs, start, logits


def oracle_groups(name, thr):
    """{did: (datasets, attrs)} from the product's features and offsets and the oracle's numeric fields."""
    _, S, stride, title, L, thrs, off, scale, seed = CASES[name]
    tok, examples, features, toffs, start, logits = build(name)
    out = {}
    for idxs in dump.documents(examples, features):
        lo = [toffs[i] + 1 for i in idxs]
        hi = [len(features[i].tokens) - 1 for i in idxs]
        rows = lambda a: np.concatenate([a[i, l:h] for i, l, h in zip(idxs, lo, hi)])       # noqa: E731
        q, f2o, s2e = dump_ref.select_document(rows(start), rows(logits[..., 0]), rows(logits[..., 1]), np.subtract(hi, lo), L, thr, off, scale)
        fl = [features[i] for i in idxs]
        context, w2s, w2e = dump.document_offsets(examples, fl, [toffs[i] for i in idxs], False, tok)
        ex = examples[fl[-1].example_index]
        out[str(ex.doc_idx)] = ({'start': q, 'len_per_para': np.subtract(hi, lo).astype(np.int64), 'start2end': s2e, 'word2char_start': w2s,
                                 'word2char_end': w2e, 'f2o_start': f2o},
                                {'context': context, 'title': ex.title, 'offset': off, 'scale': scale})
    return out


def check_value(got, want, what):
    if isinstance(want, dict):
        got = np.asarray(got)
        assert str(got.dtype) == want['dtype'] and list(got.shape) == want['shape'], f'{what}: {got.dtype} {got.shape} vs {want}'
        if 'sha256' in want:
            assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == want['sha256'], f'{what}: bytes differ'
        else:
            assert got.reshape(-1).tolist() == want['data'], f'{what}: values differ'
    else:
        assert got == want, f'{what}: {got!r} vs {want!r}'


def check_groups(groups, want):
    assert sorted(groups) == sorted(want)
    for did, (ds, attrs) in groups.items():
        assert sorted(ds) == sorted(want[did]['datasets']) and sorted(attrs) == sorted(want[did]['attrs'])
        for k, v in want[did]['datasets'].items():
            check_value(ds[k], v, f'{did}/{k}')
        for k, v in want[did]['attrs'].items():
            check_value(attrs[k], v, f'{did}@{k}')


@pytest.mark.parametrize('name', sorted(CASES))
def test_features_match_reference(name):
    _, S, stride, title, *_ = CASES[name]
    tok = dump_cases.tokenizer()
    features = dump.convert_examples_to_features(dump.read_examples(G['documents']), tok, S, stride, title)
    want = next(c for c in G['cases'] if c['name'] == name)['features']
    assert len(features) == len(want)
    for f, w in zip(features, want):
        n = sum(f.attention_mask)
        assert f.input_ids[:n] == w['input_ids'] and n == w['attention_mask'] and sorted(set(f.token_type_ids)) == w['token_type_ids']
        assert f.tokens == w['tokens'] and sorted(f.token_to_orig_map.items()) == [tuple(x) for x in w['token_to_orig_map']]
        for k in ('paragraph_len', 'title_offset', 'span_idx', 'par_idx', 'doc_idx', 'example_index', 'unique_id'):
            assert getattr(f, k) == w[k], k


@pytest.mark.parametrize('name,thr', RUNS)
def test_oracle_and_offsets_match_reference(name, thr):
    run = next(r for c in G['cases'] if c['name'] == name for r in c['runs'] if r['filter_threshold'] == thr)
    check_groups(oracle_groups(name, thr), run['groups'])


def test_threshold_is_compared_in_fp32():
    """fp32(0.1) > 0.1 in float64 but not in float32: the reference's numpy comparison keeps neither row."""
    fs = np.array([np.float32(0.1), 0.5], np.float32)
    q, f2o, s2e = dump_ref.select_document(np.zeros((2, 768), np.float32), fs, fs, [2], 2, 0.1, -2.0, 20.0)
    assert f2o.tolist() == [1] and s2e.tolist() == [[0, -1]]


def test_write_and_read_back(tmp_path):
    name, thr = RUNS[0]
    groups = oracle_groups(name, thr)
    path = str(tmp_path / 'dev.hdf5')
    first = dict(list(groups.items())[:2])
    dump.write_dump(path, first)
    dump.write_dump(path, groups)                    # appends: existing groups kept, re-dumped ones replaced
    tree = artifacts.read_hdf5(path)
    back = dump.read_dump(path)
    pd = PhraseDump(path)
    for did, (ds, attrs) in groups.items():
        for k, v in ds.items():
            assert tree[did][k].dtype == v.dtype and np.array_equal(tree[did][k], v) and np.array_equal(back[did][0][k], v)
        assert back[did][1] == attrs
        rec = pd.get(int(did))
        assert rec['context'] == attrs['context'] and rec['title'] == attrs['title']
        assert np.array_equal(np.asarray(rec['start']), ds['start']) and np.array_equal(rec['f2o_start'], ds['f2o_start'])


def many_groups(tmp_path, n):
    path = str(tmp_path / f'big{n}.hdf5')
    tree = {str(i): {'f2o_start': np.arange(i % 5, dtype=np.int64)} for i in range(n)}
    artifacts.write_hdf5(path, tree, attrs={k: {'title': f't{k}', 'offset': -2.0} for k in tree})
    return path, tree


@pytest.mark.parametrize('n', [257, 1500, 9000])
def test_many_groups_round_trip(tmp_path, n):
    """More than 256 documents in one file: group B-trees of two (257, 1500) and three (9000) levels."""
    path, tree = many_groups(tmp_path, n)
    back = dump.read_dump(path)
    assert sorted(back) == sorted(tree)
    assert all(np.array_equal(back[k][0]['f2o_start'], v['f2o_start']) and back[k][1] == {'title': f't{k}', 'offset': -2.0}
               for k, v in tree.items())


def test_group_tree_nodes_link_their_siblings(tmp_path):
    """Every B-tree node of a level points to its left and right neighbours (UNDEF at the ends), as libhdf5 expects."""
    import struct
    path, _ = many_groups(tmp_path, 9000)
    h = artifacts.open_hdf5(path)
    btree = next(struct.unpack_from('<Q', h.buf, data)[0] for t, _, data, _ in h.messages(h.root_addr) if t == 0x0011)
    level_nodes = [[btree]]
    while True:
        nodes = level_nodes[-1]
        ntype, level, used = struct.unpack_from('<BBH', h.buf, nodes[0] + 4)
        if level == 0:
            break
        level_nodes.append([struct.unpack_from('<Q', h.buf, a + 32 + 16 * i)[0] for a in nodes for i in range(struct.unpack_from('<H', h.buf, a + 6)[0])])
    assert len(level_nodes) == 3
    undef = 0xFFFFFFFFFFFFFFFF
    for nodes in level_nodes:
        for i, a in enumerate(nodes):
            left, right = struct.unpack_from('<QQ', h.buf, a + 8)
            assert left == (nodes[i - 1] if i else undef) and right == (nodes[i + 1] if i + 1 < len(nodes) else undef)


def test_many_groups_read_by_h5py(tmp_path):
    h5py = pytest.importorskip('h5py')
    path, tree = many_groups(tmp_path, 1500)
    with h5py.File(path, 'r') as f:
        assert sorted(f.keys()) == sorted(tree)
        assert all(np.array_equal(f[k]['f2o_start'][:], v['f2o_start']) and f[k].attrs['offset'] == -2.0 for k, v in tree.items())


def test_existing_writer_output_unchanged(tmp_path):
    """String-only attributes and <= 256 links: the bytes the writer produced before numeric attributes and two-level trees."""
    path = str(tmp_path / 'small.hdf5')
    artifacts.write_hdf5(path, {'7': {'start': np.arange(6, dtype=np.int8).reshape(2, 3)}}, attrs={'7': {'context': 'c', 'title': 't'}})
    assert hashlib.sha256(open(path, 'rb').read()).hexdigest()[:16] == WRITER_DIGEST


WRITER_DIGEST = 'd4a31fc7afaef0b1'          # sha256 prefix of the parent commit's writer output


def test_dump_flags_have_reference_defaults():
    from densephrases_b200.options import Options
    o = Options()
    o.add_model_options()
    o.add_data_options()
    o.add_rc_options()
    a = o.parse([])
    assert (a.predict_file, a.append_title, a.per_gpu_eval_batch_size, a.do_dump, a.filter_only, a.filter_threshold,
            a.dense_offset, a.dense_scale) == (None, False, 12, False, False, -1e8, -2, 20)
    a = o.parse(['--predict_file', 'x:y', '--append_title', '--do_dump', '--filter_only', '--filter_threshold', '-2.0'])
    assert (a.predict_file, a.append_title, a.do_dump, a.filter_only, a.filter_threshold) == ('x:y', True, True, True, -2.0)
