"""GPU: the phrase dump's device step (csrc/dump.cu) against the oracle and the unmodified reference, across forward-batch
boundaries, and dump_phrases end to end on the GPU encoder's own outputs."""
import argparse
import json
import os

import numpy as np
import pytest
import torch

from densephrases_b200 import dump
from oracle import dump_ref
from tests import dump_cases
from tests.test_dump_cpu import CASES, G, RUNS, build, check_groups, oracle_groups

pytestmark = pytest.mark.gpu


def outputs(start, logits, batch):
    for b0 in range(0, len(start), batch):
        yield b0, torch.from_numpy(start[b0:b0 + batch]).cuda(), torch.from_numpy(np.ascontiguousarray(logits[b0:b0 + batch])).cuda()


def same(a, b):
    assert sorted(a) == sorted(b)
    for did in a:
        (da, aa), (db, ab) = a[did], b[did]
        assert sorted(da) == sorted(db) and aa == ab, did
        for k in da:
            assert da[k].dtype == db[k].dtype and da[k].shape == db[k].shape and da[k].tobytes() == db[k].tobytes(), f'{did}/{k}'


@pytest.mark.parametrize('batch', [1, 3, 16])
@pytest.mark.parametrize('name,thr', RUNS)
def test_device_select_matches_oracle_and_reference(name, thr, batch):
    _, S, stride, title, L, thrs, off, scale, seed = CASES[name]
    tok, examples, features, toffs, start, logits = build(name)
    got = dump.dump_documents(examples, features, outputs(start, logits, batch), tok, L, False, thr, off, scale, title)
    same(got, oracle_groups(name, thr))
    check_groups(got, next(r for c in G['cases'] if c['name'] == name for r in c['runs'] if r['filter_threshold'] == thr)['groups'])


def test_filter_only_matches_reference():
    name = dump_cases.FILTER_ONLY_CASE
    _, S, stride, title, L, thrs, off, scale, seed = CASES[name]
    tok, examples, features, toffs, start, logits = build(name)
    got = dump.dump_documents(examples, features, outputs(start, logits, 5), tok, None, False, -1e8, off, scale, title, filter_only=True)
    check_groups(got, next(c for c in G['cases'] if c['name'] == name)['filter_only'])


def test_random_batches_cross_documents():
    """Random features (one document longer than a batch, documents ending mid-batch), random fp32 rows, each batch size."""
    rng = np.random.default_rng(7)
    S, L = 96, 12
    lens = [40, 3, 1, 17, 2, 5]                              # features per document
    lo = rng.integers(1, 12, sum(lens))
    hi = np.minimum(S - 1, lo + rng.integers(0, 80, sum(lens)))
    doc_of = np.repeat(np.arange(len(lens)), lens)
    start = rng.standard_normal((sum(lens), S, 768)).astype(np.float32) * 4
    filt = rng.standard_normal((sum(lens), S, 2)).astype(np.float32)
    filt[doc_of == 4] = -3.0
    for B in (1, 3, 16):
        sel = dump.DumpSelect(L, -0.5, -2.0, 20.0)
        kept = {d: 0 for d in range(len(lens))}
        rows = {d: 0 for d in range(len(lens))}
        got = {d: ([], [], []) for d in range(len(lens))}
        fb = {}
        for b0 in range(0, sum(lens), B):
            idx = np.arange(b0, min(b0 + B, sum(lens)))
            g0 = doc_of[idx[0]]
            n_doc = doc_of[idx[-1]] - g0 + 1
            doc = np.array([(kept[g0 + s], int(kept[g0 + s] == 0 and (g0 + s) not in fb)) for s in range(n_doc)], np.int32)
            feat = np.zeros((len(idx), 4), np.int32)
            for k, i in enumerate(idx):
                feat[k] = (lo[i], hi[i], doc_of[i] - g0, rows[doc_of[i]])
                rows[doc_of[i]] += hi[i] - lo[i]
            r = sel(torch.from_numpy(start[idx]).cuda(), torch.from_numpy(filt[idx]).cuda(), feat, doc)
            at = 0
            for s in range(n_doc):
                n = int(r['doc_kept'][s])
                for lst, key in zip(got[g0 + s], ('rows', 'f2o', 'start2end')):
                    lst.append(r[key][at:at + n])
                at += n
                kept[g0 + s] += n
                if doc[s, 1] and r['fb_f2o'][s] >= 0:
                    fb[g0 + s] = (r['fb_rows'][r['fb_slot'][s]], r['fb_f2o'][s])
        for d in range(len(lens)):
            ii = np.flatnonzero(doc_of == d)
            cat = lambda a: np.concatenate([a[i, lo[i]:hi[i]] for i in ii])          # noqa: E731
            q, f2o, s2e = dump_ref.select_document(cat(start), cat(filt[..., 0]), cat(filt[..., 1]), hi[ii] - lo[ii], L, -0.5, -2.0, 20.0)
            if kept[d]:
                assert np.array_equal(np.concatenate(got[d][0]), q) and np.array_equal(np.concatenate(got[d][1]), f2o)
                assert np.array_equal(np.concatenate(got[d][2]), s2e), (B, d)
            else:
                assert d == 4 and np.array_equal(fb[d][0][None], q) and [fb[d][1]] == f2o.tolist(), (B, d)


def gpu_dump(tmp_path):
    """dump_phrases of the golden documents on a random-weight phrase tower -> (dump file, encoder, tokenizer)."""
    from densephrases_b200.encoder import BertGeometry, Encoder, random_phrase_state_dict
    tok = dump_cases.tokenizer()
    geo = BertGeometry(vocab_size=max(tok.vocab.values()) + 1)
    enc = Encoder(geo, state_dict=random_phrase_state_dict(geo, 3), device=0, phrase_only=True)
    data_dir = tmp_path / 'data'
    data_dir.mkdir()
    (data_dir / 'dev.json').write_text(json.dumps({'data': G['documents']}))
    args = argparse.Namespace(output_dir=str(tmp_path / 'out'), data_dir=str(data_dir), predict_file='dev.json', max_seq_length=64,
                              doc_stride=20, append_title=True, per_gpu_eval_batch_size=4, max_answer_length=10, do_lower_case=False,
                              filter_threshold=0.0, dense_offset=-2.0, dense_scale=20.0, n_gpu=1)
    return dump.dump_phrases(args, enc, tok), enc, tok


def test_dump_phrases_end_to_end(tmp_path):
    """dump_phrases on the GPU encoder's own outputs == the oracle fed those outputs: every dataset and attribute."""
    path, enc, tok = gpu_dump(tmp_path)
    assert path == os.path.join(str(tmp_path / 'out'), 'dump/phrase/dev.hdf5')
    got = dump.read_dump(path)
    examples = dump.read_examples(G['documents'])
    features = dump.convert_examples_to_features(examples, tok, 64, 20, True)
    toffs = dump.title_offsets(features, tok, True)
    start = np.concatenate([s.cpu().numpy() for _, s, _ in dump.phrase_outputs(enc, features, 4)])
    filt = np.concatenate([f.cpu().numpy() for _, _, f in dump.phrase_outputs(enc, features, 4)])
    for idxs in dump.documents(examples, features):
        lo = [toffs[i] + 1 for i in idxs]
        hi = [len(features[i].tokens) - 1 for i in idxs]
        rows = lambda a: np.concatenate([a[i, l:h] for i, l, h in zip(idxs, lo, hi)])       # noqa: E731
        q, f2o, s2e = dump_ref.select_document(rows(start), rows(filt[..., 0]), rows(filt[..., 1]), np.subtract(hi, lo), 10, 0.0, -2.0, 20.0)
        fl = [features[i] for i in idxs]
        context, w2s, w2e = dump.document_offsets(examples, fl, [toffs[i] for i in idxs], False, tok)
        ex = examples[fl[-1].example_index]
        ds, attrs = got[str(ex.doc_idx)]
        want = {'start': q, 'len_per_para': np.subtract(hi, lo).astype(np.int64), 'start2end': s2e, 'word2char_start': w2s,
                'word2char_end': w2e, 'f2o_start': f2o}
        assert sorted(ds) == sorted(want)
        for k, v in want.items():
            assert ds[k].dtype == v.dtype and ds[k].shape == v.shape and ds[k].tobytes() == v.tobytes(), k
        assert attrs == {'context': context, 'title': ex.title, 'offset': -2.0, 'scale': 20.0}


class FlatIndex(object):
    """Exact inner-product search over given rows with an identity rotation: the index surface MIPS uses."""

    def __init__(self, x):
        self.x, self.d, self.ntotal, self.nprobe = np.ascontiguousarray(x, np.float32), x.shape[1], len(x), 1

    def search(self, q, k, **_):
        s = np.asarray(q, np.float32) @ self.x.T
        idx = np.argsort(-s, axis=1, kind='stable')[:, :k]
        return np.take_along_axis(s, idx, 1), idx

    def reconstruct_batch(self, ids):
        ids = np.asarray(ids, np.int64)
        ok = (ids >= 0) & (ids < self.ntotal)
        out = np.zeros((len(ids), self.d), np.float32)
        out[ok] = self.x[ids[ok]]
        return out, ok

    def opq_matrix(self):
        return np.eye(self.d, dtype=np.float32)


def test_dumped_phrase_found_through_mips(tmp_path):
    """A file written by dump_phrases, read through MIPS's phrase-dump branch (int8 rows dequantised x / 20 - 2, f2o_start,
    word2char_*, the ' [PAR] ' context): a query built from a kept row returns that phrase, at the offsets the dump gives."""
    from densephrases_b200.mips import MIPS
    from densephrases_b200.phrase_dump import PhraseDump
    path, _, _ = gpu_dump(tmp_path)
    groups = dump.read_dump(path)
    dids = sorted(groups, key=int)
    rows = np.concatenate([groups[d][0]['start'].astype(np.float64) / 20.0 - 2.0 for d in dids]).astype(np.float32)
    doc = np.concatenate([np.full(len(groups[d][0]['start']), int(d), np.int64) for d in dids])
    word = np.concatenate([np.arange(len(groups[d][0]['start']), dtype=np.int64) for d in dids])
    r = int(np.argmax((rows.astype(np.float64) ** 2).sum(1)))        # the longest row is its own best inner product
    mips = MIPS.from_components(FlatIndex(rows), {'0': {'doc': doc, 'word': word}}, None, cuda=True,
                                phrase_dump=PhraseDump(os.path.dirname(path)))
    best = mips.search(np.concatenate([rows[r], rows[r]])[None], q_texts=['q'], top_k=5)[0][0]
    ds, attrs = groups[str(doc[r])]
    w2s, w2e, f2o, context = ds['word2char_start'], ds['word2char_end'], ds['f2o_start'], attrs['context']
    assert (best['doc_idx'], best['start_idx'], best['end_idx']) == (doc[r], word[r], word[r])
    c0, c1 = int(w2s[f2o[word[r]]]), int(w2e[f2o[word[r]]])
    assert c1 > c0 and best['answer'] == context[c0:c1]
    assert best['context'] in context and best['context'][best['start_pos']:best['end_pos']] == best['answer']
    assert best['title'] == [attrs['title']]
