"""Single-passage reading on the CPU: the span oracle (oracle/rc_ref.py) driving densephrases_b200.rc reproduces the unmodified
reference compute_predictions_logits / squad_evaluate (tests/golden/rc_reference.json.gz) -- predictions, n-best text,
probabilities and logits, the candidates file, null odds, stat and EM/F1 -- byte for byte; the torch restatement of
Encoder.forward with both sides reproduces the reference class (tests/golden/encoder_rc.npz)."""
import os
import types

import numpy as np
import pytest
import torch

from tests import rc_cases

CASES = rc_cases.load_cases()
RUNS = [(c['name'], r['filter_threshold']) for c in CASES for r in c['runs']]


def case_run(name, thr):
    c = next(c for c in CASES if c['name'] == name)
    return c, next(r for r in c['runs'] if r['filter_threshold'] == thr)


@pytest.fixture
def oracle_rc(monkeypatch):
    """densephrases_b200.rc with its GPU decoder replaced by the numpy oracle; counts the decoder calls."""
    from densephrases_b200 import rc
    from oracle import rc_ref
    calls = []

    def spans(*a, **k):
        calls.append(a[-2] if len(a) >= 11 else k.get('k'))
        return rc_ref.best_spans(*a, **k)
    monkeypatch.setattr(rc, 'best_spans', spans)
    return rc, calls


@pytest.mark.parametrize('name,thr', RUNS)
def test_oracle_reproduces_reference_predictions(oracle_rc, tmp_path, name, thr):
    rc, calls = oracle_rc
    case, ref = case_run(name, thr)
    _, features, logits = rc_cases.objects(case)
    if 'error' in ref:
        with pytest.raises(ZeroDivisionError):
            rc_cases.run(rc, case, thr, str(tmp_path), tuple(logits))
        return
    for results in (tuple(logits), iter([types.SimpleNamespace(unique_id=f.unique_id, start_logits=logits[0][i].tolist(),
                                                               end_logits=logits[1][i].tolist(), sft_logits=logits[2][i].tolist(),
                                                               eft_logits=logits[3][i].tolist()) for i, f in enumerate(features)])):
        preds, stat, files = rc_cases.run(rc, case, thr, str(tmp_path), results)
        assert preds == ref['predictions'] and list(preds) == list(ref['predictions'])
        assert stat == ref['stat']
        assert sorted(files) == sorted(ref['files'])
        for k in files:
            assert files[k] == ref['files'][k], f'{name} thr={thr}: {k} file differs from the reference'
        ev = rc.squad_evaluate(rc_cases.objects(case)[0], preds, null_log_odds_file=None if not case['version_2'] else
                               os.path.join(str(tmp_path), f'null_{thr}.json'))
        assert dict(ev) == ref['eval'] and list(ev) == list(ref['eval'])
    if name.startswith('repeat_word') and thr < -1e7:
        assert max(calls) > case['n_best_size'], 'duplicate texts must force a refill with 2K'


def test_golden_covers_the_issue_cases():
    names = {c['name'] for c in CASES}
    assert {'squad_v1', 'squad_v2', 'squad_v2_null_thr', 'repeat_word', 'no_valid_span'} <= names
    nf = [np.bincount([f['example_index'] for f in c['features']]) for c in CASES]
    assert min(x.min() for x in nf) == 1 and max(x.max() for x in nf) == 4
    runs = [r for c in CASES for r in c['runs'] if 'stat' in r]
    assert any(r['stat']['save_rate'] == 1.0 for r in runs) and any(r['stat']['save_rate'] == 0.0 for r in runs)
    assert os.path.getsize(rc_cases.GOLD) < 2 * 1024 * 1024


def test_feature_masks():
    from densephrases_b200.rc import feature_masks
    f = types.SimpleNamespace(tokens=['[CLS]'] + ['w'] * 40 + ['[SEP]'], token_to_orig_map={i: i - 1 for i in range(1, 41) if i != 33},
                              token_is_max_context={i: i > 5 for i in range(1, 41)})
    n, s_ok, e_ok = feature_masks([f, f], 48)
    assert n.tolist() == [42, 42] and s_ok.shape == (2, 2) and s_ok.dtype == np.uint32
    bits = lambda m: [i for i in range(64) if (int(m[0, i >> 5]) >> (i & 31)) & 1]     # noqa: E731
    assert bits(e_ok) == [i for i in range(1, 41) if i != 33]
    assert bits(s_ok) == [i for i in range(6, 41) if i != 33]


GOLD_ENC = os.path.join(os.path.dirname(__file__), 'golden', 'encoder_rc.npz')


def test_torch_restatement_reproduces_reference_read():
    from densephrases_b200.encoder import BertGeometry
    from tests import rc_ref_torch
    g = np.load(GOLD_ENC)
    sd = rc_ref_torch.rc_state_dict(BertGeometry(vocab_size=int(g['vocab'])), int(g['seed']))
    for name in ('b3_s48_q16', 'b2_s160_q32'):
        t = {k: torch.from_numpy(g[f'{name}_{k}']) for k in ('ids', 'mask', 'tt', 'qids', 'qmask', 'qtt')}
        got = rc_ref_torch.read(sd, t['ids'], t['mask'], t['tt'], t['qids'], t['qmask'], t['qtt'])
        for x, k in zip(got, ('start', 'end', 'filter_start', 'filter_end')):
            ref = torch.from_numpy(g[f'{name}_{k}'])
            assert (x - ref).abs().max() <= 1e-3 * max(1.0, float(ref.abs().max())), (name, k)
    assert os.path.getsize(GOLD_ENC) < 2 * 1024 * 1024
