"""Single-passage reading on the GPU: Encoder.forward with a context and a question (dph_encoder_read) and the span decoder
(dph_rc_spans) behind compute_predictions_logits.

Oracle chain: the unmodified reference (tests/golden/make_rc_golden.py) -> fixtures encoder_rc.npz / rc_reference.json.gz -> (CPU,
tests/test_rc_cpu.py) the torch restatement tests/rc_ref_torch.py and the numpy span oracle oracle/rc_ref.py reproduce them ->
(here) the CUDA paths against both."""
import os

import numpy as np
import pytest
import torch

from tests import rc_cases
from tests.test_phrase_encoder import TOL

pytestmark = pytest.mark.gpu
GOLD_ENC = os.path.join(os.path.dirname(__file__), 'golden', 'encoder_rc.npz')
ENC_CASES = ('b3_s48_q16', 'b2_s160_q32')
_ENC = {}


def encoder_for(vocab, seed):
    from densephrases_b200.encoder import BertGeometry, Encoder
    from tests import rc_ref_torch
    key = (vocab, seed)
    if key not in _ENC:
        _ENC.clear()
        geo = BertGeometry(vocab_size=vocab)
        sd = rc_ref_torch.rc_state_dict(geo, seed)
        _ENC[key] = (Encoder(geo, state_dict=sd), sd)
    enc, sd = _ENC[key]
    enc.set_precision('bf16x3')
    return enc, sd


def read(enc, t):
    return enc(input_ids=t['ids'], attention_mask=t['mask'], token_type_ids=t['tt'], input_ids_=t['qids'], attention_mask_=t['qmask'],
               token_type_ids_=t['qtt'])


def check_logits(mode, got, ref, what):
    """start / end: max|diff| <= TOL[mode] * max|ref logit|; filter logits: the absolute bars of the phrase path."""
    for x, r, k in zip(got, ref, ('start', 'end', 'filter_start', 'filter_end')):
        x, r = x.float().cpu(), r.float().cpu()
        assert x.shape == r.shape and torch.isfinite(x).all()
        d = (x - r).abs().max().item()
        bar = TOL[mode] * (r.abs().max().item() if k in ('start', 'end') else 1.0)
        print(f'{what} {mode} {k}: max|diff| {d:.2e} (bar {bar:.2e})')
        assert d <= bar, (what, mode, k, d, bar)


def random_batch(B, S, Sq, vocab, seed):
    from densephrases_b200.encoder import synthetic_context_batch, synthetic_query_batch
    ids, mask, tt = synthetic_context_batch(B, S, vocab, seed, type_split=True)
    qids, qmask, qtt = synthetic_query_batch(B, Sq, vocab, seed + 1)
    return dict(ids=ids, mask=mask, tt=tt, qids=qids, qmask=qmask, qtt=qtt)


# (a)
@pytest.mark.parametrize('mode', ['tf32', '3xtf32', 'bf16x3'])
@pytest.mark.parametrize('name', ENC_CASES)
def test_read_matches_reference_fixture(name, mode):
    g = np.load(GOLD_ENC)
    enc, _ = encoder_for(int(g['vocab']), int(g['seed']))
    enc.set_precision(mode)
    t = {k: torch.from_numpy(g[f'{name}_{k}']) for k in ('ids', 'mask', 'tt', 'qids', 'qmask', 'qtt')}
    got = read(enc, t)
    B, S = t['ids'].shape
    assert all(x.shape == (B, S) and x.dtype == torch.float32 and x.device.type == 'cuda' for x in got)
    check_logits(mode, got, [torch.from_numpy(g[f'{name}_{k}']) for k in ('start', 'end', 'filter_start', 'filter_end')], name)


# (b)
def test_read_full_batch_against_torch_fp32():
    from tests import rc_ref_torch
    enc, sd = encoder_for(2000, 11)
    t = random_batch(32, 384, 64, 2000, 12)
    torch.backends.cuda.matmul.allow_tf32 = False
    ref = rc_ref_torch.read({n: w.cuda() for n, w in sd.items()}, *(t[k].cuda() for k in ('ids', 'mask', 'tt', 'qids', 'qmask', 'qtt')))
    for mode in ('tf32', '3xtf32', 'bf16x3'):
        enc.set_precision(mode)
        check_logits(mode, read(enc, t), ref, 'B32 S384 Sq64')


# (c)
@pytest.mark.parametrize('mode', ['tf32', 'bf16x3'])
def test_read_invariants(mode):
    enc, _ = encoder_for(2000, 11)
    enc.set_precision(mode)
    t = random_batch(6, 200, 24, 2000, 13)
    s, e, fs, fe = read(enc, t)
    x, _, pfs, pfe = enc(input_ids=t['ids'], attention_mask=t['mask'], token_type_ids=t['tt'], return_phrase=True)
    assert torch.equal(fs, pfs) and torch.equal(fe, pfe), 'filter logits must be bit-identical to return_phrase=True'
    qs, qe = enc.embed_query(t['qids'], t['qmask'], t['qtt'])
    for got, q in ((s, qs), (e, qe)):
        ref = x.double().matmul(q.double().transpose(1, 2)).squeeze(-1)
        assert (got.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    again = read(enc, t)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())          # one encoder's workspace serves one stream at a time
    with torch.cuda.stream(side):
        other = read(enc, t)
    torch.cuda.synchronize()
    for a, b, c in zip((s, e, fs, fe), again, other):
        assert torch.equal(a, b) and torch.equal(a, c), 'repeated calls must give identical bits'


# (d)
def decoder_inputs(F_per_ex, S, seed, ties):
    rng = np.random.default_rng(seed)
    F = int(sum(F_per_ex))
    if ties:
        logits = [(np.round(rng.normal(size=(F, S)) * 2.0) / 2.0).astype(np.float32) for _ in range(4)]
    else:
        logits = [rng.normal(size=(F, S)).astype(np.float32) * 4 for _ in range(4)]
    n_tokens = rng.integers(S // 2, S + 1, F).astype(np.int32)
    n_tokens[0] = S
    W = (S + 31) // 32
    start_ok = rng.integers(0, 2 ** 32, (F, W), dtype=np.uint64).astype(np.uint32) | np.uint32(0x7fff7ffe)
    end_ok = start_ok | rng.integers(0, 2 ** 32, (F, W), dtype=np.uint64).astype(np.uint32)
    ex_off = np.concatenate([[0], np.cumsum(F_per_ex)]).astype(np.int64)
    return logits, n_tokens, start_ok, end_ok, ex_off


def same_spans(a, b):
    for k in ('n_cand', 'total_count', 'vec_count', 'null_feature'):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    assert np.array_equal(a.null_logits.view(np.int32), b.null_logits.view(np.int32))
    for x in range(len(a.n_cand)):
        n = int(a.n_cand[x])
        assert np.array_equal(a.cand[x, :n], b.cand[x, :n]), f'example {x}: candidates differ'


@pytest.mark.parametrize('S,L,K,thr,ties,v2', [(512, 64, 1024, -1.0, False, True), (512, 64, 1024, 0.0, True, False),
                                               (384, 10, 20, -2.0, True, True), (100, 30, 7, -1e8, True, False), (48, 1, 5, -1e8, False, True)])
def test_decoder_matches_oracle(S, L, K, thr, ties, v2):
    from densephrases_b200 import rc
    from oracle import rc_ref
    per_ex = [1, 3, 2, 4, 1, 2]
    logits, n_tokens, start_ok, end_ok, ex_off = decoder_inputs(per_ex, S, S + L + K, ties)
    ref = rc_ref.best_spans(*logits, n_tokens, start_ok, end_ok, ex_off, L, thr, K, v2)
    host = rc.best_spans(*logits, n_tokens, start_ok, end_ok, ex_off, L, thr, K, v2)
    same_spans(host, ref)
    dev = rc.best_spans(*(torch.from_numpy(x).cuda() for x in logits), torch.from_numpy(n_tokens).cuda(),
                        torch.from_numpy(start_ok.view(np.int32)).cuda(), torch.from_numpy(end_ok.view(np.int32)).cuda(),
                        torch.from_numpy(ex_off).cuda(), L, thr, K, v2)
    same_spans(dev, ref)
    if L > 1 and thr < 0:
        assert (ref.vec_count > K).any() or K > 100, 'the cut to K must be exercised'


def test_decoder_on_gpu_logits_matches_oracle():
    from densephrases_b200 import rc
    from oracle import rc_ref
    enc, _ = encoder_for(2000, 11)
    t = random_batch(12, 384, 32, 2000, 21)
    logits = [x.contiguous() for x in read(enc, t)]
    n_tokens = t['mask'].sum(1).to(torch.int32)
    W = 12
    start_ok = torch.full((12, W), -1, dtype=torch.int32)
    start_ok[:, 0] = -2                                       # [CLS] cannot start a span
    ex_off = torch.tensor([0, 1, 4, 6, 10, 12], dtype=torch.int64)
    ref = rc_ref.best_spans(*(x.cpu().numpy() for x in logits), n_tokens.numpy(), start_ok.numpy(), start_ok.numpy(), ex_off.numpy(), 10,
                            -0.5, 20, True)
    got = rc.best_spans(*logits, n_tokens.cuda(), start_ok.cuda(), start_ok.cuda(), ex_off.cuda(), 10, -0.5, 20, True)
    same_spans(got, ref)


# (e)
@pytest.mark.parametrize('name', [c['name'] for c in rc_cases.load_cases() if c['name'] != 'no_valid_span'])
def test_predictions_on_gpu_logits_equal_oracle_run(name, tmp_path, monkeypatch):
    from densephrases_b200 import rc
    from oracle import rc_ref
    case = next(c for c in rc_cases.load_cases() if c['name'] == name)
    _, features, gold_logits = rc_cases.objects(case)
    enc, _ = encoder_for(2000, 11)
    t = random_batch(len(features), case['S'], 16, 2000, 31)
    gpu_logits = tuple(read(enc, t))
    for logits, label in ((gpu_logits, 'gpu'), (tuple(torch.from_numpy(x).cuda() for x in gold_logits), 'gold')):
        for r in case['runs']:
            thr = r['filter_threshold']
            for d in ('gpu', 'ref'):
                os.makedirs(tmp_path / f'{label}_{d}', exist_ok=True)
            got = rc_cases.run(rc, case, thr, str(tmp_path / f'{label}_gpu'), logits)
            with monkeypatch.context() as m:
                m.setattr(rc, 'best_spans', rc_ref.best_spans)
                want = rc_cases.run(rc, case, thr, str(tmp_path / f'{label}_ref'), tuple(x.cpu() for x in logits))
            assert got[0] == want[0] and got[1] == want[1] and got[2] == want[2], (name, label, thr)
            if label == 'gold':
                assert got[0] == r['predictions'] and got[1] == r['stat'] and got[2] == r['files']


def test_filter_test_one_forward():
    from densephrases_b200 import rc
    case = next(c for c in rc_cases.load_cases() if c['name'] == 'squad_v1')
    examples, features, _ = rc_cases.objects(case)
    enc, _ = encoder_for(2000, 11)
    t = random_batch(len(features), case['S'], 16, 2000, 41)
    for i, f in enumerate(features):
        for k, n in (('ids', 'input_ids'), ('mask', 'attention_mask'), ('tt', 'token_type_ids'), ('qids', 'input_ids_'),
                     ('qmask', 'attention_mask_'), ('qtt', 'token_type_ids_')):
            setattr(f, n, t[k][i].tolist())
    res = rc.filter_test(enc, examples, features, rc_cases.JoinTokenizer(), batch_size=7)
    assert list(res) == [f'{m}_{thr:.2f}' for thr in rc.FILTER_TEST_THRESHOLDS for m in ('exact', 'f1', 'save_rate')]
    logits = read(enc, t)
    for thr in (-4.0, 0.0):
        preds, stat = rc.compute_predictions_logits(examples, features, logits, 20, 10, False, None, None, None, False, False, 0.0,
                                                    rc_cases.JoinTokenizer(), thr, None)
        ev = rc.squad_evaluate(examples, preds)
        assert res[f'exact_{thr:.2f}'] == ev['exact'] and res[f'f1_{thr:.2f}'] == ev['f1'] and res[f'save_rate_{thr:.2f}'] == stat['save_rate']


# (f)
def test_errors():
    from densephrases_b200 import rc
    from densephrases_b200.encoder import BertGeometry, Encoder, random_phrase_state_dict, random_state_dict
    enc, _ = encoder_for(2000, 11)
    t = random_batch(2, 64, 16, 2000, 51)
    with pytest.raises(ValueError):
        enc(input_ids=t['ids'], input_ids_=t['qids'][:1], attention_mask_=t['qmask'][:1], token_type_ids_=t['qtt'][:1])
    big = random_batch(1, 513, 385, 2000, 52)
    with pytest.raises(ValueError):
        enc(input_ids=big['ids'], input_ids_=t['qids'][:1], attention_mask_=t['qmask'][:1], token_type_ids_=t['qtt'][:1])
    with pytest.raises(ValueError):
        enc(input_ids=t['ids'][:1], input_ids_=big['qids'], attention_mask_=big['qmask'], token_type_ids_=big['qtt'])
    for kw in ('start_positions', 'end_positions', 'neg_input_ids'):
        with pytest.raises(NotImplementedError):
            enc(input_ids=t['ids'], input_ids_=t['qids'], attention_mask_=t['qmask'], token_type_ids_=t['qtt'], **{kw: torch.zeros(2, dtype=torch.int64)})
    geo = BertGeometry(vocab_size=2000)
    phrase_only = Encoder(geo, state_dict=random_phrase_state_dict(geo, 3), phrase_only=True)
    query_only = Encoder(geo, state_dict=random_state_dict(geo, 3))
    for e in (phrase_only, query_only):
        with pytest.raises(NotImplementedError):
            read(e, t)
    del phrase_only, query_only
    # the device-side id latch: out-of-range ids on the GPU are reported by the next call
    bad = dict(t, ids=t['ids'].clone().cuda())
    bad['ids'][1, 3] = 5000
    read(enc, bad)
    with pytest.raises(RuntimeError, match='outside the embedding tables'):
        read(enc, t)
    read(enc, t)                                                   # the latch is cleared once reported
    bad = dict(t, qids=t['qids'].clone().cuda())
    bad['qids'][0, 1] = -1
    read(enc, bad)
    with pytest.raises(RuntimeError, match='outside the embedding tables'):
        read(enc, t)
    with pytest.raises(IndexError):                               # host ids are checked before the copy
        read(enc, dict(t, ids=t['ids'].clone().fill_(5000)))
    # decoder bounds
    logits, n_tokens, start_ok, end_ok, ex_off = decoder_inputs([1, 2], 64, 1, False)
    args = lambda **k: dict(dict(zip(('start', 'end', 'sft', 'eft'), logits), n_tokens=n_tokens, start_ok=start_ok, end_ok=end_ok,   # noqa: E731
                                 ex_off=ex_off, max_answer_length=10, filter_threshold=0.0, k=20), **k)
    rc.best_spans(**args())
    for bad_args in (dict(max_answer_length=65), dict(max_answer_length=0), dict(k=1025), dict(k=0), dict(ex_off=np.array([0, 2, 2, 3])),
                     dict(ex_off=np.array([0, 1, 2])), dict(ex_off=np.array([1, 3])), dict(n_tokens=n_tokens + 64)):
        with pytest.raises(RuntimeError):
            rc.best_spans(**args(**bad_args))
    wide = [np.zeros((3, 513), np.float32)] * 4
    with pytest.raises(RuntimeError):
        rc.best_spans(*wide, n_tokens, np.zeros((3, 17), np.uint32), np.zeros((3, 17), np.uint32), ex_off, 10, 0.0, 20)
    with pytest.raises(ValueError):
        rc.best_spans(**args(end=logits[1][:2]))
    empty = np.zeros((0, 64), np.float32)
    with pytest.raises(RuntimeError):
        rc.best_spans(empty, empty, empty, empty, n_tokens[:0], start_ok[:0], end_ok[:0], np.array([0, 0]), 10, 0.0, 20)
