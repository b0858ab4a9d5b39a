"""Single-passage reading on the GPU at its limits: the read logits of dph_encoder_read against an fp64 truth, the read path's
workspace across calls, and the span decoder dph_rc_spans at its bounds.

Read logits.  Truth: tests/rc_ref_torch.read in fp64 on the four stressed weight sets of tests/test_encoder_limits_gpu.py.  A start
or end logit is x . q (x a token vector, q its question's vector), so it carries the error bars of both vectors:
  |d| <= bar * (s_x * ||q||_1 + s_q * ||x||_1),   s_x, s_q = max(1, max |ref|) of each fp64 vector,
bar the encoder-limits bar of the mode and weight kind, with the same ill-conditioned escape (torch fp32's own error on the logit,
in the same units, over ILL: within ILL_FACTOR of it).  Filter logits keep their encoder-limits bar.  Independent of the towers,
each logit equals the fp64 dot product of the GPU's own return_phrase=True row with the GPU's own embed_query vector within
768 * 2^-24 * sum |x_i q_i|, and the filter logits are bit-identical to return_phrase=True.

Span decoder.  The edge cases of tests/test_rc_limits_cpu.py (each checked there to reach what it claims, and the oracle checked
there against a plain statement of the reference) against oracle/rc_ref.py, exactly, from host and from device buffers; the 32-bit
span index at its edge; compute_predictions_logits past 1024 candidates against tests/golden/rc_limits.json.gz."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.helpers import stressed_state_dict
from tests.test_encoder_limits_gpu import BAR, ILL, ILL_FACTOR, MASKS, MODES, TF32_STRESSED, VOCAB, make_mask, tokens
from tests.test_rc_gpu import same_spans
from tests.test_rc_limits_cpu import DECODER_CASES, HOST_FINISH, LIMIT_RUNS, limit_run

pytestmark = pytest.mark.gpu
SEED = 11
# (B, S, Sq): every S of the phrase limits and every Sq of the question limits, with Sq > S and S > Sq
READ_SHAPES = [(1, 1, 384), (3, 2, 1), (1, 63, 65), (3, 64, 64), (1, 65, 2), (3, 384, 1), (1, 385, 65), (3, 512, 384)]


@pytest.fixture(autouse=True)
def _fp32_matmuls():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def read_mem(enc, t, host):
    """dph_encoder_read from host tensors (MEM_HOST) or CUDA tensors (MEM_DEVICE) -> (start, end, filter_start, filter_end) on the CPU."""
    from densephrases_b200 import _lib as L
    dev = 'cpu' if host else 'cuda'
    ids, mask, tt, qids, qmask, qtt = (x.to(dev).contiguous() for x in t)
    B, S = ids.shape
    out = [torch.full((B, S), float('nan'), device=dev), torch.full((B, S), float('nan'), device=dev),
           torch.full((B, S, 2), float('nan'), device=dev)]
    L.check(L.lib().dph_encoder_set_stream(enc._h, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    L.check(L.lib().dph_encoder_read(enc._h, ids.data_ptr(), mask.data_ptr(), tt.data_ptr(), B, S, qids.data_ptr(), qmask.data_ptr(),
                                     qtt.data_ptr(), int(qids.shape[1]), *(o.data_ptr() for o in out), L.MEM_HOST if host else L.MEM_DEVICE))
    torch.cuda.synchronize()
    return tuple(x.cpu() for x in (out[0], out[1], out[2][..., 0], out[2][..., 1]))


def read_inputs(B, S, Sq, mask_kind, seed):
    ids, mask, tt = tokens(B, S, make_mask(mask_kind, B, S), seed, True)
    qids, qmask, qtt = tokens(B, Sq, make_mask(mask_kind, B, Sq), seed + 1, False)
    return ids, mask, tt, qids, qmask, qtt


@pytest.fixture(scope='module', params=('sharp', 'outlier', 'tails', 'all'))
def stressed(request):
    from densephrases_b200.encoder import BertGeometry, Encoder
    geo = BertGeometry(vocab_size=VOCAB)
    sd = stressed_state_dict(geo, SEED, request.param)
    yield request.param, Encoder(geo, state_dict=sd), {k: v.cuda().double() for k, v in sd.items()}, {k: v.cuda() for k, v in sd.items()}
    torch.cuda.empty_cache()


@pytest.mark.parametrize('B,S,Sq', READ_SHAPES)
def test_read_logits_against_fp64(stressed, B, S, Sq):
    """Every mode, both attention settings where the phrase tower has both (S <= 384), every mask; host and device buffers take
    turns over the masks."""
    from oracle import encoder_ref
    from tests import phrase_ref, rc_ref_torch
    kind, enc, sd64, sd32 = stressed
    wnorm = max(1.0, sd64['filter_linear.weight'].norm(dim=1).max().item())
    bad = []
    try:
        for mi, mask_kind in enumerate(MASKS):
            t = read_inputs(B, S, Sq, mask_kind, B * 1000 + S + 7 * Sq)
            ref = rc_ref_torch.read(sd64, *t, dtype=torch.float64)
            ref32 = rc_ref_torch.read(sd32, *t)
            x = phrase_ref.embed_phrase(sd64, *t[:3], dtype=torch.float64)[0]                       # [B,S,768]
            x32 = phrase_ref.embed_phrase(sd32, *t[:3])[0]
            qs = encoder_ref.embed_query(sd64, *t[3:], dtype=torch.float64)                          # 2 x [B,1,768]
            s_x, n_x = x.abs().amax(-1).clamp_min(1.0), x.abs().sum(-1)                              # [B,S]
            unit = [s_x * q.abs().sum(-1) + q.abs().amax(-1).clamp_min(1.0) * n_x for q in qs]        # [B,S] per logit
            fscale = s_x * wnorm
            f32err = (x32.double() - x).abs().amax(-1) / s_x                                         # torch fp32 per token vector
            for mode in MODES:
                for tc in ([True, False] if S <= 384 else [True]):
                    enc.set_precision(mode)
                    enc.set_attention(tc)
                    got = read_mem(enc, t, host=mi % 2 == 1)
                    bar = TF32_STRESSED.get(kind, (BAR['tf32'],))[0] if mode == 'tf32' else BAR[mode]
                    worst = []
                    for k in range(4):
                        g, r, r32 = got[k].cuda().double(), ref[k].double(), ref32[k].double()
                        u = unit[k] if k < 2 else fscale
                        d, d32 = (g - r).abs() / u, (r32 - r).abs() / u if k < 2 else f32err
                        ok = torch.isfinite(g) & ((d <= bar) | ((d32 > ILL) & (d <= ILL_FACTOR[mode] * d32)))
                        worst.append(d.max().item())
                        if not bool(ok.all()):
                            bad.append((mode, tc, mask_kind, ('start', 'end', 'fs', 'fe')[k], d.max().item()))
                    print(f"LIMITS read {kind} {mode} tc={int(tc)} B={B} S={S} Sq={Sq} {mask_kind}: max|d|/unit "
                          f"{' '.join(f'{w:.2e}' for w in worst)} (bar {bar:.0e})")
    finally:
        enc.set_precision('bf16x3')
        enc.set_attention(True)
    assert not bad, f'read {kind} B={B} S={S} Sq={Sq}: over the bar in {bad}'


@pytest.mark.parametrize('B,S,Sq', READ_SHAPES)
def test_read_logits_are_dot_products_of_own_vectors(B, S, Sq):
    """Independent of the towers: each logit == fp64 x . q of the GPU's own phrase row and question vector, within
    768 * 2^-24 * sum |x_i q_i| (padding positions included); filter logits bit-identical to return_phrase=True."""
    enc, _ = random_encoder()
    bad = []
    try:
        for mode in MODES:
            for tc in ([True, False] if S <= 384 else [True]):
                enc.set_precision(mode)
                enc.set_attention(tc)
                for mi, mask_kind in enumerate(MASKS):
                    t = read_inputs(B, S, Sq, mask_kind, 77 + B + S + Sq)
                    got = read_mem(enc, t, host=mi % 2 == 0)
                    x, _, fs, fe = enc(input_ids=t[0], attention_mask=t[1], token_type_ids=t[2], return_phrase=True)
                    for k, q in enumerate(enc.embed_query(*t[3:])):
                        prod = x.double() * q.double()                                     # [B,S,768]
                        d = (got[k].cuda().double() - prod.sum(-1)).abs()
                        if not bool((d <= 768 * 2.0 ** -24 * prod.abs().sum(-1)).all()):
                            bad.append((mode, tc, mask_kind, k, d.max().item()))
                    if not (torch.equal(got[2], fs.cpu()) and torch.equal(got[3], fe.cpu())):
                        bad.append((mode, tc, mask_kind, 'filter logits differ from return_phrase=True'))
    finally:
        enc.set_precision('bf16x3')
        enc.set_attention(True)
    assert not bad, bad


# ---- the read path's workspace across calls ----------------------------------------------------------------------------------
_SD = {}


def random_encoder():
    from densephrases_b200.encoder import BertGeometry, Encoder
    from tests import rc_ref_torch
    geo = BertGeometry(vocab_size=VOCAB)
    if not _SD:
        _SD['sd'] = rc_ref_torch.rc_state_dict(geo, 5)
    return Encoder(geo, state_dict=_SD['sd']), _SD['sd']


def fresh_read(t, mode):
    enc, _ = random_encoder()
    enc.set_precision(mode)
    out = read_mem(enc, t, host=False)
    del enc
    return out


def same(a, b, what):
    for x, y, k in zip(a, b, ('start', 'end', 'filter_start', 'filter_end')):
        assert torch.equal(x, y), f'{what}: {k} differs'


@pytest.mark.parametrize('mode', ['bf16x3', 'tf32'])
def test_read_workspace_across_calls(mode):
    """One encoder through B = 1 -> 257 -> 2 -> 257 (the question buffer regrows and then holds stale rows), with embed_query and
    return_phrase=True calls in between, and the first-call shapes Sq = 384 with S = 1 and Sq = 1 with S = 512: every read
    bit-identical to a fresh encoder's, and host buffers bit-identical to device buffers."""
    calls = [(1, 48, 16, 'suffix', 1), (257, 24, 9, 'holes', 2), (2, 40, 33, 'ones', 3), (257, 24, 9, 'suffix', 4)]
    want = [fresh_read(read_inputs(B, S, Sq, m, seed), mode) for B, S, Sq, m, seed in calls]
    enc, _ = random_encoder()
    enc.set_precision(mode)
    for i, ((B, S, Sq, m, seed), w) in enumerate(zip(calls, want)):
        t = read_inputs(B, S, Sq, m, seed)
        same(read_mem(enc, t, host=False), w, f'call {i} B={B}')
        enc.embed_query(*read_inputs(3, 70, 70, 'ones', 90 + i)[3:])
        enc(*read_inputs(5, 100, 2, 'holes', 95 + i)[:3], return_phrase=True)
        same(read_mem(enc, t, host=True), w, f'call {i} B={B}, host buffers, after embed_query and return_phrase')
    for S, Sq in ((1, 384), (512, 1)):
        t = read_inputs(2, S, Sq, 'suffix', S + Sq)
        first = fresh_read(t, mode)
        same(read_mem(enc, t, host=False), first, f'S={S} Sq={Sq} after other shapes')
        same(read_mem(enc, t, host=True), first, f'S={S} Sq={Sq} host buffers')
    del enc


# ---- the span decoder at its bounds ------------------------------------------------------------------------------------------
def decode(c, device):
    from densephrases_b200 import rc
    arrays = c['logits'] + [c['n_tokens'], c['start_ok'].view(np.int32), c['end_ok'].view(np.int32), c['ex_off']]
    if device:
        arrays = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    return rc.best_spans(*arrays, c['L'], c['thr'], c['K'], c['v2'])


@pytest.mark.parametrize('name', list(DECODER_CASES))
def test_decoder_edge_cases_match_oracle(name):
    from tests.test_rc_limits_cpu import oracle_spans
    c = DECODER_CASES[name]
    ref = oracle_spans(c)
    for device in (False, True):
        same_spans(decode(c, device), ref)


def test_decoder_span_index_at_32_bits():
    """One example of 131 071 features at S = 512 (features * S * 64 = 2^32 - 2^15): only the last three have tokens, so the
    enumeration index of their spans sits at the top of the 32-bit range.  131 072 features are rejected."""
    from densephrases_b200 import rc
    from oracle import rc_ref
    F, S, tail = 131071, 512, 3
    assert F * S * 64 == 2 ** 32 - 2 ** 15
    g = torch.Generator(device='cuda').manual_seed(3)
    lg = [torch.randn((F + 1, S), generator=g, device='cuda') for _ in range(4)]
    lg[0][:, 0] = torch.arange(F + 1, device='cuda', dtype=torch.float32) % 1000 + 10.0
    lg[0][70000, 0] = -50.0                                                          # the smallest start[0] + end[0]
    lg[1][:, 0] = 0.5
    lg[0][F - 1, 1:] += 100.0                                                        # the best spans are in the last feature
    n_tokens = torch.zeros(F + 1, dtype=torch.int32, device='cuda')
    n_tokens[F - tail:F] = torch.tensor([S, 1, S - 5], dtype=torch.int32)
    ok = torch.full((F + 1, S // 32), -1, dtype=torch.int32, device='cuda')
    args = lambda n: ([x[:n] for x in lg] + [n_tokens[:n], ok[:n], ok[:n], torch.tensor([0, n], dtype=torch.int64, device='cuda')])   # noqa: E731
    got = rc.best_spans(*args(F), 64, -0.5, 1024, True)
    a = F - tail
    tail_ref = rc_ref.best_spans(*(x[a:F].cpu().numpy() for x in lg), n_tokens[a:F].cpu().numpy(), ok[a:F].cpu().numpy(),
                                 ok[a:F].cpu().numpy(), np.array([0, tail], np.int64), 64, -0.5, 1024, False)
    tail_ref.cand[0, :, 0] += a
    assert int(tail_ref.n_cand[0]) == 1024 and (tail_ref.cand[0, :, 0] == F - 1).all()
    for k in ('n_cand', 'total_count', 'vec_count'):
        assert np.array_equal(getattr(got, k), getattr(tail_ref, k)), k
    assert np.array_equal(got.cand[0], tail_ref.cand[0])
    assert int(got.null_feature[0]) == 70000 and got.null_logits[0].tolist() == [-50.0, 0.5]
    with pytest.raises(RuntimeError, match='32 bits'):
        rc.best_spans(*args(F + 1), 64, -0.5, 1024, True)


@pytest.mark.parametrize('name,thr', LIMIT_RUNS)
def test_nbest_beyond_1024_candidates_on_gpu_decoder(name, thr, tmp_path, monkeypatch):
    """compute_predictions_logits on the GPU decoder reproduces the reference past 1024 candidates (host finish)."""
    from densephrases_b200 import rc
    host, host_spans = [], rc.host_spans
    monkeypatch.setattr(rc, 'host_spans', lambda *a: host.append(1) or host_spans(*a))
    case, run, (preds, stat, files) = limit_run(rc, name, thr, str(tmp_path))
    assert preds == run['predictions'] and stat == run['stat'] and files == run['files']
    if thr < -1e7:
        assert bool(host) == HOST_FINISH[name]
