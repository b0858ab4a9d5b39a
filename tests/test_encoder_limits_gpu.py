"""The encoder at trained-model scales and at its shape edges, against an fp64 truth.

Reference: oracle/encoder_ref.py / tests/phrase_ref.py run with dtype=torch.float64 on the GPU (cuBLAS DGEMM) -- the same code
the fixture tests pin to the unmodified reference class in fp32.  Weights: tests/helpers.stressed_state_dict ('sharp',
'outlier', 'tails', 'all'; test_encoder_limits_cpu.py shows each reaches the statistic it claims).

Bars, per vector (a [CLS] vector of the query path, a token vector of the phrase path), scale = max(1, max |ref| of the vector):
  bf16x3, 3xtf32: max |diff| <= 1e-3 * scale;
  tf32:           max |diff| <= 5e-2 * scale (the bar of tests/test_encoder.py) and cosine > 0.999 on 'sharp' and 'tails';
                  on 'outlier' and 'all' tf32 does not hold that (DESIGN §4.4: up to 0.13 * scale, cosine 0.992), and the bar
                  is 0.2 * scale, cosine > 0.99.
An ill-conditioned vector -- one on which torch fp32 itself is off by more than ILL = 6.25e-5 * scale -- may instead be within
16x (bf16x3, 3xtf32) or 4096x (tf32) torch fp32's own error on it: no fp32-class arithmetic holds 1e-3 there (measured on
'outlier' at S = 385: torch fp32 2.1e-4, bf16x3 1.3e-3, 3xtf32 2.3e-3, tf32 0.34).
The filter logits carry the bar of their token's vector through the head: |diff| <= bar * scale * max(1, ||w_row||_2).
Every case also prints torch fp32's own error against fp64 (TF32 off), the yardstick; lines starting with LIMITS are the
measurement table of DESIGN §4.4.

The attention kernels alone (dph_attention_bert: 0 SIMT, 1 TF32, 2 bf16 planes) and the GEMM epilogue (dph_gemm_tf32_nt) are
checked at logit and pre-activation ranges random weights never reach."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import STRESS_KINDS, stressed_state_dict

pytestmark = pytest.mark.gpu
VOCAB = 1000
SEED = 11
MODES = ("bf16x3", "3xtf32", "tf32")
BAR = {"bf16x3": 1e-3, "3xtf32": 1e-3, "tf32": 5e-2}
TF32_STRESSED = {"outlier": (0.2, 0.99), "all": (0.2, 0.99)}        # kind -> (tf32 bar, cosine) where 5e-2 / 0.999 do not hold
ILL = 6.25e-5
ILL_FACTOR = {"bf16x3": 16.0, "3xtf32": 16.0, "tf32": 4096.0}
QUERY_SHAPES = [(1, 1), (3, 1), (4, 2), (2, 16), (2, 17), (2, 33), (2, 64), (2, 65), (2, 97), (2, 129), (2, 384), (257, 24)]
PHRASE_S = [1, 2, 63, 64, 65, 129, 383, 384, 385, 512]
MASKS = ("suffix", "cls_only", "holes", "ones")


@pytest.fixture(autouse=True)
def _fp32_matmuls():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def make_mask(kind, B, S, device="cuda"):
    """suffix: sequence b keeps its first S - b*(S//(2B)) - b tokens (at least one); cls_only: only position 0; holes: every
    third key (2, 5, 8, ...) masked; ones: nothing masked."""
    m = torch.ones((B, S), dtype=torch.int64)
    if kind == "suffix":
        for b in range(B):
            m[b, max(1, S - b * (S // (2 * B)) - b):] = 0
    elif kind == "cls_only":
        m[:, 1:] = 0
    elif kind == "holes":
        m[:, 2::3] = 0
    else:
        assert kind == "ones"
    return m.to(device)


def tokens(B, S, mask, seed, type_split):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(200, VOCAB, (B, S), generator=g)
    ids[:, 0] = 101
    if S > 1:
        ids[:, -1] = 102
    tt = torch.zeros_like(ids)
    if type_split:
        tt[:, S // 2:] = 1
    ids, tt = ids.cuda(), tt.cuda()
    return ids * mask, mask, tt * mask                  # padding: id 0, token type 0


@pytest.fixture(scope="module", params=STRESS_KINDS)
def stressed(request):
    """(kind, Encoder with all three towers and the filter head, weights in fp64 and fp32 on the GPU): one per weight set, the
    tests of both paths grouped by it."""
    from densephrases_b200.encoder import BertGeometry, Encoder
    geo = BertGeometry(vocab_size=VOCAB)
    sd = stressed_state_dict(geo, SEED, request.param)
    yield request.param, Encoder(geo, state_dict=sd), {k: v.cuda().double() for k, v in sd.items()}, {k: v.cuda() for k, v in sd.items()}
    torch.cuda.empty_cache()


def settings(enc, S, phrase):
    """(mode, tensor-core attention) pairs that run a different kernel set at this S."""
    att = [True, False] if (S <= 64 or (phrase and S <= 384)) else [True]
    return [(m, a) for m in MODES for a in att]


def vector_errors(got, ref, ref32):
    """per row of [n, 768]: (max |diff| / scale, torch fp32's max |diff| / scale, cosine, scale)"""
    scale = ref.abs().amax(1).clamp_min(1.0)
    d = (got.double() - ref).abs().amax(1) / scale
    d32 = (ref32.double() - ref).abs().amax(1) / scale
    return d, d32, F.cosine_similarity(got.double(), ref, dim=1), scale


def judge(kind, mode, d, d32, cosine):
    """per-vector bars of the module docstring -> (every vector within, bar of the worst vector)"""
    bar, cmin = TF32_STRESSED.get(kind, (BAR["tf32"], 0.999)) if mode == "tf32" else (BAR[mode], -1.0)
    ok = (d <= bar) & (cosine > cmin)
    ok |= (d32 > ILL) & (d <= ILL_FACTOR[mode] * d32)
    return bool(ok.all()), bar


@pytest.mark.parametrize("B,S", QUERY_SHAPES)
def test_query_path_against_fp64(stressed, B, S):
    """Both query towers' [CLS] vectors, every mode, both attention settings where they differ (S <= 64), every mask."""
    from oracle import encoder_ref
    kind, enc, sd64, sd32 = stressed
    bad = []
    try:
        for mask_kind in MASKS:
            ids, mask, tt = tokens(B, S, make_mask(mask_kind, B, S), B * 1000 + S, False)
            ref = torch.cat(encoder_ref.embed_query(sd64, ids, mask, tt, dtype=torch.float64), 0).reshape(2 * B, 768)
            ref32 = torch.cat(encoder_ref.embed_query(sd32, ids, mask, tt), 0).reshape(2 * B, 768)
            for mode, tc in settings(enc, S, False):
                enc.set_precision(mode)
                enc.set_attention(tc)
                s, e = enc.embed_query(ids, mask, tt)
                d, d32, cosine, _ = vector_errors(torch.cat([s, e], 0).reshape(2 * B, 768), ref, ref32)
                ok = bool(torch.isfinite(s).all() and torch.isfinite(e).all()) and judge(kind, mode, d, d32, cosine)[0]
                print(f"LIMITS query {kind} {mode} tc={int(tc)} B={B} S={S} {mask_kind}: max|d|/scale {d.max().item():.2e} "
                      f"min cos {cosine.min().item():.6f} torch-fp32 {d32.max().item():.2e}")
                if not ok:
                    bad.append((mode, tc, mask_kind, d.max().item(), cosine.min().item()))
    finally:
        enc.set_precision("bf16x3")
        enc.set_attention(True)
    assert not bad, f"query {kind} B={B} S={S}: over the bar in {bad}"


@pytest.mark.parametrize("S", PHRASE_S)
@pytest.mark.parametrize("B", [1, 3])
def test_phrase_path_against_fp64(stressed, B, S):
    """Every token vector and both filter logits, every mode, tensor-core and SIMT attention (SIMT up to S = 384), every mask
    (at B = 1 the suffix mask pads nothing and is left out)."""
    from tests import phrase_ref
    kind, enc, sd64, sd32 = stressed
    wnorm = max(1.0, sd64["filter_linear.weight"].norm(dim=1).max().item())
    bad = []
    try:
        for mask_kind in MASKS[B == 1:]:
            ids, mask, tt = tokens(B, S, make_mask(mask_kind, B, S), B * 1000 + S + 7, True)
            rs, _, rfs, rfe = phrase_ref.embed_phrase(sd64, ids, mask, tt, dtype=torch.float64)
            rs32 = phrase_ref.embed_phrase(sd32, ids, mask, tt)[0]
            rf = torch.stack([rfs, rfe], -1).reshape(B * S, 2)
            for mode, tc in settings(enc, S, True):
                enc.set_precision(mode)
                enc.set_attention(tc)
                s, _, fs, fe = enc(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
                d, d32, cosine, scale = vector_errors(s.reshape(B * S, 768), rs.reshape(B * S, 768), rs32.reshape(B * S, 768))
                df = (torch.stack([fs, fe], -1).reshape(B * S, 2).double() - rf).abs().amax(1) / (scale * wnorm)
                ok_vec, bar = judge(kind, mode, d, d32, cosine)
                ok = bool(torch.isfinite(s).all() and torch.isfinite(fs).all() and torch.isfinite(fe).all()) and ok_vec \
                    and bool(((df <= bar) | ((d32 > ILL) & (df <= ILL_FACTOR[mode] * d32))).all())
                print(f"LIMITS phrase {kind} {mode} tc={int(tc)} B={B} S={S} {mask_kind}: max|d|/scale {d.max().item():.2e} "
                      f"filter {df.max().item():.2e} min cos {cosine.min().item():.6f} torch-fp32 {d32.max().item():.2e}")
                if not ok:
                    bad.append((mode, tc, mask_kind, d.max().item(), df.max().item(), cosine.min().item()))
    finally:
        enc.set_precision("bf16x3")
        enc.set_attention(True)
    assert not bad, f"phrase {kind} B={B} S={S}: over the bar in {bad}"


# ---- the attention kernels alone -----------------------------------------------------------------------------------------
ATT_S = [1, 2, 16, 17, 32, 33, 64, 65, 96, 97, 128, 129, 384, 385, 512]
ATT_TOL = {0: 2e-5, 1: 1e-2, 2: 1e-4}        # tests/test_encoder.py: SIMT fp32 | wgmma TF32 | wgmma bf16 (hi, lo) planes
LOGIT_UNIT = 64.0                             # the bars hold as they are up to |QK^T/8| = 64, then grow with the largest logit


def heads(qkv, B, S):
    return [qkv[:, i * 768:(i + 1) * 768].reshape(B, S, 12, 64).permute(0, 2, 1, 3) for i in range(3)]


def attention_ref(qkv, mask, B, S):
    """softmax(QK^T/8 + (1-mask)*-10000) V in the dtype of qkv -> [B*S, 768]"""
    q, k, v = heads(qkv, B, S)
    sc = q @ k.transpose(-1, -2) / 8.0 + ((1.0 - mask.to(qkv.dtype)) * -10000.0)[:, None, None, :]
    return (torch.softmax(sc, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B * S, 768)


def run_attention(qkv, mask, B, S, kernel):
    from densephrases_b200 import _lib as L
    ctx = torch.full((B * S, 768), float("nan"), device="cuda")
    L.check(L.lib().dph_attention_bert(qkv.data_ptr(), mask.data_ptr(), B, S, ctx.data_ptr(), kernel, None))
    torch.cuda.synchronize()
    return ctx


def attention_cases(B, S):
    """(name, qkv fp32 [B*S, 2304], mask) at the logit ranges and layouts where an (online) softmax goes wrong."""
    g = torch.Generator(device="cuda").manual_seed(1000 + S)
    base = torch.randn((B * S, 2304), generator=g, device="cuda")
    for scale in (1.0, 5.0, 15.0):             # logits' std ~ scale^2: up to the hundreds
        for mask_kind in MASKS:
            yield f"x{scale:g} {mask_kind}", (base * scale).contiguous(), make_mask(mask_kind, B, S)
    # ramp: the logit on key j gets + j/2 (exact: q_d0 = 8, k_d0 = j/2), so every 64-key block raises the row maximum by 32 and the
    # final block holds it; reversed, the first block holds it.  The rest of the dot product adds a unit-scale random part.
    for rev in (False, True):
        qkv = base.clone()
        q, k, _ = heads(qkv, B, S)
        j = torch.arange(S, device="cuda", dtype=torch.float32)
        q[..., 0] = 8.0
        k[..., 0] = 0.5 * ((S - 1 - j) if rev else j)
        for mask_kind in ("ones", "suffix"):
            yield f"ramp{'-reversed' if rev else ''} {mask_kind}", qkv, make_mask(mask_kind, B, S)
    # a masked key (a hole, in the last key block) whose scaled logit is 10004 against the others' unit-scale ones: exactly
    # representable (q_d1 = 320, k_d1 = 250; q_d2 = 4, k_d2 = 8; the key's other dims 0), so after the -10000 bias its logit is
    # exactly 4 in every kernel.  The reference still gives it weight, and its value is large so a kernel that drops it shows.
    if S >= 3:
        qkv = base.clone()
        mask = make_mask("holes", B, S)
        p = max(i for i in range(S) if i % 3 == 2)
        q, k, v = heads(qkv, B, S)
        q[..., 1] = 320.0
        q[..., 2] = 4.0
        k[..., 1] = 0.0
        k[..., 2] = 0.0
        k[:, :, p, :] = 0.0
        k[:, :, p, 1] = 250.0
        k[:, :, p, 2] = 8.0
        v[:, :, p, :] *= 10.0
        yield "planted-masked-key holes", qkv, mask


@pytest.mark.parametrize("S", ATT_S)
@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_attention_kernels_at_range_against_fp64(kernel, S):
    """Every kernel at every variant boundary against fp64: bar = ATT_TOL * max(1, max |v|) * max(1, L / 64), L the largest
    |QK^T/8| over unmasked keys.  Every kernel's logits carry its operand rounding relative to their size, so the error of the
    probabilities grows with L (the SIMT kernel's error equals torch fp32's at every scale)."""
    B = 3
    if kernel == 0 and S > 384:
        qkv, mask = torch.zeros((B * S, 2304), device="cuda"), make_mask("ones", B, S)
        with pytest.raises(RuntimeError, match="S <= 384"):
            run_attention(qkv, mask, B, S, 0)
        return
    bad = []
    for name, qkv, mask in attention_cases(B, S):
        ref = attention_ref(qkv.double(), mask, B, S)
        ref32 = attention_ref(qkv, mask, B, S)
        vmax = max(1.0, qkv[:, 1536:].abs().max().item())
        q, k, _ = heads(qkv.double(), B, S)
        logits = (q @ k.transpose(-1, -2) / 8.0).masked_fill(~mask.bool()[:, None, None, :], 0.0)
        bar = ATT_TOL[kernel] * max(1.0, logits.abs().max().item() / LOGIT_UNIT)
        ctx = run_attention(qkv, mask, B, S, kernel)
        d = (ctx.double() - ref).abs().max().item() / vmax
        d32 = (ref32.double() - ref).abs().max().item() / vmax
        print(f"LIMITS attention kernel={kernel} S={S} {name}: max|d|/max|v| {d:.2e} bar {bar:.1e} torch-fp32 {d32:.2e}")
        if not (torch.isfinite(ctx).all() and d <= bar):
            bad.append((name, d, bar))
    assert not bad, f"attention kernel {kernel} S={S}: over the bar in {bad}"


# ---- the GEMM epilogue away from unit scale ------------------------------------------------------------------------------
GEMM_TOL = {0: 2 ** -9, 1: 1e-5, 2: 2e-5}     # 1xTF32 (operands cut to 10 mantissa bits) | 3xTF32 | bf16x3, of sum_k |a_k w_k| + |bias| + |residual|


@pytest.mark.parametrize("variant", ["gelu_tails", "gelu_bias50", "resid_bias50"])
@pytest.mark.parametrize("M,N,K", [(333, 3072, 768), (200, 768, 3072), (1, 256, 96)])
@pytest.mark.parametrize("precise", [0, 1, 2])
def test_gemm_epilogue_at_range_against_fp64(precise, M, N, K, variant):
    """out = act(A W^T + bias) + residual with pre-activations over +-10 (GELU's tails) or a bias around +-50, every element
    within GEMM_TOL of its own magnitude scale against fp64."""
    from densephrases_b200 import _lib as L
    g = torch.Generator(device="cuda").manual_seed(M + N + K + precise)
    A = torch.randn((M, K), generator=g, device="cuda")
    W = torch.randn((N, K), generator=g, device="cuda") * (5.0 / K ** 0.5)        # A W^T: std 5, range ~ +-20
    if variant == "gelu_tails":
        bias = torch.randn((N,), generator=g, device="cuda")
    else:
        bias = 50.0 * torch.sign(torch.randn((N,), generator=g, device="cuda")) + torch.randn((N,), generator=g, device="cuda")
    resid = 10.0 * torch.randn((M, N), generator=g, device="cuda") if variant == "resid_bias50" else None
    act = 1 if variant.startswith("gelu") else 0
    out = torch.empty((M, N), device="cuda")
    L.check(L.lib().dph_gemm_tf32_nt(A.data_ptr(), W.data_ptr(), bias.data_ptr(), resid.data_ptr() if resid is not None else None,
                                     out.data_ptr(), M, N, K, act, precise, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    pre = A.double() @ W.double().T + bias.double()
    ref = F.gelu(pre) if act else pre
    ref32 = F.gelu(F.linear(A, W, bias)) if act else F.linear(A, W, bias)
    scale = A.double().abs() @ W.double().abs().T + bias.double().abs()
    if resid is not None:
        ref, ref32, scale = ref + resid.double(), ref32 + resid, scale + resid.double().abs()
    assert pre.min() < -8 and pre.max() > 8
    err = ((out.double() - ref).abs() / scale).max().item()
    err32 = ((ref32.double() - ref).abs() / scale).max().item()
    print(f"LIMITS gemm precise={precise} {M}x{N}x{K} {variant}: max|d|/scale {err:.2e} torch-fp32 {err32:.2e}")
    assert torch.isfinite(out).all() and err <= GEMM_TOL[precise], f"max |diff| / scale {err:.3e}"
