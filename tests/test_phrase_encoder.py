"""Phrase encoder parity: Encoder.embed_phrase / forward(input_ids=..., return_phrase=True) on the GPU.

Oracle chain, as for the query encoder: the UNMODIFIED reference Encoder (run in the build container by
tests/golden/make_phrase_golden.py) -> committed fixture tests/golden/encoder_phrase.npz -> (CPU test) the torch fp32
restatement tests/phrase_ref.py reproduces it -> (GPU tests) the CUDA phrase path is compared with both.

Tolerances follow the query path: 'bf16x3' and '3xtf32' within 1e-3 of fp32, 'tf32' within 5e-2 with cosine > 0.9995 per
token vector; the same bars for the filter logits (scale ~0.6)."""
import argparse
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden", "encoder_phrase.npz")
CASES = ["b3_s48", "b2_s100", "b2_s384", "b1_s512"]
TOL = {"tf32": 5e-2, "3xtf32": 1e-3, "bf16x3": 1e-3}


def load_case(name):
    g = np.load(GOLD)
    t = lambda k: torch.from_numpy(g[f"{name}_{k}"])
    return dict(seed=int(g["seed"]), vocab=int(g["vocab"]), ids=t("ids"), mask=t("mask"), tt=t("tt"), rows=t("rows"), vec=t("vec"),
                fs=t("filter_start"), fe=t("filter_end"))


def cos(a, b):
    return torch.nn.functional.cosine_similarity(a.flatten(1), b.flatten(1), dim=1)


# ---- CPU ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_torch_restatement_reproduces_reference_phrase_fixture(name):
    from densephrases_b200.encoder import BertGeometry, random_phrase_state_dict
    from tests import phrase_ref
    c = load_case(name)
    sd = random_phrase_state_dict(BertGeometry(vocab_size=c["vocab"]), c["seed"])
    start, end, fs, fe = phrase_ref.embed_phrase(sd, c["ids"], c["mask"], c["tt"])
    B, S = c["ids"].shape
    assert start.shape == (B, S, 768) and end is start and fs.shape == (B, S) and fe.shape == (B, S)
    assert (start.reshape(B * S, 768)[c["rows"]] - c["vec"]).abs().max() < 2e-4
    assert (fs - c["fs"]).abs().max() < 2e-4 and (fe - c["fe"]).abs().max() < 2e-4
    assert (fs - fe).abs().max() > 1e-2             # the two filter rows really differ


def test_fixture_is_ragged_and_small():
    for name in CASES:
        c = load_case(name)
        lens = c["mask"].sum(1)
        S = c["ids"].shape[1]
        assert (lens >= S // 2).all() and (lens <= S).all()
    assert os.path.getsize(GOLD) <= 2 * 1024 * 1024


def test_state_dict_names_and_helpers():
    from densephrases_b200.encoder import (BertGeometry, TOWERS, canonical_state_dict, random_phrase_state_dict, random_state_dict,
                                           synthetic_context_batch, tower_blob)
    from densephrases_b200.runtime import backward_compat
    geo = BertGeometry(vocab_size=1000)
    sd = random_phrase_state_dict(geo, 4)
    assert sd["filter_linear.weight"].shape == (2, 768) and sd["filter_linear.bias"].shape == (2,)
    assert all(k.startswith(("phrase_encoder.", "filter_linear.")) for k in sd)
    # the phrase tower is the query generator's tower under another prefix: the default output stays what the query goldens need
    q = random_state_dict(geo, 4)
    assert sorted({k.split(".")[0] for k in q}) == sorted(TOWERS)
    p = random_state_dict(geo, 4, prefixes=("phrase_encoder",))
    assert torch.equal(p["phrase_encoder.embeddings.word_embeddings.weight"], sd["phrase_encoder.embeddings.word_embeddings.weight"])
    # legacy checkpoint names (single_utils.backward_compat): bert_start -> phrase_encoder, in the Encoder and in runtime
    legacy = {k.replace("phrase_encoder", "bert_start"): v for k, v in sd.items()}
    for canon in (canonical_state_dict(legacy), backward_compat(legacy)):
        assert sorted(canon) == sorted(sd)
    blob = tower_blob(canonical_state_dict(legacy), "phrase_encoder", geo)
    assert np.array_equal(blob, tower_blob(sd, "phrase_encoder", geo))
    assert canonical_state_dict({"bert_q_start.x": 1, "bert_q_end.y": 2}) == {"query_start_encoder.x": 1, "query_end_encoder.y": 2}
    ids, mask, tt = synthetic_context_batch(6, 100, 5000, 3, type_split=True)
    lens = mask.sum(1)
    assert ((lens >= 50) & (lens <= 100)).all() and len(set(lens.tolist())) > 1
    assert (ids[:, 0] == 101).all() and all(ids[b, lens[b] - 1] == 102 for b in range(6)) and (ids[mask == 0] == 0).all()
    assert tt.max() == 1 and (tt[mask == 0] == 0).all()


def test_bad_phrase_shapes_are_rejected():
    from densephrases_b200.encoder import BertGeometry, check_phrase_shape
    geo = BertGeometry(vocab_size=1000)
    assert check_phrase_shape(geo, (128, 512)) == (128, 512)
    for shape in [(2, 513), (2, 0), (0, 8), (65536, 8), (2, 3, 4), (8,)]:
        with pytest.raises(ValueError):
            check_phrase_shape(geo, shape)
    with pytest.raises(ValueError):
        check_phrase_shape(BertGeometry(vocab_size=1000, max_position_embeddings=256), (1, 300))


# ---- GPU ---------------------------------------------------------------------------------------------------------------
_ENC = {}


def encoder_for(vocab, seed):
    from densephrases_b200.encoder import BertGeometry, Encoder, random_phrase_state_dict
    key = (vocab, seed)
    if key not in _ENC:
        geo = BertGeometry(vocab_size=vocab)
        sd = random_phrase_state_dict(geo, seed)
        _ENC.clear()
        _ENC[key] = (Encoder(geo, state_dict=sd, phrase_only=True), sd)
    enc, sd = _ENC[key]
    enc.set_precision("bf16x3")
    enc.set_attention(True)
    return enc, sd


def check(mode, s, fs, fe, ref_s, ref_fs, ref_fe, what):
    ds = (s - ref_s).abs().max().item()
    df = max((fs - ref_fs).abs().max().item(), (fe - ref_fe).abs().max().item())
    print(f"{what} {mode}: max|diff| vectors {ds:.2e} filter {df:.2e}")
    assert torch.isfinite(s).all() and torch.isfinite(fs).all() and torch.isfinite(fe).all()
    assert ds < TOL[mode] and df < TOL[mode]
    if mode == "tf32":
        assert cos(s, ref_s).min() > 0.9995


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tf32", "3xtf32", "bf16x3"])
@pytest.mark.parametrize("name", CASES)
def test_cuda_phrase_encoder_matches_reference_fixture(name, mode):
    c = load_case(name)
    enc, _ = encoder_for(c["vocab"], c["seed"])
    enc.set_precision(mode)
    start, end, fs, fe = enc(input_ids=c["ids"], attention_mask=c["mask"], token_type_ids=c["tt"], return_phrase=True)
    B, S = c["ids"].shape
    assert start.shape == (B, S, 768) and end is start and fs.shape == (B, S) and fe.shape == (B, S)
    check(mode, start.reshape(B * S, 768)[c["rows"].cuda()].cpu(), fs.cpu(), fe.cpu(), c["vec"], c["fs"], c["fe"], name)


@pytest.mark.gpu
@pytest.mark.parametrize("B,S", [(32, 384), (8, 512)])
def test_cuda_phrase_encoder_full_batches_against_torch_fp32(B, S):
    """Full-size batches, every row, against the torch fp32 restatement on the GPU with TF32 off, in every mode."""
    from densephrases_b200.encoder import synthetic_context_batch
    from tests import phrase_ref
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    enc, sd = encoder_for(28996, 17)
    ids, mask, tt = (t.cuda() for t in synthetic_context_batch(B, S, 28996, B + S, type_split=True))
    rs, _, rfs, rfe = phrase_ref.embed_phrase({k: v.cuda() for k, v in sd.items()}, ids, mask, tt)
    for mode in ("bf16x3", "3xtf32", "tf32"):
        enc.set_precision(mode)
        s, e, fs, fe = enc(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
        check(mode, s.reshape(B * S, 768), fs, fe, rs.reshape(B * S, 768), rfs, rfe, f"B={B} S={S}")


def ragged_qkv(B, S, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn((B * S, 2304), generator=g, device="cuda")
    mask = torch.ones((B, S), dtype=torch.int64, device="cuda")
    for b in range(B):
        mask[b, S - (b * S) // (2 * B) - 3 * b:] = 0          # ragged: from 0 to ~S/2 padded keys per sequence
    return qkv, mask


def attention_torch(qkv, mask, B, S):
    q, k, v = (qkv[:, i * 768:(i + 1) * 768].reshape(B, S, 12, 64).permute(0, 2, 1, 3) for i in range(3))
    sc = q @ k.transpose(-1, -2) / 8.0 + ((1.0 - mask.float()) * -10000.0)[:, None, None, :]
    return (torch.softmax(sc, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B * S, 768)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [65, 128, 200, 384, 512])
@pytest.mark.parametrize("tensor_core,tol", [(1, 1e-2), (2, 1e-4)])     # wgmma TF32 | wgmma bf16 (hi, lo) planes
def test_long_sequence_attention_against_torch(S, tensor_core, tol):
    """attention_flash.cu through the C ABI against torch fp32, ragged masks; at S <= 384 also against the SIMT kernels."""
    from densephrases_b200 import _lib as L
    torch.backends.cuda.matmul.allow_tf32 = False
    B = 3
    qkv, mask = ragged_qkv(B, S, S)
    ref = attention_torch(qkv, mask, B, S)

    def run(tc):
        ctx = torch.full((B * S, 768), float("nan"), device="cuda")
        L.check(L.lib().dph_attention_bert(qkv.data_ptr(), mask.data_ptr(), B, S, ctx.data_ptr(), tc, None))
        torch.cuda.synchronize()
        return ctx
    ctx = run(tensor_core)
    d = (ctx - ref).abs().max().item()
    print(f"attention B={B} S={S} tensor_core={tensor_core}: max|diff| {d:.2e}")
    assert torch.isfinite(ctx).all() and d < tol
    if S <= 384:
        assert (ctx - run(0)).abs().max().item() < tol
    else:
        with pytest.raises(RuntimeError, match="S <= 384"):
            run(0)


@pytest.mark.gpu
def test_attention_rejects_too_long_sequences():
    from densephrases_b200 import _lib as L
    qkv, mask = ragged_qkv(1, 513, 1)
    ctx = torch.zeros((513, 768), device="cuda")
    for tc in (0, 1, 2):
        with pytest.raises(RuntimeError):
            L.check(L.lib().dph_attention_bert(qkv.data_ptr(), mask.data_ptr(), 1, 513, ctx.data_ptr(), tc, None))


@pytest.mark.gpu
@pytest.mark.parametrize("S", [200, 384])
def test_flash_attention_matches_simt_inside_the_encoder(S):
    """The phrase path with the tensor-core attention against the same encoder on the SIMT attention (set_attention(False))."""
    from densephrases_b200.encoder import synthetic_context_batch
    enc, _ = encoder_for(28996, 17)
    ids, mask, tt = synthetic_context_batch(4, S, 28996, S)
    for mode, tol in (("bf16x3", 1e-4), ("tf32", 2e-2)):
        enc.set_precision(mode)
        enc.set_attention(True)
        s1, _, f1, _ = enc(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
        enc.set_attention(False)
        s0, _, f0, _ = enc(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
        d = max((s1 - s0).abs().max().item(), (f1 - f0).abs().max().item())
        print(f"S={S} {mode}: tensor-core vs SIMT attention max|diff| {d:.2e}")
        assert d < tol
    enc.set_attention(True)


@pytest.mark.gpu
def test_phrase_host_and_device_inputs_streams_and_forward():
    import ctypes as C
    from densephrases_b200 import _lib as L
    from densephrases_b200.encoder import synthetic_context_batch
    enc, _ = encoder_for(28996, 17)
    ids, mask, tt = synthetic_context_batch(3, 150, 28996, 9, type_split=True)
    s_dev, e_dev, fs, fe = enc(input_ids=ids.cuda(), attention_mask=mask.cuda(), token_type_ids=tt.cuda(), return_phrase=True)
    assert e_dev is s_dev and s_dev.is_cuda and fs.is_cuda
    s2, e2 = enc.embed_phrase(ids, mask, tt)                       # CPU tensors in, GPU out; no filter
    assert e2 is s2 and torch.equal(s2, s_dev)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        s3, _, fs3, fe3 = enc(input_ids=ids.cuda(), attention_mask=mask.cuda(), token_type_ids=tt.cuda(), return_phrase=True)
    st.synchronize()
    assert torch.equal(s3, s_dev) and torch.equal(fs3, fs) and torch.equal(fe3, fe)
    # the C ABI with host buffers: synchronous, same numbers
    out = np.zeros((3, 150, 768), np.float32)
    fo = np.zeros((3, 150, 2), np.float32)
    i64 = lambda t: np.ascontiguousarray(t.numpy().astype(np.int64))
    hi, hm, ht = i64(ids), i64(mask), i64(tt)
    L.check(L.lib().dph_encoder_embed_phrase(enc._h, hi.ctypes.data_as(C.c_void_p), hm.ctypes.data_as(C.c_void_p), ht.ctypes.data_as(C.c_void_p),
                                             3, 150, out.ctypes.data_as(C.c_void_p), fo.ctypes.data_as(C.c_void_p), L.MEM_HOST))
    assert np.array_equal(out, s_dev.cpu().numpy()) and np.array_equal(fo[..., 0], fs.cpu().numpy()) and np.array_equal(fo[..., 1], fe.cpu().numpy())
    with pytest.raises(NotImplementedError):
        enc(input_ids_=ids, attention_mask_=mask, token_type_ids_=tt, return_query=True)     # phrase-only: no query towers


@pytest.mark.gpu
def test_phrase_errors():
    from densephrases_b200.encoder import BertGeometry, Encoder, random_phrase_state_dict, random_state_dict
    geo = BertGeometry(vocab_size=500)
    q_only = Encoder(geo, state_dict=random_state_dict(geo, 1))
    ids = torch.full((2, 80), 3, dtype=torch.int64)
    mask, tt = torch.ones_like(ids), torch.zeros_like(ids)
    with pytest.raises(NotImplementedError):
        q_only(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
    with pytest.raises(NotImplementedError):
        q_only.embed_phrase(ids, mask, tt)
    both = Encoder(geo, state_dict={**random_state_dict(geo, 1), **random_phrase_state_dict(geo, 2)})
    both.embed_query(ids[:, :16], mask[:, :16], tt[:, :16])
    both.embed_phrase(ids, mask, tt)
    long_ids = torch.full((1, 513), 3, dtype=torch.int64)
    with pytest.raises(ValueError):
        both.embed_phrase(long_ids, torch.ones_like(long_ids), torch.zeros_like(long_ids))
    both.set_attention(False)
    with pytest.raises(RuntimeError, match="S <= 384"):
        both.embed_phrase(ids.repeat(1, 5), mask.repeat(1, 5), tt.repeat(1, 5))       # S = 400 on the SIMT attention
    both.set_attention(True)
    bad = ids.clone(); bad[1, 70] = 500
    with pytest.raises(IndexError):
        both.embed_phrase(bad, mask, tt)                          # host tensor: range-checked before the copy
    with pytest.raises(IndexError):
        both.embed_phrase(ids, mask, tt + 2)
    both.embed_phrase(bad.cuda(), mask.cuda(), tt.cuda())         # device tensor: the kernel clamps the row and latches a flag ...
    with pytest.raises(RuntimeError, match="embedding tables"):
        both.embed_phrase(ids.cuda(), mask.cuda(), tt.cuda())     # ... which the next call reports
    both.embed_phrase(ids.cuda(), mask.cuda(), tt.cuda())         # and the encoder stays usable
    with pytest.raises(KeyError):
        Encoder(geo, state_dict=random_state_dict(geo, 1), phrase_only=True)


@pytest.mark.gpu
def test_load_encoder_phrase_only_random_init():
    from densephrases_b200.runtime import load_encoder
    args = argparse.Namespace(load_dir="", pretrained_name_or_path="", tokenizer_name="", cache_dir="", do_lower_case=False,
                              allow_random_init=True, seed=5)
    model, tok, config = load_encoder("cuda", args, phrase_only=True)
    ids = torch.randint(1000, config.vocab_size, (2, 96))
    mask, tt = torch.ones_like(ids), torch.zeros_like(ids)
    s, e, fs, fe = model(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
    assert s.shape == (2, 96, 768) and e is s and fs.shape == (2, 96) and torch.isfinite(s).all() and torch.isfinite(fs).all()
    with pytest.raises(NotImplementedError):
        model(input_ids_=ids, attention_mask_=mask, token_type_ids_=tt, return_query=True)


@pytest.mark.gpu
def test_phrase_batch_of_65536_tokens():
    """B = 128 at S = 512 (T = 65 536 tokens) in one call: finite everywhere, and the first and last sequences match the torch fp32
    restatement run on them alone (a sequence's result does not depend on the rest of the batch)."""
    from densephrases_b200.encoder import synthetic_context_batch
    from tests import phrase_ref
    torch.backends.cuda.matmul.allow_tf32 = False
    enc, sd = encoder_for(28996, 17)
    B, S = 128, 512
    ids, mask, tt = (t.cuda() for t in synthetic_context_batch(B, S, 28996, 65536))
    s, _, fs, fe = enc(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
    assert torch.isfinite(s).all() and torch.isfinite(fs).all() and torch.isfinite(fe).all()
    sd_gpu = {k: v.cuda() for k, v in sd.items()}
    for b in (0, B - 1):
        rs, _, rfs, rfe = phrase_ref.embed_phrase(sd_gpu, ids[b:b + 1], mask[b:b + 1], tt[b:b + 1])
        check("bf16x3", s[b], fs[b:b + 1], fe[b:b + 1], rs[0], rfs, rfe, f"T=65536 sequence {b}")
    del s, fs, fe
    torch.cuda.empty_cache()
