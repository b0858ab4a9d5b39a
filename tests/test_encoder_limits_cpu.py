"""The trained-like weight constructions of tests/helpers.stressed_state_dict do what they claim, shown on the fp64 reference
(oracle/encoder_ref.tower_forward with a trace hook), and the fp64 reference is the fp32 restatement run in another dtype."""
import pytest
import torch

from tests.helpers import OUTLIER_DIMS, SHARP_SELF_HEADS, STRESS_KINDS, stressed_state_dict

B, S = 2, 16


def batch():
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(200, 1000, (B, S), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    mask = torch.ones_like(ids)
    mask[1, 12:] = 0
    return ids, mask, torch.zeros_like(ids)


def statistics(sd, prefix):
    """Run one tower in fp64 and collect: largest |logit| over unmasked keys, largest probability per head, LayerNorm input
    magnitude per hidden dimension, GELU input range, and the rms of the last LayerNorm input per layer."""
    from oracle.encoder_ref import tower_forward
    ids, mask, tt = batch()
    keep = mask.bool()[:, None, None, :]
    st = {"logit": 0.0, "p_head": torch.zeros(12, dtype=torch.float64), "ln_dim": torch.zeros(768, dtype=torch.float64),
          "gelu": (0.0, 0.0), "rms": []}

    def trace(l, what, x):
        if what == "logits":
            st["logit"] = max(st["logit"], x.masked_select(keep.expand_as(x)).abs().max().item())
        elif what == "probs":
            st["p_head"] = torch.maximum(st["p_head"], x.amax(dim=(0, 2, 3)))
        elif what == "ln_in":
            st["ln_dim"] = torch.maximum(st["ln_dim"], x.abs().amax(dim=(0, 1)))
            st["rms"].append(x.pow(2).mean().sqrt().item())
        elif what == "gelu_in":
            st["gelu"] = (min(st["gelu"][0], x.min().item()), max(st["gelu"][1], x.max().item()))
    out = tower_forward(sd, prefix, ids, mask, tt, dtype=torch.float64, trace=trace)
    assert out.dtype == torch.float64 and torch.isfinite(out).all()
    return st


@pytest.fixture(scope="module")
def geo():
    from densephrases_b200.encoder import BertGeometry
    return BertGeometry(vocab_size=1000)


@pytest.mark.parametrize("kind", STRESS_KINDS + ("random",))
def test_stressed_weights_reach_their_statistics(geo, kind):
    from densephrases_b200.encoder import TOWERS, random_state_dict
    sd = random_state_dict(geo, 3, prefixes=("phrase_encoder",)) if kind == "random" else stressed_state_dict(geo, 3, kind)
    for prefix in ("phrase_encoder",) if kind == "random" else ("query_start_encoder", "phrase_encoder"):
        st = statistics(sd, prefix)
        sharp = st["logit"] >= 20 and st["p_head"][list(SHARP_SELF_HEADS)].max() >= 0.9
        ln_planted = st["ln_dim"][list(OUTLIER_DIMS)].max().item()
        outlier = ln_planted >= 20
        tails = st["gelu"][0] <= -8 and st["gelu"][1] >= 8
        print(f"{kind} {prefix}: max|logit| {st['logit']:.1f}, max p per head {st['p_head'].max().item():.4f}, "
              f"max|LayerNorm in| {st['ln_dim'].max().item():.1f} (planted dims {ln_planted:.1f}), GELU in {st['gelu'][0]:.1f}..{st['gelu'][1]:.1f}, "
              f"rms of the last LayerNorm input, layer 0 / 11: {st['rms'][2]:.2f} / {st['rms'][-1]:.2f}")
        if kind == "random":          # what random initialisation reaches: none of it
            assert not sharp and not outlier and not tails
            assert st["logit"] < 10 and st["ln_dim"].max() < 15
        if kind in ("sharp", "all"):
            assert sharp
        if kind in ("outlier", "all"):
            assert outlier
        if kind == "outlier":         # the planted dimensions are the largest of the residual stream
            assert st["ln_dim"].argmax().item() in OUTLIER_DIMS
        if kind in ("tails", "all"):
            assert tails
        if kind == "tails":           # the hidden states grow from layer to layer
            assert st["rms"][-1] > 2 * st["rms"][2]


def test_stressed_state_dict_names(geo):
    from densephrases_b200.encoder import PHRASE_TOWER, TOWERS, random_phrase_state_dict, random_state_dict, tower_blob
    ref = {**random_state_dict(geo, 1), **random_phrase_state_dict(geo, 1)}
    for kind in STRESS_KINDS:
        sd = stressed_state_dict(geo, 1, kind)
        assert sorted(sd) == sorted(ref) and all(sd[k].shape == ref[k].shape for k in sd)
    for prefix in TOWERS + (PHRASE_TOWER,):
        assert tower_blob(sd, prefix, geo).size == tower_blob(ref, prefix, geo).size
    with pytest.raises(ValueError):
        stressed_state_dict(geo, 1, "soft")


def test_fp64_reference_is_the_fp32_restatement_in_another_dtype(geo):
    """The default stays fp32 (and the trace hook changes nothing); fp64 runs the same operations: on random weights the two agree
    to fp32 rounding, and the query and phrase entry points pass the dtype through."""
    from densephrases_b200.encoder import random_phrase_state_dict, random_state_dict
    from oracle import encoder_ref
    from tests import phrase_ref
    ids, mask, tt = batch()
    sd = {**random_state_dict(geo, 2), **random_phrase_state_dict(geo, 2)}
    x32 = encoder_ref.tower_forward(sd, "query_start_encoder", ids, mask, tt)
    seen = []
    assert torch.equal(x32, encoder_ref.tower_forward(sd, "query_start_encoder", ids, mask, tt, trace=lambda *a: seen.append(a[1])))
    assert x32.dtype == torch.float32 and seen.count("logits") == 12 and seen.count("ln_in") == 25 and seen.count("gelu_in") == 12
    s32, e32 = encoder_ref.embed_query(sd, ids, mask, tt)
    s64, e64 = encoder_ref.embed_query(sd, ids, mask, tt, dtype=torch.float64)
    assert s64.dtype == e64.dtype == torch.float64
    assert (s64 - s32.double()).abs().max() < 1e-4 and (e64 - e32.double()).abs().max() < 1e-4
    assert torch.equal(s32, x32[:, :1])
    p32 = phrase_ref.embed_phrase(sd, ids, mask, tt)
    p64 = phrase_ref.embed_phrase(sd, ids, mask, tt, dtype=torch.float64)
    for a, b in zip(p32, p64):
        assert b.dtype == torch.float64 and (b - a.double()).abs().max() < 1e-4
