"""Shared test helpers: matched (oracle, CUDA) index pairs, the top-k comparator, and encoder weights with trained-like statistics."""
import numpy as np

D_MODEL = 768


def opq_matrix(seed, d=D_MODEL):
    rng = np.random.default_rng(seed)
    return np.linalg.qr(rng.standard_normal((d, d)))[0].astype(np.float32)


def uniform_lens(N, nlist):
    base, rem = divmod(N, nlist)
    return np.array([base + (1 if l < rem else 0) for l in range(nlist)], dtype=np.int64)


def near_queries(ref, n, seed, noise=0.3):
    """SURVEY 8d 'near' queries: q = A^T (centroid + decode(code_j)) + N(0, noise^2)."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, max(ref.ntotal, 1), n)
    v, _ = ref.reconstruct(ids) if ref.ids is None else ref.reconstruct(ref.ids[ids])
    q = v @ ref.A            # un-rotate: A^T v  (row-vector form v A)
    return (q + noise * rng.standard_normal(q.shape)).astype(np.float32)


def assert_topk_equal(D, I, Dref, Iref, what=""):
    """Bit-identical scores; identical labels up to permutations inside exactly-equal-score groups (faiss' heap
    order among equal scores is unspecified); in the boundary group only the group size is compared."""
    D = np.asarray(D); I = np.asarray(I); Dref = np.asarray(Dref); Iref = np.asarray(Iref)
    assert D.shape == Dref.shape and I.shape == Iref.shape, what
    bits, bits_ref = D.view(np.int32), Dref.view(np.int32)
    bad = np.argwhere(bits != bits_ref)
    assert bad.size == 0, f"{what}: score bits differ at {bad[:5].tolist()}: {D[tuple(bad[0])]!r} vs {Dref[tuple(bad[0])]!r}"
    for r in range(D.shape[0]):
        if np.array_equal(I[r], Iref[r]):
            continue
        last = D[r, -1]
        for v in np.unique(D[r]):
            a, b = sorted(I[r][D[r] == v].tolist()), sorted(Iref[r][Dref[r] == v].tolist())
            if v == last:
                assert len(a) == len(b), f"{what}: row {r} boundary tie group size"
            else:
                assert a == b, f"{what}: row {r} labels differ at score {v}: {a} vs {b}"


# ---- encoder weights with the statistics of a trained BERT ---------------------------------------------------------------
STRESS_KINDS = ('sharp', 'outlier', 'tails', 'all')
OUTLIER_DIMS = (77, 308, 588)           # hidden dimensions that every LayerNorm of an `outlier` tower blows up
SHARP_SELF_HEADS = {0: 2.5, 1: 2.5, 2: -2.5}     # head -> W_k = scale * W_q + noise: QK^T/8 ~ +-scale * |q|^2 / 8 on the diagonal
SHARP_POS0_HEADS = (3, 4)               # heads whose queries all look for the direction planted in position 0's embedding


def stressed_state_dict(config, seed, kind):
    """Seeded weights in the reference's naming (query_start_encoder, query_end_encoder, phrase_encoder, filter_linear) built on
    random_state_dict, changed so the forward sees what a trained BERT shows and random initialisation does not:
      sharp   -- in heads 0-2 of every layer W_k = +-2.5 W_q + noise, so a token's logit on itself is ~+-25 (QK^T/8 spans +-20..30
                 and a head puts nearly all its weight on one key); heads 3-4 read a unit direction planted in position 0's
                 embedding through one key dimension that every query weights by 2, so they lean on [CLS];
      outlier -- every LayerNorm has gains 6..10 and biases +-3..5 in OUTLIER_DIMS, and the output dense adds a bias there too:
                 the residual stream carries three dimensions many times larger than the rest;
      tails   -- intermediate.dense x2.5 and output.dense x2, LayerNorm gains growing by 10 % a layer: GELU inputs reach +-8 and
                 beyond and the hidden states grow from layer to layer;
      all     -- the three together.
    tests/test_encoder_limits_cpu.py checks that each kind reaches the statistic it claims."""
    import torch
    from densephrases_b200.encoder import PHRASE_TOWER, TOWERS, random_state_dict
    if kind not in STRESS_KINDS:
        raise ValueError(f'kind {kind!r} not in {STRESS_KINDS}')
    towers = TOWERS + (PHRASE_TOWER,)
    sd = random_state_dict(config, seed, prefixes=towers)
    g = torch.Generator().manual_seed(seed + 1)
    sd['filter_linear.weight'] = torch.randn(2, config.hidden_size, generator=g) * 0.02
    sd['filter_linear.bias'] = torch.randn(2, generator=g) * 0.05
    H, dh = config.hidden_size, config.hidden_size // config.num_attention_heads
    sharp, outlier, tails = kind in ('sharp', 'all'), kind in ('outlier', 'all'), kind in ('tails', 'all')
    D = list(OUTLIER_DIMS)
    for prefix in towers:
        u = torch.randn(H, generator=g)
        u /= u.norm()
        if sharp:
            sd[f'{prefix}.embeddings.position_embeddings.weight'][0] += u
        lns = [f'{prefix}.embeddings.LayerNorm']
        for l in range(config.num_hidden_layers):
            p = f'{prefix}.encoder.layer.{l}'
            lns += [f'{p}.attention.output.LayerNorm', f'{p}.output.LayerNorm']
            if sharp:
                Wq, Wk, bq = (sd[f'{p}.attention.self.{n}'] for n in ('query.weight', 'key.weight', 'query.bias'))
                for h, scale in SHARP_SELF_HEADS.items():
                    Wk[h * dh:(h + 1) * dh] = scale * Wq[h * dh:(h + 1) * dh] + 0.2 * Wk[h * dh:(h + 1) * dh]
                for h in SHARP_POS0_HEADS:
                    Wk[h * dh] += 2.0 * u
                    bq[h * dh] = 2.0
            if outlier:
                sd[f'{p}.output.dense.bias'][D] += torch.tensor([3.0, -3.0, 2.0])
            if tails:
                sd[f'{p}.intermediate.dense.weight'] *= 2.5
                sd[f'{p}.output.dense.weight'] *= 2.0
                for n in ('attention.output.LayerNorm', 'output.LayerNorm'):
                    sd[f'{p}.{n}.weight'] *= 1.0 + 0.1 * l
        if outlier:
            for n in lns:
                sd[f'{n}.weight'][D] = torch.tensor([6.0, 8.0, 10.0]) * sd[f'{n}.weight'][D].sign()
                sd[f'{n}.bias'][D] = torch.tensor([4.0, -3.0, 5.0])
    return sd
