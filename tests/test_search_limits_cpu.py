"""Constructions that drive the grouped scan filters to their arithmetic limits, and CPU checks that they do what they claim.

The quad scan (four queries per gather) quantises every PQ table entry to 8 bits and adds four queries' entries in one 32-bit word;
the pair scan quantises to 10 bits (0 ... 682) and adds two queries' entries per word.  Both are exact only while the packed sums
stay inside their lanes, and the filter is sound only while eps covers the quantisation error.  The constructions here are built so
that, with A = I (xr = x), the PQ table of one chosen query is a table we choose entry by entry:
    pq[m][j] = u_m t[m, j] / |u_m|^2,  u_m = x_m   ->   LUT[m][j] = x_m . pq[m][j] ~= t[m, j].
  * saturated codes: every sub-quantizer has the same range, so the argmax bytes quantise to the largest level in all 96 lanes and
    the packed sums reach 96 * 255 (quad) and 96 * 682 (pair);
  * worst-case rounding: two sub-quantizers set the step, and every other entry a vector uses sits 0.49 step above a level (rounds
    down) or 0.51 step above it (rounds up), so a target and its competitors are reordered by the quantisation.
The quantisation is restated from lutq_kernel (prep.cu) in fp32.  The GPU tests (test_search_limits_gpu.py) run the same data."""
import numpy as np
import pytest

from oracle.ivfpq_ref import fma32, np_lut, np_matmul_nt_seq

M, KSUB, DSUB, D = 96, 256, 8, 768
QMAX = {4: 255, 2: 682}                # largest quantised level: quad (8-bit lanes), pair (10-bit entries in 16-bit lanes)
QUAD_KEEP_MAX, PAIR_KEEP_MAX = 256, 1024


def keep_quad(k):
    return k + max(2 * k, 100)


def keep_pair(k):
    return k + max(k // 2, 32)


def quantise_lut(lut, qmax):
    """lutq_kernel restated: step = max(max_m range_m / QMAX, 1e-30) and inv = 1 / step in fp32, qv = (int)((entry - min_m) * inv
    + 0.5f) clamped to [0, QMAX].  The kernel's (e - min) * inv + 0.5f may be contracted to one FMA; both roundings are returned
    so that a construction can require them to agree.  Returns (qv_fma, qv_two_roundings, step, base = sum_m min_m)."""
    lut = np.asarray(lut, dtype=np.float32)
    lo, hi = lut.min(axis=1), lut.max(axis=1)
    r = np.max((hi - lo).astype(np.float32))
    step = np.maximum(np.float32(r) / np.float32(qmax), np.float32(1e-30)).astype(np.float32)
    inv = np.float32(np.float32(1.0) / step)
    d = (lut - lo[:, None]).astype(np.float32)
    half = np.float32(0.5)
    q_fma = fma32(d, np.full_like(d, inv), np.full_like(d, half))
    q_two = ((d * inv).astype(np.float32) + half).astype(np.float32)
    conv = lambda v: np.clip(np.trunc(v).astype(np.int64), 0, qmax)
    return conv(q_fma), conv(q_two), step, float(lo.astype(np.float64).sum())


def built_codebooks(x, t):
    """pq[m][j] = u_m t[m, j] / |u_m|^2 with u_m the m-th 8-dim slice of x: the query's LUT entries are ~t[m, j]."""
    u = np.asarray(x, dtype=np.float64).reshape(M, DSUB)
    pq = u[:, None, :] * (np.asarray(t, dtype=np.float64)[:, :, None] / (u * u).sum(axis=1)[:, None, None])
    return pq.astype(np.float32)


def limit_query(seed):
    """A query with no zero 8-dim slice (every u_m is usable)."""
    x = np.random.default_rng(seed).standard_normal(D).astype(np.float32)
    assert (np.abs(x.reshape(M, DSUB)).sum(axis=1) > 0.1).all()
    return x


# ---- saturated codes ------------------------------------------------------------------------------------------------------
def saturating_codebooks(x, seed):
    """Codebooks whose LUT for x has the same range (0 ... 1) in all 96 sub-quantizers, maximum at a random code per sub-quantizer."""
    rng = np.random.default_rng(seed)
    t = rng.uniform(0.05, 0.95, (M, KSUB))
    t[:, 0] = 0.0
    jmax = rng.integers(1, KSUB, M)
    t[np.arange(M), jmax] = 1.0
    return built_codebooks(x, t)


def saturated_codes(x, pq):
    """The argmax code (every byte selects its sub-quantizer's largest LUT entry) and variants that differ in one or two bytes
    (there the argmin entry): rows [saturated, one byte off, two bytes off]."""
    lut = np_lut(x, pq)
    top, bot = lut.argmax(axis=1).astype(np.uint8), lut.argmin(axis=1).astype(np.uint8)
    one, two = top.copy(), top.copy()
    one[37] = bot[37]
    two[5] = bot[5]; two[90] = bot[90]
    return np.stack([top, one, two])


@pytest.mark.parametrize("group", [4, 2])
def test_saturated_codes_reach_the_packed_limits(group):
    """With equal LUT ranges the argmax vector's quantised sum is exactly 96 * QMAX: 24480 < 2^15 in a quad byte lane, 65472 < 2^16
    (64 counts of headroom) in a pair lane -- the largest sum either packed scan can meet."""
    qmax = QMAX[group]
    x = limit_query(3)
    pq = saturating_codebooks(x, 4)
    lut = np_lut(x, pq)
    rng_m = lut.max(axis=1) - lut.min(axis=1)
    assert np.abs(rng_m / rng_m.max() - 1).max() < 1e-5, "ranges must be equal for every lane to saturate"
    q_fma, q_two, _, _ = quantise_lut(lut, qmax)
    assert np.array_equal(q_fma, q_two)
    codes = saturated_codes(x, pq)
    sums = [int(q_fma[np.arange(M), c.astype(np.int64)].sum()) for c in codes]
    assert sums[0] == M * qmax
    assert sums[0] == (65472 if group == 2 else 24480)
    assert M * qmax * (1 if group == 2 else 2) < (1 << 16), "the limit itself fits its lane"
    assert sums[0] > sums[1] > sums[2] > 0.9 * M * qmax
    # and the saturated vector is the exact best of all codes
    exact = [float(lut[np.arange(M), c.astype(np.int64)].astype(np.float64).sum()) for c in codes]
    assert exact[0] > exact[1] > exact[2]


def test_saturated_codes_with_generated_codebooks(oracle):
    """With gen_pq codebooks the ranges differ: the argmax vector still has the largest sum, but below 96 * 255."""
    x = limit_query(3)
    pq = oracle.gen_pq(1234)
    lut = np_lut(x, pq)
    q, _, _, _ = quantise_lut(lut, 255)
    c = saturated_codes(x, pq)[0].astype(np.int64)
    s = int(q[np.arange(M), c].sum())
    assert s == int(q.max(axis=1).sum()) and s < M * 255


# ---- worst-case LUT rounding ------------------------------------------------------------------------------------------------
def rounding_case(group, seed=11):
    """Codebooks, a target code and a competitor code for the chosen query x (with A = I) such that
      * sub-quantizers 0 and 1 have range QMAX (step 1) and both codes select their entry 0 (value 0),
      * in the other 94 the target's entry lies 0.49 above a level (rounds down by 0.49 step) and the competitor's 0.51 above one
        (rounds up by 0.49 step); in 20 of them the target's level is one higher than the competitor's.
    Exact: target - competitor = 20 * 0.98 - 74 * 0.02 = 18.12 steps.  Quantised: target - competitor = 20 - 94 = -74 steps.
    Returns (x, pq, target_code, competitor_code)."""
    qmax = QMAX[group]
    rng = np.random.default_rng(seed)
    x = limit_query(seed)
    t = rng.uniform(0.0, 60.0, (M, KSUB))
    t[:, 0] = 0.0
    t[0:2, 1] = float(qmax)
    n_comp = rng.integers(5, 40, M)
    up = np.zeros(M, dtype=bool)
    up[rng.choice(np.arange(2, M), 20, replace=False)] = True
    n_tgt = n_comp + up
    t[2:, 1] = n_tgt[2:] + 0.49
    t[2:, 2] = n_comp[2:] + 0.51
    target = np.ones(M, np.uint8); target[:2] = 0
    comp = np.full(M, 2, np.uint8); comp[:2] = 0
    return x, built_codebooks(x, t), target, comp


def filter_and_exact(x, pq, codes, qmax):
    """(quantised filter score, exact canonical score) of each code row against query x; dis0 = 0 (zero centroid)."""
    lut = np_lut(x, pq)
    q, q2, step, base = quantise_lut(lut, qmax)
    assert np.array_equal(q, q2), "the construction must not depend on how the kernel rounds (e - min) * inv + 0.5"
    rows = np.asarray(codes).astype(np.int64)
    S = q[np.arange(M)[None, :], rows].sum(axis=1)
    filt = float(step) * S + base
    exact = np.zeros(len(rows), dtype=np.float32)
    for m in range(M):                                 # canonical m-ascending fp32 sum from dis0 = 0
        exact = (exact + lut[m, rows[:, m]]).astype(np.float32)
    return filt, exact, float(step), S


def eps_of(x, pq, qmax, coef=0.502):
    """plan_segs_kernel's eps for the grouped modes, dis0 = 0: 2 gamma_96 sum_m max|LUT_m| 1.01 + 96 coef step + 8e-6 sum_m max|LUT_m|."""
    lut = np_lut(x, pq)
    lsum = float(np.abs(lut).max(axis=1).astype(np.float64).sum())
    _, _, step, _ = quantise_lut(lut, qmax)
    return 2 * 5.7221e-6 * lsum * 1.01 + 96 * coef * float(step) + 8e-6 * lsum


@pytest.mark.parametrize("group,k", [(4, 1), (4, 10), (4, 85), (2, 86), (2, 300)])
def test_rounding_construction_reverses_the_order(group, k):
    """The quantisation puts the target 74 steps BELOW a competitor whose exact score is 18 steps below the target's.
      * with keep + 1 competitors in its list segment the target is dropped before the merge, and the proof must flag the query;
      * with k competitors the target stays in the buffer, and only eps (96 * 0.502 steps) brings it into the band the merge
        re-scores: 2 eps > 74 steps > 2 eps' for eps' with a quantisation term of 96 * 0.25 steps."""
    qmax = QMAX[group]
    keep = keep_quad(k) if group == 4 else keep_pair(k)
    assert keep <= (QUAD_KEEP_MAX if group == 4 else PAIR_KEEP_MAX)
    x, pq, target, comp = rounding_case(group)
    filt, exact, step, S = filter_and_exact(x, pq, np.stack([target, comp]), qmax)
    assert abs(step - 1.0) < 1e-5
    assert exact[0] > exact[1] and 17.5 < (exact[0] - exact[1]) / step < 19
    assert S[1] - S[0] == 74
    gap = filt[1] - filt[0]
    assert 73.9 * step < gap < 74.1 * step, "quantised: the competitor is tens of steps above the target"
    eps = eps_of(x, pq, qmax)
    assert 2 * eps > gap + step, "the true eps keeps the target in the re-scored band"
    assert 2 * eps_of(x, pq, qmax, coef=0.25) < gap - step, "a quantisation term of 0.25 step per entry would drop it"
    # every per-entry rounding error is close to its worst case
    lut = np_lut(x, pq)
    q, _, _, _ = quantise_lut(lut, qmax)
    for code, sign in ((target, -1), (comp, 1)):
        c = code.astype(np.int64)
        err = (q[np.arange(2, M), c[2:]] * step - lut[np.arange(2, M), c[2:]]) / step
        assert (sign * err > 0.48).all() and (sign * err < 0.5).all()


def test_sequential_matmul_helper_matches_numpy_definition(oracle):
    """The SGEMM tests take their reference from the C oracle's coarse scores; at small shapes it equals the numpy FMA chain."""
    from tests.test_sgemm_seq_gpu import seq_matmul_ref
    rng = np.random.default_rng(0)
    for n, m, K in ((3, 5, 32), (4, 9, 96), (2, 17, 768)):
        X = rng.standard_normal((n, K)).astype(np.float32)
        W = rng.standard_normal((m, K)).astype(np.float32)
        assert np.array_equal(seq_matmul_ref(X, W).view(np.int32), np_matmul_nt_seq(X, W).view(np.int32))
