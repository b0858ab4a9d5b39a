"""Single-passage reading and the phrase dump at their limits, on the CPU.

- compute_predictions_logits where an example's n-best list needs more than the decoder's 1024 candidates: the spans of such an
  example are enumerated on the host (rc.host_spans).  With the numpy span oracle standing in for the GPU decoder, the host path
  reproduces the unmodified reference (tests/golden/rc_limits.json.gz, made by tests/golden/make_rc_limits_golden.py).
- The decoder's edge cases (DECODER_CASES, also run on the GPU by tests/test_rc_limits_gpu.py): each case asserts it reaches what
  it claims, and the numpy oracle oracle/rc_ref.py and rc.host_spans agree with a plain-Python statement of the reference's
  double loop and its sorted(..., key=start + end, reverse=True).
- The dump step's edge values (DUMP_CASES, also run on the GPU by tests/test_dump_limits_gpu.py): oracle/dump_ref.select_document
  agrees with a plain-Python statement of filter_metadata and compress_metadata (fp32 comparisons and arithmetic, round half to
  even)."""
import gzip
import json
import os

import numpy as np
import pytest

from tests import rc_cases

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'rc_limits.json.gz')
with gzip.open(GOLD, 'rt') as _f:
    LIMIT_CASES = json.load(_f)['configs']
LIMIT_RUNS = [(c['name'], r['filter_threshold']) for c in LIMIT_CASES for r in c['runs']]
HOST_FINISH = {'repeat_word_200': True, 'repeat_word_200_v2': True, 'overlap_windows': True, 'z_at_candidate_1024': False,
               'z_at_candidate_1025': True}
f32 = np.float32


# ---- n-best beyond 1024 candidates ---------------------------------------------------------------------------------------------
def limit_run(rc, name, thr, tmp):
    case = next(c for c in LIMIT_CASES if c['name'] == name)
    run = next(r for r in case['runs'] if r['filter_threshold'] == thr)
    _, _, logits = rc_cases.objects(case)
    return case, run, rc_cases.run(rc, case, thr, tmp, tuple(logits))


@pytest.mark.parametrize('name,thr', LIMIT_RUNS)
def test_nbest_beyond_1024_candidates_matches_reference(name, thr, tmp_path, monkeypatch):
    from densephrases_b200 import rc
    from oracle import rc_ref
    ks, host, host_spans = [], [], rc.host_spans
    monkeypatch.setattr(rc, 'best_spans', lambda *a: ks.append(a[10]) or rc_ref.best_spans(*a))
    monkeypatch.setattr(rc, 'host_spans', lambda *a: host.append(1) or host_spans(*a))
    case, run, (preds, stat, files) = limit_run(rc, name, thr, str(tmp_path))
    assert preds == run['predictions'] and stat == run['stat'] and files == run['files']
    if thr < -1e7:
        assert bool(host) == HOST_FINISH[name], 'the case must (not) need more than 1024 candidates'
        assert max(ks) == 1024, 'the decoder is asked for 1024 candidates before the host takes over'


def test_limit_fixture_cases():
    """The fixture reaches what make_rc_limits_golden.py claims: 'z' is the n-best's second entry, and a repeated word gives 9 texts."""
    for c in LIMIT_CASES:
        nbest = json.loads(c['runs'][0]['files']['nbest'])['q0']
        if c['name'].startswith('z_at'):
            assert [e['text'] for e in nbest] == ['w', 'z']
        elif c['name'].startswith('repeat_word'):
            assert sorted(e['text'] for e in nbest) == sorted(['', *(' '.join(['w'] * n) for n in range(1, 10))][not c['version_2']:])
    assert os.path.getsize(GOLD) < 256 * 1024


# ---- the span decoder's edge cases ---------------------------------------------------------------------------------------------
def all_bits(F, S):
    return np.full((F, (S + 31) // 32), 0xffffffff, np.uint32)


def decoder_case(logits, ex_off=None, n_tokens=None, start_ok=None, end_ok=None, L=10, thr=-1e30, K=1024, v2=False):
    F, S = logits[0].shape
    end_ok = all_bits(F, S) if end_ok is None else end_ok
    start_ok = (all_bits(F, S) if start_ok is None else start_ok) & end_ok     # a start is in token_to_orig_map too
    return dict(logits=[np.ascontiguousarray(x, np.float32) for x in logits], n_tokens=np.full(F, S, np.int32) if n_tokens is None else
                np.asarray(n_tokens, np.int32), start_ok=start_ok, end_ok=end_ok, ex_off=np.array([0, F], np.int64) if ex_off is None else
                np.asarray(ex_off, np.int64), L=L, thr=thr, K=K, v2=v2)


def bits_of(F, S, pos):
    m = np.zeros((F, (S + 31) // 32), np.uint32)
    for f, p in pos:
        m[f, p >> 5] |= np.uint32(1) << np.uint32(p & 31)
    return m


def _tie_count_case(K, V):
    """every logit 0 (every span ties), L = 2 (one span per valid position), exactly V valid positions over features of S = 512"""
    S = 512
    F = max(1, -(-V // 500))
    pos = [(i // 500, i % 500) for i in range(V)]
    m = bits_of(F, S, pos)
    z = np.zeros((F, S), np.float32)
    return decoder_case([z, z, z, z], start_ok=m, end_ok=m, L=2, K=K)


def _cases():
    rng = np.random.default_rng(2024)
    c = {}
    # score arithmetic
    big = rng.uniform(-3.4e38, 3.4e38, (4, 2, 64)).astype(np.float32)
    big[:, :, ::3] = rng.choice(np.array([3.0e38, 3.2e38, 3.4e38, 3.1e38], np.float32), (4, 2, 22))
    c['overflow'] = decoder_case([big[0], big[1], big[2] * 0, big[3] * 0], ex_off=[0, 1, 2], L=64, K=300)
    base = np.where(rng.random((3, 96)) < 0.5, f32(1e8), f32(-1e8)).astype(np.float32)
    small = rng.choice(np.array([0.0, 1.0, 2.0, 3.0, 0.5, -1.0], np.float32), (3, 96))
    c['close_1e8'] = decoder_case([base, small, small, small], L=12, K=500)
    sub = rng.choice(np.array([1e-45, 2e-45, 1e-40, -1e-40, 5e-39, -1e-45, 0.0, 1.17e-38], np.float32), (4, 2, 80))
    c['subnormal'] = decoder_case(list(sub), L=20, K=1024)
    zs = rng.choice(np.array([0.0, -0.0], np.float32), (2, 2, 70))
    zs[:, :, ::17] = 1.0
    c['signed_zero'] = decoder_case([zs[0], zs[1], np.zeros((2, 70), np.float32), np.zeros((2, 70), np.float32)], L=8, K=700)
    # ties across the cut: K at the cap doubling edges, vec_count at K - 1, K, K + 1
    for K in (1, 256, 257, 768, 769, 1024):
        for dv in (-1, 0, 1):
            if K + dv >= 1:
                c[f'ties_K{K}_V{K + dv}'] = _tie_count_case(K, K + dv)
    z = np.zeros((1, 512), np.float32)
    c['ties_all_L64'] = decoder_case([z, z, z, z], L=64, K=1024)
    rise = np.arange(512, dtype=np.float32)[None]
    for K in (256, 257, 1024):                    # scores rise with the end index: most rounds beat the running K-th entry
        c[f'rising_K{K}'] = decoder_case([z, rise, z, z], L=64, K=K)
    # filter threshold
    for thr in (0.1, 1 / 3, 0.7, 0.9):
        t = f32(thr)
        vals = np.array([np.nextafter(t, f32(-1)), t, np.nextafter(t, f32(1))], np.float32)
        sf, ef = rng.choice(vals, (2, 2, 48))
        c[f'thr_{thr:.4f}'] = decoder_case([rng.normal(size=(2, 48)), rng.normal(size=(2, 48)), sf, ef], L=6, thr=thr, K=200)
    eq = np.round(rng.normal(size=(2, 40)) * 2) / 2
    c['thr_equal_logit'] = decoder_case([rng.normal(size=(2, 40)), rng.normal(size=(2, 40)), eq, eq], L=5, thr=0.5, K=100)
    c['thr_keep_all'] = decoder_case([rng.normal(size=(2, 40)), rng.normal(size=(2, 40)), eq, eq], L=5, thr=-1e30, K=100)
    c['thr_keep_none'] = decoder_case([rng.normal(size=(2, 40)), rng.normal(size=(2, 40)), eq, eq], L=5, thr=1e30, K=100)
    # layout
    lg = [rng.normal(size=(6, 64)) for _ in range(4)]
    sok, eok = all_bits(6, 64), all_bits(6, 64)
    sok[3] = 0
    eok[4] = 0
    c['layout_ntok_0_1'] = decoder_case(lg, ex_off=[0, 2, 3, 6], n_tokens=[0, 1, 64, 64, 64, 1], start_ok=sok, end_ok=eok, L=10, K=50, v2=True)
    c['layout_L1'] = decoder_case(lg, L=1, K=5)
    c['layout_L2'] = decoder_case(lg, L=2, K=64)
    many = [rng.normal(size=(230, 32)) for _ in range(4)]
    nt = rng.integers(0, 33, 230)
    c['layout_100_features'] = decoder_case(many, ex_off=[0, 1, 121, 123, 230], n_tokens=nt, L=16, K=1024, v2=True,
                                            start_ok=rng.integers(0, 2 ** 32, (230, 1), dtype=np.uint64).astype(np.uint32))
    # version-2 null
    st0 = rng.normal(size=(5, 16)).astype(np.float32)
    en0 = rng.normal(size=(5, 16)).astype(np.float32)
    st0[:, 0], en0[:, 0] = [2.0, -1.0, 0.5, -1.0, -1.0], [1.0, 0.25, -0.25, 0.25, 0.25]   # features 1, 3, 4 tie at -0.75
    c['null_tie'] = decoder_case([st0, en0, st0, en0], L=4, K=20, v2=True)
    n1, n2 = st0.copy(), en0.copy()
    n1[:, 0], n2[:, 0] = [5e5, 1e6, 1e6, 4e5, 2e6], [5e5, 0.0, 1.0, 6e5, -5e5]          # sums 1e6, 1e6, 1e6 + 1, 1e6, 1.5e6
    c['null_at_1e6'] = decoder_case([n1, n2, n1, n2], ex_off=[0, 1, 3, 5], L=4, K=20, v2=True)
    n3, n4 = n1.copy(), n2.copy()
    n4[0, 0] = np.nextafter(f32(5e5), f32(0))                                                # just below 1e6: chosen
    c['null_below_1e6'] = decoder_case([n3, n4, n3, n4], ex_off=[0, 1, 3, 5], L=4, K=20, v2=True)
    return c


DECODER_CASES = _cases()


def plain_prelim(c):
    """The reference's enumeration and ordering in plain Python -> per example (spans [(f, s, e)] best first, total, kept, null)."""
    st, en, sf, ef = (x.tolist() for x in c['logits'])            # Python floats, as SquadResult holds them
    bit = lambda m, f, i: (int(m[f, i >> 5]) >> (i & 31)) & 1      # noqa: E731
    out = []
    for x in range(len(c['ex_off']) - 1):
        spans, total, null, best = [], 0, -1, 1000000
        for fi, f in enumerate(range(int(c['ex_off'][x]), int(c['ex_off'][x + 1]))):
            if c['v2'] and st[f][0] + en[f][0] < best:
                best, null = st[f][0] + en[f][0], fi
            n = int(c['n_tokens'][f])
            for s in range(n):
                for e in range(s, min(n, s + c['L'] - 1)):
                    if not (bit(c['end_ok'], f, s) and bit(c['end_ok'], f, e) and bit(c['start_ok'], f, s)):
                        continue
                    total += 1
                    if sf[f][s] < c['thr'] or ef[f][e] < c['thr']:
                        continue
                    spans.append((fi, s, e, st[f][s] + en[f][e]))
        spans = sorted(spans, key=lambda p: p[3], reverse=True)
        out.append(([p[:3] for p in spans], total, len(spans), null))
    return out


def oracle_spans(c, k=None):
    from oracle import rc_ref
    return rc_ref.best_spans(*c['logits'], c['n_tokens'], c['start_ok'], c['end_ok'], c['ex_off'], c['L'], c['thr'],
                             c['K'] if k is None else k, c['v2'])


def test_decoder_cases_reach_their_claims():
    c = DECODER_CASES
    st, en = (x.astype(np.float32) for x in c['overflow']['logits'][:2])
    with np.errstate(over='ignore'):
        s32 = st[:, :, None] + en[:, None, :]
    s64 = st.astype(np.float64)[:, :, None] + en.astype(np.float64)[:, None, :]
    assert np.isinf(s32).sum() > 100 and np.isfinite(s64).all() and np.abs(s64).max() > 6e38
    st, en = (x.astype(np.float32) for x in c['close_1e8']['logits'][:2])
    assert (st[0, 1] + en[0, 2:10]).tolist().count(float(st[0, 1])) > 1 and len(set((st[0, 1].astype(np.float64) + en[0, 2:10]).tolist())) > 1
    st = c['subnormal']['logits'][0]
    assert ((st != 0) & (np.abs(st) < np.finfo(np.float32).tiny)).sum() > 50
    st, en = c['signed_zero']['logits'][:2]
    sums = (st[:, :, None] + en[:, None, :]).ravel()
    assert (np.signbit(sums) & (sums == 0)).sum() > 100 and (~np.signbit(sums) & (sums == 0)).sum() > 100
    for name, cs in c.items():
        if name.startswith('ties_K'):
            r = oracle_spans(cs)
            K, V = (int(p[1:]) for p in name.split('_')[1:])
            assert int(r.vec_count[0]) == V and int(r.n_cand[0]) == min(K, V)
    for name in ('rising_K256', 'rising_K257', 'rising_K1024', 'ties_all_L64'):
        cap = 512
        while cap < c[name]['K'] + 256:
            cap *= 2
        assert int(oracle_spans(c[name]).vec_count[0]) > 10 * cap                # the buffer is cut to K many times
    down = [t for t in (0.1, 1 / 3, 0.7, 0.9) if float(f32(t)) < t]
    up = [t for t in (0.1, 1 / 3, 0.7, 0.9) if float(f32(t)) > t]
    assert down and up                                          # fp32(thr) on both sides of thr: the double comparison shows
    r = oracle_spans(c['thr_equal_logit'])
    assert 0 < r.vec_count.sum() < r.total_count.sum() and (c['thr_equal_logit']['logits'][2] == 0.5).any()
    assert (oracle_spans(c['thr_keep_all']).vec_count == oracle_spans(c['thr_keep_all']).total_count).all()
    assert (oracle_spans(c['thr_keep_none']).vec_count == 0).all() and (oracle_spans(c['thr_keep_none']).total_count > 0).all()
    assert (oracle_spans(c['layout_L1']).total_count == 0).all()
    r = oracle_spans(c['layout_100_features'])
    assert np.diff(c['layout_100_features']['ex_off']).max() >= 100 and r.vec_count.max() > 1024
    assert oracle_spans(c['null_tie']).null_feature.tolist() == [1]
    assert oracle_spans(c['null_at_1e6']).null_feature.tolist() == [-1, -1, -1]
    assert oracle_spans(c['null_below_1e6']).null_feature.tolist() == [0, -1, -1]


@pytest.mark.parametrize('name', list(DECODER_CASES))
def test_span_oracle_and_host_spans_match_plain_reference(name):
    """oracle/rc_ref.py (first K) and rc.host_spans (every span) against the reference's loop and sort stated in plain Python."""
    from densephrases_b200 import rc
    c = DECODER_CASES[name]
    want = plain_prelim(c)
    r = oracle_spans(c)
    for x, (spans, total, kept, null) in enumerate(want):
        a, b = int(c['ex_off'][x]), int(c['ex_off'][x + 1])
        assert int(r.total_count[x]) == total and int(r.vec_count[x]) == kept and int(r.null_feature[x]) == (null if c['v2'] else -1)
        assert r.cand[x, :r.n_cand[x]].tolist() == [list(p) for p in spans[:c['K']]]
        h = rc.host_spans(*(x_[a:b] for x_ in c['logits']), c['n_tokens'][a:b], c['start_ok'][a:b], c['end_ok'][a:b], c['L'], c['thr'])
        assert h.dtype == np.int32 and h.tolist() == [list(p) for p in spans]


# ---- the dump step's edge values ----------------------------------------------------------------------------------------------
def plain_select(start, fs, fe, rows_per_feature, L, thr, off, scale):
    """filter_metadata + compress_metadata of one document in plain Python: numpy compares a float32 array with a Python float
    in float32 and computes (x - offset) * scale in float32; np.round rounds half to even (Python's round does too)."""
    t32 = float(f32(thr))
    T = len(fs)
    s_set = {i for i in range(T) if float(fs[i]) > t32}
    e_set = {i for i in range(T) if float(fe[i]) > t32}
    keep = sorted(s_set | e_set)
    end_short = {r: k for k, r in enumerate(keep) if r in e_set}
    if not keep:
        keep = [i for i in range(T) if float(fs[i]) > -999999.0][:1]
        end_short = {r: k for k, r in enumerate(keep)}
    feat_end, at = [], 0
    for n in rows_per_feature:
        feat_end += [at + n] * n
        at += n
    s2e = [[end_short.get(r + j, -1) if r + j < feat_end[r] else -1 for j in range(L)] for r in keep]
    o32, sc32 = f32(off), f32(scale)
    q = []
    for r in keep:
        row = []
        for v in start[r]:
            with np.errstate(over='ignore'):
                y = float((f32(v) - o32) * sc32)
            row.append(int(round(min(max(y, -128.0), 127.0))))
        q.append(row)
    return np.array(q, np.int8).reshape(len(keep), 768), np.array(keep, np.int64), np.array(s2e, np.int32).reshape(len(keep), L)


def quant_values(off, scale):
    """fp32 x values whose (x - off) * scale lands on k + 0.5, on 126.5 / 127.5 / -127.5 / -128.5, past the clip, on -0.0 (x = -0.0
    with off = 0) and on +-inf before the clip, each with its two fp32 neighbours."""
    o, s = f32(off), f32(scale)
    targets = [k + 0.5 for k in range(-129, 128)] + [-0.0, 0.0, 300.0, -300.0, 1e30, -1e30]
    xs = [f32(t) / s + o for t in targets] + [f32(3e38), f32(-3e38), f32(-0.0)]
    out = []
    for x in xs:
        x = f32(x)
        out += [np.nextafter(x, f32(-np.inf)), x, np.nextafter(x, f32(np.inf))]
    return np.array(out, np.float32)


def dump_quant_case(off, scale):
    """start rows filled with quant_values (padded with repeats) -> fp32 [T,768]."""
    v = quant_values(off, scale)
    T = -(-len(v) // 768) + 1
    return np.resize(v, (T, 768)).astype(np.float32)


def dump_thr_case(thr):
    t = f32(thr)
    vals = np.array([np.nextafter(t, f32(-np.inf)), t, np.nextafter(t, f32(np.inf)), f32(-999999.0),
                     np.nextafter(f32(-999999.0), f32(0)), f32(-1e7)], np.float32)
    return vals


def test_dump_quant_values_reach_their_claims():
    with np.errstate(over='ignore'):
        for off, scale in ((-2.0, 20.0), (0.1, 4.0), (0.0, 1e37)):
            v = quant_values(off, scale)
            y = (v - f32(off)) * f32(scale)
            assert y.dtype == np.float32
            frac = np.where(np.isfinite(y), y - np.floor(np.where(np.isfinite(y), y, 0)), 0)
            assert ((frac == 0.5) & (np.abs(y) < 128)).sum() >= (20 if scale < 1e30 else 0)
            for t in (126.5, 127.5, -127.5, -128.5) if scale < 1e30 else ():
                assert (y == t).any(), (off, scale, t)
            assert (y > 127).any() and (y < -128).any() and ((y == 0) & (np.signbit(y) == (off == 0.0))).any()
            if scale > 1e30:
                assert np.isinf(y).any()


@pytest.mark.parametrize('off,scale', [(-2.0, 20.0), (0.1, 4.0), (0.0, 1e37)])
@pytest.mark.parametrize('thr', [0.1, 0.7, -2.0, 1e30])
def test_dump_oracle_matches_plain_reference(off, scale, thr):
    """oracle/dump_ref.select_document against plain_select: quantisation edges, fp32 thresholds and the -999999 fallback."""
    from oracle import dump_ref
    rng = np.random.default_rng(int(scale) % 1000 + int(thr * 10) % 97)
    start = dump_quant_case(off, scale)
    T = len(start)
    vals = dump_thr_case(thr)
    fs, fe = rng.choice(vals, T), rng.choice(vals, T)
    rows = [T // 3, 0, T - T // 3]
    for L in (1, 7, 64):
        for fs_, fe_ in ((fs, fe), (np.full(T, f32(-999999.0)), fe * 0 - 1e7),
                         (np.where(np.arange(T) == T - 2, np.nextafter(f32(-999999.0), f32(0)), f32(-999999.0)), np.full(T, f32(-1e7)))):
            with np.errstate(over='ignore', invalid='ignore'):
                got = dump_ref.select_document(start, fs_, fe_, rows, L, thr, off, scale)
            want = plain_select(start, fs_, fe_, rows, L, thr, off, scale)
            for g, w in zip(got, want):
                assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes()
