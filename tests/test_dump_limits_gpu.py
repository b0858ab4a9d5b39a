"""The phrase dump's device step (dph_dump_select) at its bounds, byte for byte against oracle/dump_ref.select_document.

Sizes: 16 features of S = 512 with rows [1, 511) in one batch (8 160 rows, eight rounds of the 1024-row scan), kept rows at the
round boundary (batch rows 1023 and 1024), every row kept, none, and every other row.  Quantisation: the x values of
tests/test_rc_limits_cpu.quant_values ((x - offset) * scale in fp32 on k + 0.5, on 126.5 / 127.5 / -127.5 / -128.5, past the
clip, on -0.0 and on +-inf).  Threshold: logits at fp32(thr) and its neighbours, and filter_start at -999999 and just above it
(the fallback).  Layout: empty features at the start, middle and end of a document, a document of empty features only,
row_lo == row_hi == S, start2end at the end of a feature with L = 64, a fallback document that spans batches and keeps rows in a
later batch.  Output buffer: exactly dph_dump_layout bytes, followed by a guard that must stay untouched; one byte less raises."""
import numpy as np
import pytest
import torch

from densephrases_b200 import dump
from oracle import dump_ref
from tests.test_rc_limits_cpu import dump_quant_case, dump_thr_case

pytestmark = pytest.mark.gpu
f32 = np.float32


def run_documents(start, filt, lo, hi, doc_of, B, L, thr, off, scale):
    """Feed features (start [F,S,768], filt [F,S,2], rows [lo, hi), document of each) to DumpSelect in batches of B, carrying
    kept counts and the fallback across batches as dump_documents does; check each document against the oracle."""
    n_feat, n_docs = len(lo), int(doc_of.max()) + 1
    sel = dump.DumpSelect(L, thr, off, scale)
    kept, rows, fb = [0] * n_docs, [0] * n_docs, {}
    got = [([], [], []) for _ in range(n_docs)]
    for b0 in range(0, n_feat, B):
        idx = np.arange(b0, min(b0 + B, n_feat))
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
                fb[g0 + s] = (r['fb_rows'][r['fb_slot'][s]][None], np.array([r['fb_f2o'][s]], np.int64))
        assert at == r['n_kept']
    for d in range(n_docs):
        ii = np.flatnonzero(doc_of == d)
        cat = lambda a: np.concatenate([a[i, lo[i]:hi[i]] for i in ii])          # noqa: E731
        with np.errstate(over='ignore', invalid='ignore'):
            q, f2o, s2e = dump_ref.select_document(cat(start), cat(filt[..., 0]), cat(filt[..., 1]), hi[ii] - lo[ii], L, thr, off, scale)
        want = (q, f2o, s2e)
        if kept[d]:
            mine = [np.concatenate(x) for x in got[d]]
        elif d in fb:
            mine, want = fb[d], (q, f2o)                    # a fallback row's start2end is built on the host
        else:
            mine = [np.zeros((0, 768), np.int8), np.zeros(0, np.int64), np.zeros((0, L), np.int32)]
        for m, w, k in zip(mine, want, ('rows', 'f2o', 'start2end')):
            assert m.dtype == w.dtype and m.shape == w.shape and m.tobytes() == w.tobytes(), (d, k, B)
    return kept, fb


def features(F, S, seed, lo=1, hi=None):
    rng = np.random.default_rng(seed)
    start = (rng.standard_normal((F, S, 768)) * 3).astype(np.float32)
    filt = (np.round(rng.normal(size=(F, S, 2)) * 4) / 4).astype(np.float32)
    return start, filt, np.full(F, lo), np.full(F, S - 1 if hi is None else hi)


@pytest.mark.parametrize('pattern', ['all', 'none', 'alternate', 'round_edge'])
def test_eight_scan_rounds(pattern):
    """B = 16 at S = 512, rows [1, 511): 8 160 rows in one batch, one document and four documents."""
    F, S = 16, 512
    start, filt, lo, hi = features(F, S, 1)
    flat = np.zeros((F, S - 2), bool)
    if pattern == 'all':
        flat[:] = True
    elif pattern == 'alternate':
        flat.ravel()[::2] = True
    elif pattern == 'round_edge':
        flat.ravel()[[1023, 1024, 2047, 8159]] = True
    filt[:] = -3.0
    filt[:, 1:S - 1, 0] = np.where(flat, 1.0, -3.0)
    assert F * (S - 2) == 8160
    for doc_of in (np.zeros(F, int), np.repeat(np.arange(4), 4)):
        kept, fb = run_documents(start, filt, lo, hi, doc_of, 16, 10, 0.0, -2.0, 20.0)
        assert sum(kept) == int(flat.sum()) and (pattern != 'none' or len(fb) == doc_of.max() + 1)


@pytest.mark.parametrize('off,scale', [(-2.0, 20.0), (0.1, 4.0), (0.0, 1e37)])
def test_quantisation_edges(off, scale):
    """Every row kept; rows hold the quantisation edge values and their fp32 neighbours."""
    rows = dump_quant_case(off, scale)
    F, S = 2, 64
    start = np.resize(rows, (F * S, 768)).reshape(F, S, 768).astype(np.float32)
    filt = np.ones((F, S, 2), np.float32)
    run_documents(start, filt, np.array([1, 0]), np.array([63, 64]), np.zeros(F, int), 2, 64, 0.0, off, scale)


@pytest.mark.parametrize('thr', [0.1, 0.7, -2.0])
def test_threshold_edges(thr):
    """Logits at fp32(thr) and its two neighbours (kept only strictly above fp32(thr)); documents with nothing kept take the
    first row with filter_start > -999999 (exactly -999999 does not qualify)."""
    rng = np.random.default_rng(int(abs(thr) * 10))
    F, S = 12, 48
    start, _, lo, hi = features(F, S, 5)
    vals = dump_thr_case(thr)
    filt = rng.choice(vals, (F, S, 2)).astype(np.float32)
    low = vals[vals <= f32(thr)]
    filt[6:9] = rng.choice(low, (3, S, 2))                               # document 2: nothing above the threshold
    filt[6:9, :, 0] = f32(-999999.0)
    filt[7, 20, 0] = np.nextafter(f32(-999999.0), f32(0))               # its fallback row
    filt[9:] = rng.choice(low, (3, S, 2))                                # document 3: no row qualifies for the fallback either
    filt[9:, :, 0] = f32(-999999.0)
    doc_of = np.repeat(np.arange(4), 3)
    for B in (1, 5, 12):
        kept, fb = run_documents(start, filt, lo, hi, doc_of, B, 8, thr, -2.0, 20.0)
        assert kept[2] == 0 and kept[3] == 0 and 2 in fb and 3 not in fb and kept[0] and kept[1]


def test_layout_edges():
    """Empty features (row_lo == row_hi) at a document's start, middle and end, a document of empty features only, row_lo ==
    row_hi == S, start2end across a feature's last rows with L = 64, and a fallback document whose rows are kept one batch later."""
    F, S = 14, 96
    start, filt, lo, hi = features(F, S, 9)
    lo[:], hi[:] = 1, S - 1
    lo[0] = hi[0] = 5                      # document 0: empty first feature
    lo[2] = hi[2] = 0                      # ... middle
    lo[3] = hi[3] = S                      # ... last, at S
    lo[4:6] = hi[4:6] = 7                  # document 1: only empty features
    hi[6] = 70                             # document 2: feature end inside the row range; every row kept
    filt[6:8] = 1.0
    filt[8:11] = -3.0                      # document 3: nothing kept in features 8-10 (fallback candidates) ...
    filt[11] = -3.0
    filt[11, 30, 1] = 1.0                  # ... one row kept in feature 11
    doc_of = np.array([0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 3, 3, 4, 4])
    for B in (1, 3, 9, 14):
        kept, fb = run_documents(start, filt, lo, hi, doc_of, B, 64, 0.0, -2.0, 20.0)
        assert kept[1] == 0 and 1 not in fb and kept[3] == 1


def test_output_buffer_exact_size_and_guard():
    """out_bytes == dph_dump_layout: the call fills it and leaves the guard behind it untouched; one byte less raises."""
    import ctypes as C
    from densephrases_b200 import _lib as L
    F, S, Lm = 3, 64, 64
    start, filt, lo, hi = features(F, S, 11)
    filt[:] = 1.0
    feat = np.array([(1, 63, 0, 0), (1, 63, 0, 62), (0, 64, 1, 0)], np.int32)
    doc = np.array([(0, 1), (0, 1)], np.int32)
    R = int((feat[:, 1] - feat[:, 0]).sum())
    offs = np.zeros(7, np.int64)
    need = int(L.lib().dph_dump_layout(R, 2, Lm, offs.ctypes.data))
    buf = torch.full((need + 4096,), 0xA5, dtype=torch.uint8, pin_memory=True)
    s, f = torch.from_numpy(start).cuda(), torch.from_numpy(np.ascontiguousarray(filt)).cuda()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = lambda n: L.lib().dph_dump_select(s.data_ptr(), f.data_ptr(), F, S, feat.ctypes.data, 2, doc.ctypes.data, Lm, 0.0, -2.0, 20.0,   # noqa: E731
                                             buf.data_ptr(), n, stream)
    L.check(call(need))
    torch.cuda.synchronize()
    raw = buf.numpy()
    assert int(raw[:8].view(np.int64)[0]) == R and (raw[need:] == 0xA5).all()
    with pytest.raises(RuntimeError, match='smaller than dph_dump_layout'):
        L.check(call(need - 1))
