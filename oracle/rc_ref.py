"""oracle/rc_ref.py -- TEST INFRASTRUCTURE.  Plain numpy restatement of the span enumeration of the reference's
compute_predictions_logits (densephrases/utils/squad_metrics.py:490-544, 547-557, 569-571) with the interface of
densephrases_b200.rc.best_spans (the binding of dph_rc_spans): per example the first K prelim candidates in the reference's
order, the valid-span counts before and after the filter, and the version-2 null choice.  tests/test_rc_cpu.py pins it against
the unmodified reference (tests/golden/rc_reference.json.gz)."""
import numpy as np


def best_spans(start, end, sft, eft, n_tokens, start_ok, end_ok, ex_off, max_answer_length, filter_threshold, k, version_2=False):
    """Same arguments and result fields as densephrases_b200.rc.best_spans (numpy in, numpy out)."""
    from densephrases_b200.rc import Spans
    st, en, sf, ef = (np.asarray(x, dtype=np.float32) for x in (start, end, sft, eft))
    n_tokens, ex_off = np.asarray(n_tokens, np.int64), np.asarray(ex_off, np.int64)
    start_ok, end_ok = np.asarray(start_ok).view(np.uint32), np.asarray(end_ok).view(np.uint32)
    F, S = st.shape
    E, L, thr = len(ex_off) - 1, int(max_answer_length), float(filter_threshold)
    bit = lambda m, f, i: bool((int(m[f, i >> 5]) >> (i & 31)) & 1)          # noqa: E731
    out = dict(cand=np.zeros((E, k, 3), np.int32), n_cand=np.zeros(E, np.int32), total_count=np.zeros(E, np.int64),
               vec_count=np.zeros(E, np.int64), null_feature=np.full(E, -1, np.int32), null_logits=np.zeros((E, 2), np.float32))
    for x in range(E):
        fs, ss, es, scores = [], [], [], []
        total = 0
        for fi, f in enumerate(range(ex_off[x], ex_off[x + 1])):
            n = int(n_tokens[f])
            for s in range(n):
                if not bit(start_ok, f, s):
                    continue
                e = np.arange(s, min(n, s + L - 1))
                e = e[[bit(end_ok, f, int(i)) for i in e]] if len(e) else e
                total += len(e)
                if float(sf[f, s]) < thr:
                    continue
                e = e[~(ef[f, e].astype(np.float64) < thr)]
                fs += [fi] * len(e)
                ss += [s] * len(e)
                es += e.tolist()
                scores += (float(st[f, s]) + en[f, e].astype(np.float64)).tolist()
        scores = np.asarray(scores, np.float64) + 0.0              # -0.0 ranks with +0.0, as in Python's comparison
        order = np.lexsort((np.arange(len(scores)), -scores))     # score descending, then enumeration order
        m = min(k, len(order))
        out['cand'][x, :m] = np.stack([np.asarray(fs)[order[:m]], np.asarray(ss)[order[:m]], np.asarray(es)[order[:m]]], 1) if m else 0
        out['n_cand'][x], out['total_count'][x], out['vec_count'][x] = m, total, len(scores)
        if version_2:
            best = 1000000.0
            for fi, f in enumerate(range(ex_off[x], ex_off[x + 1])):
                sc = float(st[f, 0]) + float(en[f, 0])
                if sc < best:
                    best = sc
                    out['null_feature'][x], out['null_logits'][x] = fi, (st[f, 0], en[f, 0])
    return Spans(**out)
