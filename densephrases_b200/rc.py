"""Single-passage reading: answers from the start / end / filter logits of Encoder.forward with a context and a question.

Mirror of the reference's evaluation path of train_rc.py (:307-431): `compute_predictions_logits`
(densephrases/utils/squad_metrics.py:408-684) turns the logits of every SQuAD feature into answers and JSON files,
`squad_evaluate` (:221-254) scores them, and `filter_test` runs the filter-threshold sweep of `make filter-test`.

The span enumeration -- every (start, end) of every feature, S * (L - 1) pairs per feature -- runs on the GPU (`best_spans`,
csrc/spans.cu): per example it returns the first K prelim candidates in the reference's order (score float(start) + float(end)
descending, ties in enumeration order), the counts before and after the filter, and the version-2 null choice.  The host keeps
the text side: get_final_text, the softmax, the null handling, the "empty" nonce entries and the files.  The n-best loop skips
duplicate texts, so it can use up the K candidates of an example before it has n_best_size entries; that example is then decoded
again with 2K (up to 1024), and past 1024 its spans are enumerated on the host (host_spans), so the result stays exact.

Reference behaviour reproduced on purpose (pinned by tests/golden/rc_reference.json.gz):
- the end index runs up to start + max_answer_length - 2, so a span has at most max_answer_length - 1 tokens;
- `candidates` is never filled, so every `recall` is False, answer recall is 0 and each example's `save_rate` is 0.0;
- that per-example save_rate divides by the example's valid-span count, so an example without any valid span (or without
  features) raises ZeroDivisionError;
- a candidate starting at token 0 gets the text "" (only the null entry does in practice);
- in the non-null branch duplicates are skipped, but "" entries are not de-duplicated."""
import collections
import json
import logging
import math
import re
import string

import numpy as np
import torch

from . import _lib as L
from .tokenization import basic_tokenize

logger = logging.getLogger(__name__)

MAX_ANSWER_LENGTH = 64   # max_answer_length bound of dph_rc_spans
MAX_K = 1024             # candidates per example per call

Spans = collections.namedtuple('Spans', ['cand', 'n_cand', 'total_count', 'vec_count', 'null_feature', 'null_logits'])
Spans.__doc__ = """Per example: cand int32 [E,K,3] (feature within the example, start, end; the first n_cand rows are valid),
n_cand int32 [E], total_count / vec_count int64 [E] (valid spans before / after the filter), null_feature int32 [E] (within the
example, -1 when no feature's start[0] + end[0] is below 1e6) and null_logits fp32 [E,2]."""


def feature_masks(features, S):
    """-> (n_tokens int32 [F], start_ok uint32 [F,W], end_ok uint32 [F,W]), W = ceil(S/32), from the reference's feature objects:
    a token may end a span when it is in token_to_orig_map, and start one when token_is_max_context is also true for it."""
    F, W = len(features), (S + 31) // 32
    n_tokens = np.fromiter((len(f.tokens) for f in features), dtype=np.int32, count=F)
    e_rows, e_cols, s_rows, s_cols = [], [], [], []
    for i, f in enumerate(features):
        keys = [t for t in f.token_to_orig_map if 0 <= t < S]
        e_rows.append(np.full(len(keys), i, np.int64))
        e_cols.append(np.asarray(keys, np.int64))
        starts = [t for t in keys if f.token_is_max_context.get(t, False)]
        s_rows.append(np.full(len(starts), i, np.int64))
        s_cols.append(np.asarray(starts, np.int64))

    def pack(rows, cols):
        m = np.zeros((F, W), np.uint32)
        rows, cols = np.concatenate(rows + [np.zeros(0, np.int64)]), np.concatenate(cols + [np.zeros(0, np.int64)])
        np.bitwise_or.at(m, (rows, cols >> 5), (np.uint32(1) << (cols & 31).astype(np.uint32)))
        return m
    return n_tokens, pack(s_rows, s_cols), pack(e_rows, e_cols)


def best_spans(start, end, sft, eft, n_tokens, start_ok, end_ok, ex_off, max_answer_length, filter_threshold, k, version_2=False):
    """The binding of dph_rc_spans.  start / end / sft / eft: [F,S] fp32 logits, n_tokens [F], start_ok / end_ok [F, ceil(S/32)] bit
    masks (feature_masks), ex_off [E+1] int64 example offsets (each example's features contiguous and in order).  Torch tensors or
    numpy arrays; when every input is a CUDA tensor the decoder reads them in place, otherwise from host memory.  -> Spans (numpy)."""
    arrays = (start, end, sft, eft, n_tokens, start_ok, end_ok, ex_off)
    on_gpu = all(isinstance(x, torch.Tensor) and x.is_cuda for x in arrays)
    dtypes = (torch.float32,) * 4 + (torch.int32, torch.int32, torch.int32, torch.int64)
    if on_gpu:
        dev = start.device
        start, end, sft, eft, n_tokens, start_ok, end_ok, ex_off = ((x.view(torch.int32) if x.dtype == torch.uint32 else x).to(dev, dt).contiguous()
                                                                     for x, dt in zip(arrays, dtypes))
    else:
        np_dt = (np.float32,) * 4 + (np.int32, np.uint32, np.uint32, np.int64)
        start, end, sft, eft, n_tokens, start_ok, end_ok, ex_off = (
            np.ascontiguousarray(x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)).astype(dt, copy=False)
            for x, dt in zip(arrays, np_dt))
    if len(start.shape) != 2:
        raise ValueError(f'logits must be [F, S], got {tuple(start.shape)}')
    F, S = int(start.shape[0]), int(start.shape[1])
    W = (S + 31) // 32
    for name, x in (('end', end), ('sft', sft), ('eft', eft)):
        if tuple(x.shape) != (F, S):
            raise ValueError(f'{name} logits {tuple(x.shape)} do not match start {(F, S)}')
    if tuple(n_tokens.shape) != (F,) or tuple(start_ok.shape) != (F, W) or tuple(end_ok.shape) != (F, W):
        raise ValueError(f'n_tokens must be [{F}] and the masks [{F}, {W}]')
    if len(ex_off.shape) != 1 or ex_off.shape[0] < 2:
        raise ValueError('ex_off must be [E+1] with E >= 1')
    E, K = int(ex_off.shape[0]) - 1, int(k)
    if on_gpu:
        out = dict(cand=torch.empty((E, K, 3), dtype=torch.int32, device=dev), n_cand=torch.empty(E, dtype=torch.int32, device=dev),
                   total_count=torch.empty(E, dtype=torch.int64, device=dev), vec_count=torch.empty(E, dtype=torch.int64, device=dev),
                   null_feature=torch.empty(E, dtype=torch.int32, device=dev), null_logits=torch.empty((E, 2), dtype=torch.float32, device=dev))
        ptr = lambda x: x.data_ptr()                                          # noqa: E731
        stream, mem = torch.cuda.current_stream(dev).cuda_stream, L.MEM_DEVICE
    else:
        out = dict(cand=np.empty((E, K, 3), np.int32), n_cand=np.empty(E, np.int32), total_count=np.empty(E, np.int64),
                   vec_count=np.empty(E, np.int64), null_feature=np.empty(E, np.int32), null_logits=np.empty((E, 2), np.float32))
        ptr = lambda x: x.ctypes.data                                         # noqa: E731
        stream, mem = torch.cuda.current_stream().cuda_stream, L.MEM_HOST
    L.check(L.lib().dph_rc_spans(ptr(start), ptr(end), ptr(sft), ptr(eft), F, S, ptr(n_tokens), ptr(start_ok), ptr(end_ok), ptr(ex_off), E,
                                 int(max_answer_length), float(filter_threshold), K, int(bool(version_2)), *(ptr(out[n]) for n in Spans._fields),
                                 mem, stream))
    if on_gpu:
        out = {n: v.cpu().numpy() for n, v in out.items()}
    return Spans(**out)


def host_spans(start, end, sft, eft, n_tokens, start_ok, end_ok, max_answer_length, filter_threshold):
    """Every span of one example that is valid and passes the filter, in the order of best_spans -> int32 [n,3] (feature within the
    example, start, end).  numpy [F,S] arrays and masks as best_spans takes them.  For the rare example whose n-best list needs more
    than MAX_K candidates."""
    F, S = start.shape
    bits = lambda m: np.unpackbits(np.ascontiguousarray(m).view('<u4').view(np.uint8), axis=1, bitorder='little')[:, :S].astype(bool)   # noqa: E731
    inside = np.arange(S)[None, :] < np.asarray(n_tokens)[:, None]
    thr = float(filter_threshold)
    s_ok = bits(start_ok) & inside & ~(np.asarray(sft, np.float64) < thr)
    e_ok = bits(end_ok) & inside & ~(np.asarray(eft, np.float64) < thr)
    s, j = np.meshgrid(np.arange(S), np.arange(max(0, int(max_answer_length) - 1)), indexing='ij')
    s, e = s.ravel(), (s + j).ravel()
    s, e = s[e < S], e[e < S]                          # (start, end) in enumeration order
    rows, scores = [], []
    for f in range(F):
        ok = s_ok[f, s] & e_ok[f, e]
        rows.append(np.stack([np.full(int(ok.sum()), f), s[ok], e[ok]], 1))
        scores.append(np.asarray(start[f], np.float64)[s[ok]] + np.asarray(end[f], np.float64)[e[ok]])
    rows, scores = np.concatenate(rows), np.concatenate(scores)
    return rows[np.lexsort((np.arange(len(scores)), -scores))].astype(np.int32)   # score descending (-0.0 == 0.0), then enumeration

# ---- text side (squad_metrics.py:256-406) -------------------------------------------------------------------------------------------
def tokens_to_string(tokenizer, tokens):
    """The tokenizer's convert_tokens_to_string when it has one, else BERT's WordPiece rule."""
    f = getattr(tokenizer, 'convert_tokens_to_string', None)
    return f(tokens) if f is not None else ' '.join(tokens).replace(' ##', '').strip()


def get_final_text(pred_text, orig_text, do_lower_case, verbose_logging=False):
    """Map a normalised prediction back onto the original text: basic-tokenise orig_text, align the two texts character by
    character once spaces are removed, and cut orig_text at the aligned ends.  orig_text when the alignment fails."""
    lo, hi = final_text_span(pred_text, orig_text, do_lower_case, verbose_logging)
    return orig_text[lo:hi] if (lo, hi) != (0, len(orig_text)) else orig_text


def final_text_span(pred_text, orig_text, do_lower_case, verbose_logging=False):
    """get_final_text(..., return_pos=True): the aligned [start, end) character range in orig_text, (0, len(orig_text)) when the
    alignment fails."""
    def no_spaces(text):
        chars, where = [], {}
        for i, c in enumerate(text):
            if c != ' ':
                where[len(chars)] = i
                chars.append(c)
        return ''.join(chars), where

    tok_text = ' '.join(basic_tokenize(orig_text, do_lower_case=do_lower_case))
    first = tok_text.find(pred_text)
    fail = (0, len(orig_text))
    if first == -1:
        if verbose_logging:
            logger.info("Unable to find text: '%s' in '%s'", pred_text, orig_text)
        return fail
    last = first + len(pred_text) - 1
    orig_ns, orig_map = no_spaces(orig_text)
    tok_ns, tok_map = no_spaces(tok_text)
    if len(orig_ns) != len(tok_ns):
        if verbose_logging:
            logger.info("Length not equal after stripping spaces: '%s' vs '%s'", orig_ns, tok_ns)
        return fail
    tok_to_ns = {pos: i for i, pos in tok_map.items()}
    lo = orig_map.get(tok_to_ns[first]) if first in tok_to_ns else None
    if lo is None:
        if verbose_logging:
            logger.info("Couldn't map start position")
        return fail
    hi = orig_map.get(tok_to_ns[last]) if last in tok_to_ns else None
    if hi is None:
        if verbose_logging:
            logger.info("Couldn't map end position")
        return fail
    return lo, hi + 1


def _compute_softmax(scores):
    if not scores:
        return []
    top = max(scores)
    exps = [math.exp(s - top) for s in scores]
    total = 0.0
    for x in exps:
        total += x
    return [x / total for x in exps]


def _logit_rows(all_results, order, n_features):
    """-> four fp32 [F,S] arrays (start, end, sft, eft) with row i = the i-th feature in decoding order.  all_results: the
    reference's SquadResult iterator (consumed in decoding order) or four [F,S] tensors / arrays indexed like all_features."""
    if isinstance(all_results, (tuple, list)) and len(all_results) == 4 and all(hasattr(x, 'shape') for x in all_results):
        rows = torch.as_tensor(np.asarray(order, dtype=np.int64))
        out = []
        for x in all_results:
            x = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x))
            if x.shape[0] != n_features:
                raise ValueError(f'logits have {x.shape[0]} rows for {n_features} features')
            out.append(x.detach()[rows.to(x.device)].to(torch.float32).cpu().numpy())
        return out, None
    it = iter(all_results)
    results = [next(it) for _ in order]
    cols = [np.asarray([getattr(r, n) for r in results], dtype=np.float32) for n in ('start_logits', 'end_logits', 'sft_logits', 'eft_logits')]
    return cols, [r.unique_id for r in results]


def compute_predictions_logits(all_examples, all_features, all_results, n_best_size, max_answer_length, do_lower_case,
                               output_prediction_file, output_nbest_file, output_null_log_odds_file, verbose_logging,
                               version_2_with_negative, null_score_diff_threshold, tokenizer, filter_threshold, output_candidates_file):
    """== squad_metrics.compute_predictions_logits (same arguments, same files, same (predictions, stat) result), with the span
    enumeration on the GPU.  all_results: the reference's iterator of SquadResult, or (start, end, sft, eft) [F,S] logits indexed
    like all_features (Encoder.forward's outputs, concatenated).  Output file names may be None (no file)."""
    by_example = collections.defaultdict(list)
    for i, f in enumerate(all_features):
        by_example[f.example_index].append(i)
    groups = [by_example[x] for x in range(len(all_examples))]
    if any(not g for g in groups):
        raise ZeroDivisionError('float division by zero')          # the reference's per-example save_rate with no valid span
    order = [i for g in groups for i in g]
    feats = [all_features[i] for i in order]
    (st, en, sft, eft), uids = _logit_rows(all_results, order, len(all_features))
    if uids is not None:
        for u, f in zip(uids, feats):
            assert u == f.unique_id
    S = st.shape[1]
    n_tokens, start_ok, end_ok = feature_masks(feats, S)
    ex_off = np.zeros(len(groups) + 1, np.int64)
    ex_off[1:] = np.cumsum([len(g) for g in groups])
    k0 = min(MAX_K, max(1, int(n_best_size)))
    sp = best_spans(st, en, sft, eft, n_tokens, start_ok, end_ok, ex_off, max_answer_length, filter_threshold, k0, version_2_with_negative)
    if (sp.total_count == 0).any():
        raise ZeroDivisionError('float division by zero')

    Nbest = collections.namedtuple('NbestPrediction', ['text', 'start_logit', 'end_logit'])
    all_predictions, all_nbest_json, scores_diff_json, id2candidates = (collections.OrderedDict(), collections.OrderedDict(),
                                                                        collections.OrderedDict(), {})

    def span_text(example, feature, s, e):
        tok_text = ' '.join(tokens_to_string(tokenizer, feature.tokens[s:e + 1]).strip().split())
        orig_text = ' '.join(example.doc_tokens[feature.token_to_orig_map[s]:feature.token_to_orig_map[e] + 1])
        return get_final_text(tok_text, orig_text, do_lower_case, verbose_logging)

    def nbest_of(x, example, cand, n_cand, null):
        """The reference's n-best loop over the merged prelim list, or None when it needs candidates beyond the first n_cand."""
        f0 = ex_off[x]
        prelim = [(int(fi), int(s), int(e), float(st[f0 + fi, s]), float(en[f0 + fi, e]), False) for fi, s, e in cand[:n_cand]]
        if null is not None:
            prelim.append(null)
        prelim.sort(key=lambda p: p[3] + p[4], reverse=True)
        more = int(sp.vec_count[x]) > n_cand
        seen, nbest, used = {}, [], 0
        for fi, s, e, sl, el, is_null in prelim:
            if len(nbest) >= n_best_size:
                return nbest, seen
            if used == n_cand and more:
                return None
            used += not is_null
            if s > 0:
                text = span_text(example, feats[f0 + fi], s, e)
                if text in seen:
                    continue
            else:
                text = ''
            seen[text] = True
            nbest.append(Nbest(text, sl, el))
        if len(nbest) < n_best_size and more:
            return None
        return nbest, seen

    for x, example in enumerate(all_examples):
        features = [feats[i] for i in range(ex_off[x], ex_off[x + 1])]
        null, score_null = None, 1000000
        if version_2_with_negative:
            nf = int(sp.null_feature[x])
            if nf >= 0:
                ns, ne = float(sp.null_logits[x, 0]), float(sp.null_logits[x, 1])
                null, score_null = (nf, 0, 0, ns, ne, True), ns + ne
            else:
                null = (0, 0, 0, 0, 0, True)
        id2candidates[example.qas_id] = {'candidates': [], 'text': example.context_text, 'answer': example.answers, 'recall': False}
        id2candidates[features[-1].qas_id]['save_rate'] = float(0 / int(sp.total_count[x]))
        cand, n_cand, k = sp.cand[x], int(sp.n_cand[x]), k0
        got = nbest_of(x, example, cand, n_cand, null)
        while got is None:
            a, b = ex_off[x], ex_off[x + 1]
            if k < MAX_K:
                k = min(MAX_K, 2 * k)
                one = best_spans(st[a:b], en[a:b], sft[a:b], eft[a:b], n_tokens[a:b], start_ok[a:b], end_ok[a:b], np.array([0, b - a], np.int64),
                                 max_answer_length, filter_threshold, k, version_2_with_negative)
                cand, n_cand = one.cand[0], int(one.n_cand[0])
            else:          # past the decoder's K bound (repeated tokens): the whole ordered list, enumerated on the host
                cand = host_spans(st[a:b], en[a:b], sft[a:b], eft[a:b], n_tokens[a:b], start_ok[a:b], end_ok[a:b], max_answer_length,
                                  filter_threshold)
                n_cand = len(cand)
                if n_cand != int(sp.vec_count[x]):
                    raise RuntimeError(f'example {x}: {n_cand} spans enumerated on the host, the decoder counted {int(sp.vec_count[x])}')
            got = nbest_of(x, example, cand, n_cand, null)
        nbest, seen = got
        if version_2_with_negative:
            if '' not in seen:
                nbest.append(Nbest('', null[3], null[4]))
            if len(nbest) == 1:
                nbest.insert(0, Nbest('empty', 0.0, 0.0))
        if not nbest:
            nbest.append(Nbest('empty', 0.0, 0.0))
        total_scores = [p.start_logit + p.end_logit for p in nbest]
        best_non_null = next((p for p in nbest if p.text), None)
        probs = _compute_softmax(total_scores)
        nbest_json = [collections.OrderedDict([('text', p.text), ('probability', probs[i]), ('start_logit', p.start_logit),
                                               ('end_logit', p.end_logit)]) for i, p in enumerate(nbest)]
        if not version_2_with_negative:
            all_predictions[example.qas_id] = nbest_json[0]['text']
        else:
            diff = score_null - best_non_null.start_logit - best_non_null.end_logit
            scores_diff_json[example.qas_id] = diff
            all_predictions[example.qas_id] = '' if diff > null_score_diff_threshold else best_non_null.text
        all_nbest_json[example.qas_id] = nbest_json

    vec_count, total_count = int(sp.vec_count.sum()), int(sp.total_count.sum())
    logger.info('saved vecs=%d/%d, save rate=%.4f', vec_count, total_count, vec_count / total_count)
    stat = {'save_rate': vec_count / total_count}
    for path, obj, on in ((output_prediction_file, all_predictions, True), (output_nbest_file, all_nbest_json, True),
                          (output_null_log_odds_file, scores_diff_json, version_2_with_negative),
                          (output_candidates_file, id2candidates, True)):
        if path and on:
            with open(path, 'w') as w:
                w.write(json.dumps(obj, indent=4) + '\n')
    return all_predictions, stat


# ---- squad_evaluate (squad_metrics.py:34-254, the arguments train_rc.py passes) ----------------------------------------------------
def normalize_answer(s):
    """Lower case, drop punctuation and the articles a / an / the, collapse whitespace (the SQuAD rule)."""
    s = ''.join(ch for ch in s.lower() if ch not in set(string.punctuation))
    s = re.sub(r'\b(a|an|the)\b', ' ', s, flags=re.UNICODE)
    return ' '.join(s.split())


def compute_exact(a_gold, a_pred):
    return int(normalize_answer(a_gold) == normalize_answer(a_pred))


def compute_f1(a_gold, a_pred):
    gold = normalize_answer(a_gold).split() if a_gold else []
    pred = normalize_answer(a_pred).split() if a_pred else []
    if not gold or not pred:
        return int(gold == pred)
    same = sum((collections.Counter(gold) & collections.Counter(pred)).values())
    if same == 0:
        return 0
    p, r = 1.0 * same / len(pred), 1.0 * same / len(gold)
    return (2 * p * r) / (p + r)


def _eval_dict(exact, f1, qids=None):
    qids = list(exact) if not qids else qids
    n = len(qids)
    return collections.OrderedDict([('exact', 100.0 * sum(exact[q] for q in qids) / n), ('f1', 100.0 * sum(f1[q] for q in qids) / n),
                                    ('total', n)])


def _best_thresh(preds, scores, na_probs, has_ans):
    cur = best = sum(1 for q in has_ans if not has_ans[q])
    thresh = 0.0
    for q in sorted(na_probs, key=lambda k: na_probs[k]):
        if q not in scores:
            continue
        cur += scores[q] if has_ans[q] else (-1 if preds[q] else 0)
        if cur > best:
            best, thresh = cur, na_probs[q]
    return 100.0 * best / len(scores), thresh


def squad_evaluate(examples, preds, no_answer_probs=None, no_answer_probability_threshold=1.0, null_log_odds_file=None):
    """== squad_metrics.squad_evaluate: exact / f1 / total, HasAns_* / NoAns_*, best_exact(_thresh) / best_f1(_thresh)."""
    has_ans = {ex.qas_id: bool(ex.answers) for ex in examples}
    if no_answer_probs is None:
        if null_log_odds_file is not None:
            with open(null_log_odds_file) as f:
                no_answer_probs = json.load(f)
        else:
            no_answer_probs = {k: 0.0 for k in preds}
    exact, f1 = {}, {}
    for ex in examples:
        golds = [a['text'] for a in ex.answers if normalize_answer(a['text'])] or ['']
        if ex.qas_id not in preds:
            print('Missing prediction for %s' % ex.qas_id)
            continue
        p = preds[ex.qas_id]
        exact[ex.qas_id] = max(compute_exact(a, p) for a in golds)
        f1[ex.qas_id] = max(compute_f1(a, p) for a in golds)

    def thresholded(scores):
        return {q: float(not has_ans[q]) if no_answer_probs[q] > no_answer_probability_threshold else s for q, s in scores.items()}
    exact_t, f1_t = thresholded(exact), thresholded(f1)
    evaluation = _eval_dict(exact_t, f1_t)
    for prefix, want in (('HasAns', True), ('NoAns', False)):
        qids = [q for q, h in has_ans.items() if h == want]
        if qids:
            for k, v in _eval_dict(exact_t, f1_t, qids).items():
                evaluation[f'{prefix}_{k}'] = v
    if no_answer_probs:
        evaluation['best_exact'], evaluation['best_exact_thresh'] = _best_thresh(preds, exact, no_answer_probs, has_ans)
        evaluation['best_f1'], evaluation['best_f1_thresh'] = _best_thresh(preds, f1, no_answer_probs, has_ans)
    return evaluation


# ---- the filter test (train_rc.py:410-431) -----------------------------------------------------------------------------------------
FILTER_TEST_THRESHOLDS = (-4.0, -3.0, -2.0, -1.0, -0.5, 0.0, 1.0)       # make filter-test's --filter_threshold_list


def read_features(encoder, features, batch_size=64):
    """One Encoder.forward over the features' context and question ids, in batches -> (start, end, sft, eft) fp32 [F,S] on the GPU."""
    outs = []
    for i in range(0, len(features), batch_size):
        fb = features[i:i + batch_size]
        t = [torch.from_numpy(np.asarray([getattr(f, n) for f in fb], dtype=np.int64))
             for n in ('input_ids', 'attention_mask', 'token_type_ids', 'input_ids_', 'attention_mask_', 'token_type_ids_')]
        outs.append(encoder(input_ids=t[0], attention_mask=t[1], token_type_ids=t[2], input_ids_=t[3], attention_mask_=t[4], token_type_ids_=t[5]))
    return tuple(torch.cat([o[j] for o in outs]) for j in range(4))


def filter_test(encoder, examples, features, tokenizer, thresholds=FILTER_TEST_THRESHOLDS, n_best_size=20, max_answer_length=10,
                do_lower_case=False, version_2_with_negative=False, null_score_diff_threshold=0.0, batch_size=64, logits=None):
    """train_rc.py --do_filter_test with one forward: the logits once (or `logits`, four [F,S] tensors indexed like `features`),
    then one decode and one squad_evaluate per threshold -> {'exact_T', 'f1_T', 'save_rate_T'} per threshold T (formatted '%.2f')."""
    if logits is None:
        logits = read_features(encoder, features, batch_size)
    results = {}
    for thr in thresholds:
        preds, stat = compute_predictions_logits(examples, features, logits, n_best_size, max_answer_length, do_lower_case, None, None, None,
                                                 False, version_2_with_negative, null_score_diff_threshold, tokenizer, thr, None)
        ev = squad_evaluate(examples, preds)
        results[f'exact_{thr:.2f}'] = ev['exact']
        results[f'f1_{thr:.2f}'] = ev['f1']
        results[f'save_rate_{thr:.2f}'] = stat['save_rate']
    return results
