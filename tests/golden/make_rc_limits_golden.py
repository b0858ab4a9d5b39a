"""Golden outputs of the UNMODIFIED reference compute_predictions_logits (densephrases/utils/squad_metrics.py
:408-684) where the n-best list needs more than 1024 prelim candidates -> tests/golden/rc_limits.json.gz.

The reference module is loaded as tests/golden/make_rc_golden.py loads it, with the same stand-ins; every line of the function is
the reference's code.  The cases:
- one feature of 200 copies of one word, in version 1 and 2: 1 764 valid spans, 9 distinct texts, so n_best_size = 20 is never
  reached and the whole prelim list is read;
- one example of three overlapping windows over two alternating words (18 distinct texts, over 1 024 spans), next to an ordinary
  example;
- a document of one repeated word and one other word, spans of one token (max_answer_length = 2) and n_best_size = 2: the other
  word is the 1 024th prelim candidate in one case and the 1 025th in the next.
Each case is checked here to reach what it claims.  Same file format as rc_reference.json.gz.

    python tests/golden/make_rc_limits_golden.py"""
import gzip
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_rc_golden import Example, Feature, JoinTokenizer, ex_json, feat_json, reference_metrics   # noqa: E402


def windows(x, words, starts, win, max_context):
    """Features of example x over `words`: one window of `win` words at each start; token_is_max_context from max_context(f, j)."""
    feats = []
    for f, lo in enumerate(starts):
        span = list(range(lo, min(len(words), lo + win)))
        tokens = ['[CLS]'] + [words[i] for i in span] + ['[SEP]']
        feats.append(Feature(x, 1000 * (x + 1) + f, f'q{x}', tokens, {1 + j: i for j, i in enumerate(span)},
                             {1 + j: bool(max_context(f, j)) for j in range(len(span))}))
    return feats


def grid(rng, F, S):
    return [(np.round(rng.normal(size=(F, S)) * 3.0) / 2.0).astype(np.float32) for _ in range(4)]


def prelim_order(features, logits, L):
    """The reference's prelim list (valid spans, no filter) in its sorted order -> [(feature, start, end)]."""
    st, en = logits[0], logits[1]
    spans = []
    for fi, f in enumerate(features):
        for s in range(len(f.tokens)):
            for e in range(s, min(len(f.tokens), s + L - 1)):
                if s in f.token_to_orig_map and e in f.token_to_orig_map and f.token_is_max_context.get(s, False):
                    spans.append((fi, s, e, float(st[fi, s]) + float(en[fi, e])))
    return [p[:3] for p in sorted(spans, key=lambda p: p[3], reverse=True)]


def repeat_word(v2):
    rng = np.random.default_rng(21 + v2)
    words = ['w'] * 200
    feats = windows(0, words, [0], 200, lambda f, j: True)
    logits = grid(rng, 1, 256)
    assert len(prelim_order(feats, logits, 10)) == 1764
    return dict(name=f'repeat_word_200{"_v2" if v2 else ""}', S=256, n_best_size=20, max_answer_length=10, version_2=v2,
                examples=[Example('q0', words, [{'text': 'w w', 'answer_start': 0}])], features=feats, logits=logits, thrs=[-1e8, -1.0])


def overlap():
    rng = np.random.default_rng(23)
    words = ['x' if i % 2 == 0 else 'y' for i in range(150)]
    other = ['Paris', 'river', 'Seine', 'flows', 'through', 'the', 'city']
    feats = windows(0, words, [0, 35, 70], 80, lambda f, j: f == 0 or j > 20) + windows(1, other, [0], 7, lambda f, j: True)
    logits = grid(rng, len(feats), 96)
    n = len(prelim_order(feats[:3], [x[:3] for x in logits], 10))
    assert n > 1024, n
    return dict(name='overlap_windows', S=96, n_best_size=20, max_answer_length=10, version_2=False,
                examples=[Example('q0', words, []), Example('q1', other, [{'text': 'Seine', 'answer_start': 0}])], features=feats,
                logits=logits, thrs=[-1e8])


def nth_candidate(need):
    """n_best_size = 2 over one-token spans of 'w' and a single 'z': 'z' placed at prelim rank `need` (1-based)."""
    rng = np.random.default_rng(25)
    words = ['w'] * 1050
    feats = windows(0, words, [0, 350, 700], 350, lambda f, j: True)
    logits = grid(rng, 3, 352)
    fi, s, _ = prelim_order(feats, logits, 2)[need - 1]
    words[feats[fi].token_to_orig_map[s]] = 'z'
    feats[fi].tokens[s] = 'z'
    return dict(name=f'z_at_candidate_{need}', S=352, n_best_size=2, max_answer_length=2, version_2=False,
                examples=[Example('q0', words, [{'text': 'z', 'answer_start': 0}])], features=feats, logits=logits, thrs=[-1e8])


def main():
    sm, SquadResult = reference_metrics()
    tok = JoinTokenizer()
    out = {'configs': []}
    with tempfile.TemporaryDirectory() as tmp:
        for c in (repeat_word(False), repeat_word(True), overlap(), nth_candidate(1024), nth_candidate(1025)):
            examples, features, logits = c['examples'], c['features'], c['logits']
            case = {'name': c['name'], 'S': c['S'], 'n_best_size': c['n_best_size'], 'max_answer_length': c['max_answer_length'],
                    'do_lower_case': False, 'version_2': c['version_2'], 'null_score_diff_threshold': 0.0,
                    'examples': [ex_json(e) for e in examples], 'features': [feat_json(f) for f in features],
                    'logits': [x.tolist() for x in logits], 'runs': []}
            for thr in c['thrs']:
                results = iter([SquadResult(f.unique_id, *(x[i].tolist() for x in logits)) for i, f in enumerate(features)])
                files = {k: os.path.join(tmp, f'{k}.json') for k in ('pred', 'nbest', 'null', 'cand')}
                for p in files.values():
                    if os.path.exists(p):
                        os.remove(p)
                v2 = c['version_2']
                preds, stat = sm.compute_predictions_logits(examples, features, results, c['n_best_size'], c['max_answer_length'], False,
                                                            files['pred'], files['nbest'], files['null'] if v2 else None, False, v2, 0.0,
                                                            tok, thr, files['cand'])
                files = {k: open(p).read() for k, p in files.items() if os.path.exists(p)}
                case['runs'].append({'filter_threshold': thr, 'predictions': preds, 'stat': stat, 'files': files})
            print(c['name'], [(r['filter_threshold'], r['predictions'], r['stat']) for r in case['runs']])
            out['configs'].append(case)
    path = os.path.join(ROOT, 'tests', 'golden', 'rc_limits.json.gz')
    with open(path, 'wb') as f, gzip.GzipFile(fileobj=f, mode='wb', mtime=0) as z:
        z.write(json.dumps(out, separators=(',', ':')).encode())
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
