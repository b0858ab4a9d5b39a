"""TEST INFRASTRUCTURE.  The reference reading cases of tests/golden/rc_reference.json.gz (made by tests/golden/make_rc_golden.py from
the unmodified reference compute_predictions_logits / squad_evaluate) as example / feature objects and logits, and one run of
densephrases_b200.rc.compute_predictions_logits on a case that returns the files it wrote."""
import gzip
import json
import os
import types

import numpy as np

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'rc_reference.json.gz')


class JoinTokenizer(object):
    def convert_tokens_to_string(self, tokens):
        return ' '.join(tokens).replace(' ##', '').strip()


def load_cases():
    with gzip.open(GOLD, 'rt') as f:
        return json.load(f)['configs']


def objects(case):
    examples = [types.SimpleNamespace(qas_id=e['qas_id'], doc_tokens=e['doc_tokens'], answers=e['answers'], context_text=' '.join(e['doc_tokens']))
                for e in case['examples']]
    features = [types.SimpleNamespace(example_index=f['example_index'], unique_id=f['unique_id'], qas_id=f['qas_id'], tokens=f['tokens'],
                                      token_to_orig_map={int(k): v for k, v in f['token_to_orig_map']},
                                      token_is_max_context={int(k): v for k, v in f['token_is_max_context']}) for f in case['features']]
    logits = [np.asarray(x, dtype=np.float32) for x in case['logits']]
    return examples, features, logits


def run(rc, case, thr, tmp, all_results):
    """compute_predictions_logits with the case's settings -> (predictions, stat, {file key: text})."""
    examples, features, _ = objects(case)
    v2 = case['version_2']
    files = {k: os.path.join(tmp, f'{k}_{thr}.json') for k in ('pred', 'nbest', 'null', 'cand')}
    preds, stat = rc.compute_predictions_logits(examples, features, all_results, case['n_best_size'], case['max_answer_length'],
                                                case['do_lower_case'], files['pred'], files['nbest'], files['null'] if v2 else None, False, v2,
                                                case['null_score_diff_threshold'], JoinTokenizer(), thr, files['cand'])
    return preds, stat, {k: open(p).read() for k, p in files.items() if os.path.exists(p)}
