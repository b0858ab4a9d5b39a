"""Golden outputs of the UNMODIFIED reference reading path:
(1) /root/reference/densephrases/utils/squad_metrics.py `compute_predictions_logits` (:408-684) and `squad_evaluate` (:221-254) on
    synthetic examples, features and results -> tests/golden/rc_reference.json.gz;
(2) /root/reference/densephrases/encoder.py `Encoder.forward` with a context and a question (neither return_phrase nor
    return_query) on seeded random weights and small ragged batches -> tests/golden/encoder_rc.npz.

The reference modules are loaded by file path.  squad_metrics' unavailable imports get stand-ins: h5py (never called here),
transformers.tokenization_bert.BasicTokenizer (-> the installed transformers' BERT BasicTokenizer) and its sibling squad_utils
(-> the two result classes it takes).  The tokenizer argument is a stand-in with BERT's convert_tokens_to_string.  Every line of
the two functions is the reference's code.

The synthetic data covers: examples with 1-4 features (overlapping windows, token_is_max_context False in the overlap), gaps in
token_to_orig_map ([CLS], [SEP], question-free padding), word pieces, logits on a coarse grid (many exact ties of start + end),
spans that reach n_tokens, thresholds that keep every span and that remove every span of an example, version 2 with
null_score_diff_threshold, lower-cased and cased text, documents of one repeated word (duplicate texts: the n-best list cannot
fill from the first K candidates), and an example without any valid span (ZeroDivisionError in the reference).

    python tests/golden/make_rc_golden.py"""
import gzip
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = '/root/reference/densephrases'

WORDS = ['Paris', 'river', 'Seine', 'flows', 'through', 'the', 'city', "France's", 'capital', 'since', '1850,', 'bridges', 'cross',
         'it', 'many', 'times', 'and', 'boats', 'carry', 'tourists', 'unbelievably', 'slowly', '(north)', 'St.', 'Louis']


class Example(object):
    def __init__(self, qas_id, doc_tokens, answers):
        self.qas_id, self.doc_tokens, self.answers = qas_id, doc_tokens, answers
        self.context_text = ' '.join(doc_tokens)


class Feature(object):
    def __init__(self, example_index, unique_id, qas_id, tokens, token_to_orig_map, token_is_max_context):
        self.example_index, self.unique_id, self.qas_id = example_index, unique_id, qas_id
        self.tokens, self.token_to_orig_map, self.token_is_max_context = tokens, token_to_orig_map, token_is_max_context


class JoinTokenizer(object):
    """BERT's convert_tokens_to_string (transformers BertTokenizer)."""
    def convert_tokens_to_string(self, tokens):
        return ' '.join(tokens).replace(' ##', '').strip()


def pieces(word):
    """A deterministic WordPiece-like split: words longer than 6 characters become two pieces."""
    return [word] if len(word) <= 6 else [word[:4], '##' + word[4:]]


def make_data(rng, n_examples, S, repeat_word=False, lower=False, no_span_example=False):
    examples, features = [], []
    for x in range(n_examples):
        n_words = int(rng.integers(6, 40))
        words = ['alpha'] * n_words if repeat_word else [WORDS[i] for i in rng.integers(0, len(WORDS), n_words)]
        if lower:
            words = [w.lower() if rng.random() < 0.5 else w for w in words]
        qid = f'q{x}'
        if rng.random() < 0.3:
            answers = []
        else:
            a = int(rng.integers(0, n_words - 2))
            answers = [{'text': ' '.join(words[a:a + int(rng.integers(1, 3))]), 'answer_start': 0}]
        examples.append(Example(qid, words, answers))
        toks, tok_word = [], []
        for w, word in enumerate(words):
            for p in pieces(word):
                toks.append(p)
                tok_word.append(w)
        n_feat = int(rng.integers(1, 5))
        win = max(4, min(S - 2, -(-len(toks) // n_feat) + 3))
        stride = max(1, (len(toks) - win) // max(1, n_feat - 1)) if n_feat > 1 else win
        for f in range(n_feat):
            lo = min(f * stride, max(0, len(toks) - win))
            span = list(range(lo, min(len(toks), lo + win)))
            tokens = ['[CLS]'] + [toks[i] for i in span] + ['[SEP]']
            t2o = {1 + j: tok_word[i] for j, i in enumerate(span)}
            if rng.random() < 0.3 and len(t2o) > 3:              # a gap inside the context
                del t2o[sorted(t2o)[len(t2o) // 2]]
            mid = lambda j: f == 0 or j > len(span) // 3            # noqa: E731  earlier windows hold the max context of the overlap
            tmc = {1 + j: bool(mid(j)) for j in range(len(span))}
            if no_span_example and x == n_examples - 1:
                t2o = {}
            features.append(Feature(x, 1000 + len(features), qid, tokens, t2o, tmc))
    F = len(features)
    grid = lambda: (np.round(rng.normal(size=(F, S)) * 3.0) / 2.0).astype(np.float32)   # noqa: E731  coarse grid: exact ties
    return examples, features, [grid(), grid(), grid(), grid()]


def ex_json(e):
    return {'qas_id': e.qas_id, 'doc_tokens': e.doc_tokens, 'answers': e.answers}


def feat_json(f):
    return {'example_index': f.example_index, 'unique_id': f.unique_id, 'qas_id': f.qas_id, 'tokens': f.tokens,
            'token_to_orig_map': sorted(f.token_to_orig_map.items()), 'token_is_max_context': sorted(f.token_is_max_context.items())}


def load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_metrics():
    from transformers.models.bert.tokenization_bert_legacy import BasicTokenizer
    sys.modules['h5py'] = types.ModuleType('h5py')
    tb = types.ModuleType('transformers.tokenization_bert')
    tb.BasicTokenizer = BasicTokenizer
    sys.modules['transformers.tokenization_bert'] = tb
    for pkg in ('densephrases', 'densephrases.utils'):
        m = types.ModuleType(pkg)
        m.__path__ = []
        sys.modules[pkg] = m
    su = types.ModuleType('densephrases.utils.squad_utils')

    class SquadResult(object):
        def __init__(self, unique_id, start_logits, end_logits, sft_logits, eft_logits):
            self.start_logits, self.end_logits, self.sft_logits, self.eft_logits, self.unique_id = (start_logits, end_logits, sft_logits,
                                                                                                   eft_logits, unique_id)
    su.SquadResult, su.QuestionResult = SquadResult, object
    sys.modules['densephrases.utils.squad_utils'] = su
    return load('densephrases.utils.squad_metrics', os.path.join(REF, 'utils', 'squad_metrics.py')), SquadResult


CONFIGS = [  # name, data seed, examples, S, repeat_word, lower, no-span example, n_best, L, thresholds, version 2, null threshold
    ('squad_v1', 1, 6, 48, False, False, False, 5, 10, [-1e8, 0.0, 10.0], False, 0.0),
    ('squad_v1_lower_L4', 2, 5, 40, False, True, False, 5, 4, [0.0], False, 0.0),
    ('squad_v2', 3, 6, 48, False, False, False, 5, 10, [-1e8, 0.0], True, 0.0),
    ('squad_v2_null_thr', 4, 5, 64, False, False, False, 5, 12, [-1.0], True, 1.5),
    ('repeat_word', 5, 2, 48, True, False, False, 20, 10, [-1e8], False, 0.0),
    ('repeat_word_v2', 6, 2, 40, True, False, False, 20, 10, [-1e8], True, 0.0),
    ('no_valid_span', 7, 3, 32, False, False, True, 20, 10, [-1e8], False, 0.0),
]


def rc_golden():
    sm, SquadResult = reference_metrics()
    out = {'configs': []}
    tok = JoinTokenizer()
    with tempfile.TemporaryDirectory() as tmp:
        for name, seed, n_ex, S, rep, lower, nospan, n_best, L, thrs, v2, null_thr in CONFIGS:
            rng = np.random.default_rng(seed)
            examples, features, logits = make_data(rng, n_ex, S, rep, lower, nospan)
            case = {'name': name, 'S': S, 'n_best_size': n_best, 'max_answer_length': L, 'do_lower_case': lower, 'version_2': v2,
                    'null_score_diff_threshold': null_thr, 'examples': [ex_json(e) for e in examples], 'features': [feat_json(f) for f in features],
                    'logits': [x.tolist() for x in logits], 'runs': []}
            for thr in thrs:
                results = iter([SquadResult(f.unique_id, *(x[i].tolist() for x in logits)) for i, f in enumerate(features)])
                files = {k: os.path.join(tmp, f'{k}.json') for k in ('pred', 'nbest', 'null', 'cand')}
                for p in files.values():
                    if os.path.exists(p):
                        os.remove(p)
                run = {'filter_threshold': thr}
                try:
                    preds, stat = sm.compute_predictions_logits(examples, features, results, n_best, L, lower, files['pred'], files['nbest'],
                                                                files['null'] if v2 else None, False, v2, null_thr, tok, thr, files['cand'])
                except ZeroDivisionError:
                    run['error'] = 'ZeroDivisionError'
                    case['runs'].append(run)
                    continue
                run['predictions'], run['stat'] = preds, stat
                run['files'] = {k: open(p).read() for k, p in files.items() if os.path.exists(p)}
                run['eval'] = sm.squad_evaluate(examples, preds, null_log_odds_file=files['null'] if v2 else None)
                case['runs'].append(run)
            print(name, [(r['filter_threshold'], r.get('stat', r.get('error'))) for r in case['runs']])
            out['configs'].append(case)
    path = os.path.join(ROOT, 'tests', 'golden', 'rc_reference.json.gz')
    with open(path, 'wb') as f, gzip.GzipFile(fileobj=f, mode='wb', mtime=0) as z:
        z.write(json.dumps(out, separators=(',', ':')).encode())
    print('wrote', path, os.path.getsize(path), 'bytes')


ENC_CASES = {'b3_s48_q16': (3, 48, 16), 'b2_s160_q32': (2, 160, 32)}


def encoder_golden():
    from transformers import BertConfig, BertModel
    from densephrases_b200.encoder import BertGeometry, random_phrase_state_dict, random_state_dict, synthetic_context_batch, synthetic_query_batch
    from tests import rc_ref_torch
    from tests.golden.make_encoder_golden import load_reference_encoder
    torch.manual_seed(0)
    seed, vocab = 20241101, 28996
    geo = BertGeometry(vocab_size=vocab)
    cfg = BertConfig(vocab_size=vocab, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                     max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12, hidden_act='gelu',
                     hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    model = load_reference_encoder()(cfg, tokenizer=None, transformer_cls=BertModel).eval()
    sd = rc_ref_torch.rc_state_dict(geo, seed)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all(not m.startswith(('phrase_encoder.encoder', 'query_start_encoder.encoder', 'query_end_encoder.encoder', 'filter_linear')) for m in missing), missing
    out = {'seed': np.array(seed), 'vocab': np.array(vocab)}
    for name, (B, S, Sq) in ENC_CASES.items():
        ids, mask, tt = synthetic_context_batch(B, S, vocab, seed + S, type_split=True)
        qids, qmask, qtt = synthetic_query_batch(B, Sq, vocab, seed + Sq)
        with torch.no_grad():
            got = model(input_ids=ids, attention_mask=mask, token_type_ids=tt, input_ids_=qids, attention_mask_=qmask, token_type_ids_=qtt)
        assert len(got) == 4 and all(x.shape == (B, S) for x in got)
        mine = rc_ref_torch.read(sd, ids, mask, tt, qids, qmask, qtt)
        d = max((a - b).abs().max().item() for a, b in zip(got, mine))
        print(name, 'reference class vs torch restatement: max abs diff', d, '| logit scale', got[0].abs().max().item())
        assert d < 1e-3 * max(1.0, got[0].abs().max().item()), d
        for k, v in (('ids', ids), ('mask', mask), ('tt', tt), ('qids', qids), ('qmask', qmask), ('qtt', qtt)):
            out[f'{name}_{k}'] = v.numpy()
        for k, v in zip(('start', 'end', 'filter_start', 'filter_end'), got):
            out[f'{name}_{k}'] = v.numpy()
    path = os.path.join(ROOT, 'tests', 'golden', 'encoder_rc.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    rc_golden()
    encoder_golden()
