"""Golden outputs of the UNMODIFIED reference dump path (generate_phrase_vecs.py --do_dump):
/root/reference/densephrases/utils/squad_utils.py `_create_examples(context_only=True)` (:811-865) and
`squad_convert_examples_to_features(context_only=True)` (:441-560, 96-433), then embed_utils.py `write_phrases` (:201-301, with
get_metadata, filter_metadata and compress_metadata) and `write_filter` (:304-382) -> tests/golden/dump_reference.json.gz.

The reference modules are loaded by file path.  Stand-ins, as in make_rc_golden.py: h5py is a dict recorder of the groups,
datasets and attributes write_phrases creates; transformers.tokenization_bert.BasicTokenizer is the installed transformers' BERT
BasicTokenizer; squad_utils' file_utils / data_utils imports and its TrueCaser (unused for contexts) are minimal stand-ins; the
tokenizer wraps this repo's WordPiece vocabulary and implements transformers 2.9's encode_plus (prepare_for_model and
truncate_sequences with overflowing tokens).  Every line of the reference functions is the reference's code.

Inputs (tests/dump_cases.py): synthetic documents and, per case, fp32 phrase vectors and filter logits drawn from a seed, which
the tests draw again.  The int8 vectors are stored as SHA-256 digests to keep the fixture small.

    python tests/golden/make_dump_golden.py"""
import argparse
import gzip
import hashlib
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = '/root/reference/densephrases'

from tests import dump_cases  # noqa: E402

RECORD = {}


class _Group(dict):
    def __init__(self):
        super().__init__()
        self.attrs = {}

    def create_dataset(self, name, data):
        self[name] = np.asarray(data)


class _File(object):
    def __init__(self, path, mode='r'):
        self.g = RECORD.setdefault(path, {})

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def __contains__(self, k):
        return k in self.g

    def __delitem__(self, k):
        del self.g[k]

    def create_group(self, k):
        self.g[k] = _Group()
        return self.g[k]


class Tokenizer29(object):
    """transformers 2.9 BertTokenizer surface over the repo's vocabulary."""
    padding_side = 'right'
    max_len, max_len_single_sentence, max_len_sentences_pair = 512, 510, 509

    def __init__(self, wp):
        self.wp = wp
        self.cls_token_id, self.sep_token_id, self.pad_token_id = wp.cls_token_id, wp.sep_token_id, wp.pad_token_id

    def tokenize(self, text):
        return self.wp.tokenize(text)

    def convert_tokens_to_ids(self, tokens):
        return [self.wp.vocab.get(t, self.wp.unk_token_id) for t in tokens]

    def convert_ids_to_tokens(self, ids):
        return [self.wp.ids_to_tokens[i] for i in ids]

    def convert_tokens_to_string(self, tokens):
        return ' '.join(tokens).replace(' ##', '').strip()

    def truncate_sequences(self, ids, pair_ids=None, num_tokens_to_remove=0, truncation_strategy='longest_first', stride=0):
        if num_tokens_to_remove <= 0:
            return ids, pair_ids, []
        if truncation_strategy == 'only_first':
            assert len(ids) > num_tokens_to_remove
            window_len = min(len(ids), stride + num_tokens_to_remove)
            overflowing_tokens = ids[-window_len:]
            ids = ids[:-num_tokens_to_remove]
        elif truncation_strategy == 'only_second':
            assert pair_ids is not None and len(pair_ids) > num_tokens_to_remove
            window_len = min(len(pair_ids), stride + num_tokens_to_remove)
            overflowing_tokens = pair_ids[-window_len:]
            pair_ids = pair_ids[:-num_tokens_to_remove]
        else:
            raise NotImplementedError(truncation_strategy)
        return ids, pair_ids, overflowing_tokens

    def encode_plus(self, text, text_pair=None, max_length=None, stride=0, truncation_strategy='longest_first', pad_to_max_length=False,
                    return_token_type_ids=True, return_overflowing_tokens=False, **_):
        get = lambda t: self.convert_tokens_to_ids(t) if t and isinstance(t[0], str) else list(t)      # noqa: E731
        ids = get(text)
        pair_ids = get(text_pair) if text_pair is not None else None
        pair = pair_ids is not None
        total_len = len(ids) + (len(pair_ids) if pair else 0) + (3 if pair else 2)
        enc = {}
        if max_length and total_len > max_length:
            ids, pair_ids, overflowing = self.truncate_sequences(ids, pair_ids, total_len - max_length, truncation_strategy, stride)
            if return_overflowing_tokens:
                enc['overflowing_tokens'] = overflowing
                enc['num_truncated_tokens'] = total_len - max_length
        seq = [self.cls_token_id] + ids + [self.sep_token_id] + (pair_ids + [self.sep_token_id] if pair else [])
        tt = [0] * (len(ids) + 2) + ([1] * (len(pair_ids) + 1) if pair else [])
        enc['input_ids'], enc['token_type_ids'] = seq, tt
        if pad_to_max_length and max_length and len(seq) < max_length:
            d = max_length - len(seq)
            enc['attention_mask'] = [1] * len(seq) + [0] * d
            enc['token_type_ids'] = tt + [0] * d
            enc['input_ids'] = seq + [self.pad_token_id] * d
        else:
            enc['attention_mask'] = [1] * len(seq)
        return enc


def load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_modules():
    from transformers.models.bert.tokenization_bert_legacy import BasicTokenizer
    h5 = types.ModuleType('h5py')
    h5.File = _File
    sys.modules['h5py'] = h5
    tb = types.ModuleType('transformers.tokenization_bert')
    tb.BasicTokenizer = BasicTokenizer
    sys.modules['transformers.tokenization_bert'] = tb
    for pkg in ('densephrases', 'densephrases.utils'):
        m = types.ModuleType(pkg)
        m.__path__ = []
        sys.modules[pkg] = m
    fu = types.ModuleType('densephrases.utils.file_utils')
    fu.is_tf_available, fu.is_torch_available = (lambda: False), (lambda: True)
    sys.modules['densephrases.utils.file_utils'] = fu
    du = types.ModuleType('densephrases.utils.data_utils')
    du.DataProcessor = object
    du.whitespace_tokenize = lambda text: text.strip().split() if text.strip() else []
    sys.modules['densephrases.utils.data_utils'] = du
    su = load('densephrases.utils.squad_utils', os.path.join(REF, 'utils', 'squad_utils.py'))
    su.TrueCaser = lambda path: None                                    # contexts are not true-cased
    load('densephrases.utils.squad_metrics', os.path.join(REF, 'utils', 'squad_metrics.py'))
    eu = load('densephrases.utils.embed_utils', os.path.join(REF, 'utils', 'embed_utils.py'))
    return su, eu


def feat_json(f):
    n = f.input_ids.index(0) if 0 in f.input_ids else len(f.input_ids)
    return {'input_ids': f.input_ids[:n], 'attention_mask': sum(f.attention_mask), 'token_type_ids': sorted(set(f.token_type_ids)),
            'tokens': f.tokens, 'token_to_orig_map': sorted(f.token_to_orig_map.items()), 'paragraph_len': f.paragraph_len,
            'title_offset': f.title_offset, 'span_idx': f.span_idx, 'par_idx': f.par_idx, 'doc_idx': f.doc_idx,
            'example_index': f.example_index, 'unique_id': f.unique_id}


def value_json(v):
    if isinstance(v, np.ndarray):
        if v.dtype == np.int8 or v.dtype == np.float32:
            return {'dtype': str(v.dtype), 'shape': list(v.shape), 'sha256': hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest()}
        return {'dtype': str(v.dtype), 'shape': list(v.shape), 'data': v.reshape(-1).tolist()}
    return v


def groups_json(rec):
    return {did: {'attrs': {k: value_json(v) for k, v in g.attrs.items()}, 'datasets': {k: value_json(v) for k, v in g.items()}}
            for did, g in rec.items()}


def main():
    su, eu = reference_modules()
    os.environ.setdefault('DATA_DIR', '')
    tok = Tokenizer29(dump_cases.tokenizer())
    data = dump_cases.documents()
    out = {'documents': data, 'cases': []}
    args = argparse.Namespace(truecase_path='unused')
    with tempfile.TemporaryDirectory() as tmp:
        for name, S, stride, title, L, thrs, off, scale, seed in dump_cases.CASES:
            examples = su.SquadV1Processor()._create_examples(data, 'dev', False, context_only=True, args=args)
            features, _ = su.squad_convert_examples_to_features(examples, tok, S, stride, 64, False, return_dataset='pt', threads=1,
                                                                tqdm_enabled=False, context_only=True, append_title=title)
            row_lo = [(f.input_ids.index(tok.sep_token_id) if title else 0) + 1 for f in features]
            start, logits = dump_cases.phrase_outputs(features, S, seed, row_lo)
            results = lambda: (su.ContextResult(f.unique_id, start[i], start[i], logits[i, :, 0], logits[i, :, 1])    # noqa: E731
                               for i, f in enumerate(features))
            case = {'name': name, 'features': [feat_json(f) for f in features], 'runs': []}
            for thr in thrs:
                path = os.path.join(tmp, f'{name}_{thr}.hdf5')
                eu.write_phrases(examples, features, results(), L, False, tok, path, thr, False, off, scale, has_title=title)
                case['runs'].append({'filter_threshold': thr, 'groups': groups_json(RECORD.pop(path))})
                print(name, thr, {d: len(g['datasets']['f2o_start']['data']) for d, g in case['runs'][-1]['groups'].items()})
            if name == dump_cases.FILTER_ONLY_CASE:
                path = os.path.join(tmp, f'{name}_filter.hdf5')
                eu.write_filter(examples, features, results(), tok, path, -1e8, False, has_title=title)
                case['filter_only'] = groups_json(RECORD.pop(path))
            out['cases'].append(case)
    path = os.path.join(ROOT, 'tests', 'golden', 'dump_reference.json.gz')
    with open(path, 'wb') as f, gzip.GzipFile(fileobj=f, mode='wb', mtime=0) as z:
        z.write(json.dumps(out, separators=(',', ':')).encode())
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
