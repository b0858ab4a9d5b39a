"""Phrase dump benchmark at the gen-vecs settings (Makefile gen-vecs: --max_seq_length 512 --doc_stride 500 --append_title):
synthetic documents, the random-weight phrase tower in bf16x3, thresholds -2.0 and -1e8, and the median of max(filter_start,
filter_end) over the first batch (random weights put every logit above -2.0, so that third threshold is the one that drops rows;
the median includes padding positions, so it keeps fewer than half of the valid rows).  Prints one JSON line per threshold:
documents/s and tokens/s, kept rows and device-to-host bytes against the reference's 6 KB (fp32 start + end) per token, seconds per
stage (features, forward, device select/quantise from CUDA events, host copies out of the pinned buffer, character offsets,
write), and the numpy restatement's post-processing time on the same fp32 outputs (the reference arm:
the rows copied to the host and selected / re-indexed / quantised there).

    python tools/bench_dump.py [--docs 64] [--batch 12]"""
import argparse
import json
import os
import sys
import tempfile
import timeit

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from densephrases_b200 import dump  # noqa: E402
from densephrases_b200.encoder import BertGeometry, Encoder, random_phrase_state_dict  # noqa: E402
from oracle import dump_ref  # noqa: E402
from tests import dump_cases  # noqa: E402


def corpus(n_docs, seed=0):
    rng = np.random.default_rng(seed)
    words = dump_cases.WORDS
    return [{'title': f'Document {d} {words[d % len(words)]}',
             'paragraphs': [{'context': ' '.join(words[i] for i in rng.integers(0, len(words), int(rng.integers(80, 400))))}
                            for _ in range(int(rng.integers(1, 6)))]} for d in range(n_docs)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--docs', type=int, default=64)
    ap.add_argument('--batch', type=int, default=12)
    a = ap.parse_args()
    S, stride, L = 512, 500, 10
    tok = dump_cases.tokenizer()
    geo = BertGeometry(vocab_size=max(tok.vocab.values()) + 1)
    enc = Encoder(geo, state_dict=random_phrase_state_dict(geo, 3), device=0, phrase_only=True, precise='bf16x3')
    gpu = torch.cuda.get_device_name(0)
    data = corpus(a.docs)
    t0 = timeit.default_timer()
    examples = dump.read_examples(data)
    features = dump.convert_examples_to_features(examples, tok, S, stride, True)
    t_feat = timeit.default_timer() - t0
    toffs = dump.title_offsets(features, tok, True)
    tokens = sum(len(f.tokens) - 1 - (t + 1) for f, t in zip(features, toffs))
    median = None
    for _, _, filt in dump.phrase_outputs(enc, features[:a.batch], a.batch):     # warm-up
        median = float(np.median(filt.amax(-1).cpu().numpy()))
    for thr in (-2.0, -1e8, median):
        tm = {}
        t0 = timeit.default_timer()
        groups = dump.dump_documents(examples, features, dump.phrase_outputs(enc, features, a.batch), tok, L, False, thr, -2.0, 20.0, True,
                                     timings=tm)
        t_dump = timeit.default_timer() - t0
        with tempfile.TemporaryDirectory() as tmp:
            t0 = timeit.default_timer()
            dump.write_dump(os.path.join(tmp, 'bench.hdf5'), groups)
            t_write = timeit.default_timer() - t0
        # reference arm: the same fp32 outputs on the host, selected / re-indexed / quantised by the numpy restatement
        t_ref, t_copy = 0.0, 0.0
        docs = dump.documents(examples, features)
        outs = list(dump.phrase_outputs(enc, features, a.batch))
        t0 = timeit.default_timer()
        host = [(s.cpu().numpy(), f.cpu().numpy()) for _, s, f in outs]
        t_copy = timeit.default_timer() - t0
        start = np.concatenate([h[0] for h in host])
        filt = np.concatenate([h[1] for h in host])
        del outs, host
        t0 = timeit.default_timer()
        for idxs in docs:
            lo = [toffs[i] + 1 for i in idxs]
            hi = [len(features[i].tokens) - 1 for i in idxs]
            rows = lambda x: np.concatenate([x[i, l:h] for i, l, h in zip(idxs, lo, hi)])       # noqa: E731
            dump_ref.select_document(rows(start), rows(filt[..., 0]), rows(filt[..., 1]), np.subtract(hi, lo), L, thr, -2.0, 20.0)
        t_ref = timeit.default_timer() - t0
        del start, filt
        kept = sum(len(g[0]['f2o_start']) for g in groups.values())
        total = t_feat + t_dump + t_write
        print(json.dumps({
            'gpu': gpu, 'filter_threshold': thr, 'docs': len(groups), 'features': len(features), 'tokens': tokens, 'kept_rows': kept,
            'docs_per_s': len(groups) / total, 'tokens_per_s': tokens / total,
            'd2h_bytes': tm.get('d2h_bytes', 0), 'reference_d2h_bytes': tokens * 6144,
            'seconds': {'features': t_feat, 'forward': tm.get('forward', 0.0), 'select_device': tm.get('select_device_ms', 0.0) / 1e3,
                        'select_host': tm.get('select', 0.0), 'copy': tm.get('copy', 0.0), 'offsets': tm.get('offsets', 0.0),
                        'write': t_write, 'total': total},
            'reference_arm_seconds': {'copy_fp32': t_copy, 'numpy_select': t_ref}}))


if __name__ == '__main__':
    main()
