"""Single-passage reading on one GPU, on a SQuAD-dev-shaped synthetic workload: ~10^4 features (1-3 per example) of context S = 384
with questions of Sq = 64, n_best 20, max_answer_length 10, and the 7 thresholds of `make filter-test`.
Reports Encoder.forward with both sides (dph_encoder_read) per precision mode, the span decoder (dph_rc_spans) per threshold,
compute_predictions_logits per threshold, the whole filter test (one forward, then decode + squad_evaluate per threshold), the
reference's torch fp32 forward on the same GPU (tests/rc_ref_torch.py, TF32 off) on a slice, and the reference's Python span
loop (a restatement of squad_metrics.py:490-544, which reads every logit through Python) on the host over a slice.
    python tools/bench_rc.py [--features 10240] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

S, SQ, N_BEST, L, SEED, VOCAB = 384, 64, 20, 10, 7, 28996


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    return {'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': q}


def workload(F, rng):
    """Features padded to S with real lengths over [S/2, S]: [CLS] + question-free context + [SEP], every context token mapped to a
    word (word pieces share words), token_is_max_context False on the first quarter of every window but an example's first."""
    from densephrases_b200.encoder import synthetic_context_batch, synthetic_query_batch
    ids, mask, tt = synthetic_context_batch(F, S, VOCAB, SEED)
    qids, qmask, qtt = synthetic_query_batch(F, SQ, VOCAB, SEED + 1)
    sizes = []
    while sum(sizes) < F:
        sizes.append(int(rng.choice([1, 1, 1, 1, 1, 2, 2, 3])))
    sizes[-1] -= sum(sizes) - F
    sizes = [s for s in sizes if s > 0]
    examples, features = [], []
    words = ['w%d' % i for i in range(400)]
    for x, n in enumerate(sizes):
        examples.append(types.SimpleNamespace(qas_id=f'q{x}', doc_tokens=[words[int(i)] for i in rng.integers(0, 400, 400)],
                                              answers=[{'text': 'w1 w2'}], context_text=''))
        for j in range(n):
            f = len(features)
            nt = int(mask[f].sum())
            toks = ['[CLS]'] + [words[int(i)] for i in rng.integers(0, 400, nt - 2)] + ['[SEP]']
            t2o = {t: t - 1 for t in range(1, nt - 1)}
            tmc = {t: (j == 0 or t > nt // 4) for t in range(1, nt - 1)}
            features.append(types.SimpleNamespace(example_index=x, unique_id=f, qas_id=f'q{x}', tokens=toks, token_to_orig_map=t2o,
                                                  token_is_max_context=tmc))
    return examples, features, dict(ids=ids, mask=mask, tt=tt, qids=qids, qmask=qmask, qtt=qtt)


def reference_loop(features, logits, thr, lo, hi):
    """The reference's per-feature enumeration (squad_metrics.py:490-544) over logits as Python lists (to_list), features lo..hi."""
    st, en, sf, ef = (x[lo:hi].tolist() for x in logits)
    n = 0
    prelim = []
    for i, f in enumerate(features[lo:hi]):
        for s in range(len(f.tokens)):
            for e in range(s, min(len(f.tokens), s + L - 1)):
                if s not in f.token_to_orig_map or e not in f.token_to_orig_map or not f.token_is_max_context.get(s, False) or e - s + 1 > L:
                    continue
                n += 1
                if sf[i][s] < thr or ef[i][e] < thr:
                    continue
                prelim.append((i, s, e, st[i][s], en[i][e]))
    return sorted(prelim, key=lambda p: p[3] + p[4], reverse=True), n


def events_ms(fn, reps=1):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--features', type=int, default=10240)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from densephrases_b200 import rc
    from densephrases_b200.encoder import BertGeometry, Encoder
    from tests import rc_ref_torch
    rng = np.random.default_rng(SEED)
    F = args.features
    res = {'workload': {'features': F, 'S': S, 'Sq': SQ, 'n_best_size': N_BEST, 'max_answer_length': L,
                        'thresholds': list(rc.FILTER_TEST_THRESHOLDS)}, **gpu_info()}
    examples, features, t = workload(F, rng)
    res['workload']['examples'] = len(examples)
    geo = BertGeometry(vocab_size=VOCAB)
    sd = rc_ref_torch.rc_state_dict(geo, SEED)
    enc = Encoder(geo, state_dict=sd)
    dev = {k: v.cuda() for k, v in t.items()}
    B = 64

    def forward():
        outs = [enc(input_ids=dev['ids'][i:i + B], attention_mask=dev['mask'][i:i + B], token_type_ids=dev['tt'][i:i + B],
                    input_ids_=dev['qids'][i:i + B], attention_mask_=dev['qmask'][i:i + B], token_type_ids_=dev['qtt'][i:i + B])
                for i in range(0, F, B)]
        return tuple(torch.cat([o[j] for o in outs]) for j in range(4))
    res['forward'] = {}
    for mode in ('tf32', 'bf16x3', '3xtf32'):
        enc.set_precision(mode)
        enc(input_ids=dev['ids'][:B], attention_mask=dev['mask'][:B], token_type_ids=dev['tt'][:B], input_ids_=dev['qids'][:B],
            attention_mask_=dev['qmask'][:B], token_type_ids_=dev['qtt'][:B])
        ms = events_ms(forward)
        res['forward'][mode] = {'ms': round(ms, 1), 'features_per_s': round(F / ms * 1e3)}
        print(mode, res['forward'][mode], flush=True)
    enc.set_precision('bf16x3')
    logits = forward()
    torch.backends.cuda.matmul.allow_tf32 = False
    gsd = {n: w.cuda() for n, w in sd.items()}
    sl = 256
    ref_fw = lambda: [rc_ref_torch.read(gsd, *(dev[k][i:i + B] for k in ('ids', 'mask', 'tt', 'qids', 'qmask', 'qtt'))) for i in range(0, sl, B)]  # noqa: E731
    ref_fw()
    ms = events_ms(ref_fw)
    res['torch_fp32_forward'] = {'features': sl, 'ms': round(ms, 1), 'features_per_s': round(sl / ms * 1e3)}
    print('torch fp32', res['torch_fp32_forward'], flush=True)
    del gsd
    # decoder alone and compute_predictions_logits, per threshold
    n_tokens, start_ok, end_ok = rc.feature_masks(features, S)
    ex_off = np.concatenate([[0], np.cumsum(np.bincount([f.example_index for f in features]))]).astype(np.int64)
    g_masks = [torch.from_numpy(x).cuda() for x in (n_tokens, start_ok.view(np.int32), end_ok.view(np.int32), ex_off)]
    res['decode'] = {}
    for thr in rc.FILTER_TEST_THRESHOLDS:
        rc.best_spans(*logits, *g_masks, L, thr, N_BEST)
        t0 = time.perf_counter()
        sp = rc.best_spans(*logits, *g_masks, L, thr, N_BEST)
        dec = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        preds, stat = rc.compute_predictions_logits(examples, features, logits, N_BEST, L, False, None, None, None, False, False, 0.0, None, thr, None)
        full = (time.perf_counter() - t0) * 1e3
        res['decode'][f'{thr:g}'] = {'dph_rc_spans_ms': round(dec, 2), 'compute_predictions_logits_ms': round(full, 1),
                                     'save_rate': round(stat['save_rate'], 4), 'spans': int(sp.total_count.sum())}
        print(thr, res['decode'][f'{thr:g}'], flush=True)
    for i, f in enumerate(features):
        for k, n in (('ids', 'input_ids'), ('mask', 'attention_mask'), ('tt', 'token_type_ids'), ('qids', 'input_ids_'),
                     ('qmask', 'attention_mask_'), ('qtt', 'token_type_ids_')):
            setattr(f, n, t[k][i].numpy())
    t0 = time.perf_counter()
    ft = rc.filter_test(enc, examples, features, None, batch_size=B)
    torch.cuda.synchronize()
    res['filter_test'] = {'s': round(time.perf_counter() - t0, 2), 'result': {k: round(v, 4) for k, v in ft.items()}}
    print('filter test', res['filter_test']['s'], 's', flush=True)
    host = [x.cpu().numpy() for x in logits]
    sl = 200
    t0 = time.perf_counter()
    reference_loop(features, host, -2.0, 0, sl)
    s_ref = time.perf_counter() - t0
    res['reference_python_loop'] = {'features': sl, 's': round(s_ref, 3), 'features_per_s': round(sl / s_ref, 1),
                                    'filter_test_s_extrapolated': round(s_ref / sl * F * len(rc.FILTER_TEST_THRESHOLDS), 1)}
    print('reference loop', res['reference_python_loop'], flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_rc.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
