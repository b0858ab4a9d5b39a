"""Generates tests/golden/encoder_phrase.npz by running the UNMODIFIED reference class
/root/reference/densephrases/encoder.py:Encoder (fp32, CPU, eager), loaded like make_encoder_golden.py, through
forward(input_ids=..., return_phrase=True) on seeded random phrase-tower and filter weights
(densephrases_b200.encoder.random_phrase_state_dict) and synthetic ragged contexts (synthetic_context_batch).
Stored: inputs, seed, all filter logits, and the token vectors of a subset of rows (every row for S <= 64; else every 8th
row of each sequence plus its first and last real token) so the fixture stays small.  The weights are regenerated from the seed.
Run in the build container (needs /root/reference):  python tests/golden/make_phrase_golden.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from densephrases_b200.encoder import BertGeometry, random_phrase_state_dict, synthetic_context_batch  # noqa: E402
from tests import phrase_ref  # noqa: E402
from tests.golden.make_encoder_golden import load_reference_encoder  # noqa: E402

CASES = {'b3_s48': (3, 48, False), 'b2_s100': (2, 100, True), 'b2_s384': (2, 384, False), 'b1_s512': (1, 512, True)}


def stored_rows(mask):
    """Flat row indices b * S + s kept for the token vectors."""
    B, S = mask.shape
    if S <= 64:
        return np.arange(B * S, dtype=np.int64)
    rows = []
    for b in range(B):
        n = int(mask[b].sum())
        rows.append(sorted(set(range(0, S, 8)) | {0, n - 1}))
        rows[-1] = [b * S + s for s in rows[-1]]
    return np.array([r for rs in rows for r in rs], dtype=np.int64)


if __name__ == '__main__':
    from transformers import BertConfig, BertModel
    torch.manual_seed(0)
    seed, vocab = 20241015, 28996
    geo = BertGeometry(vocab_size=vocab)
    cfg = BertConfig(vocab_size=vocab, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                     max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12, hidden_act='gelu',
                     hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    RefEncoder = load_reference_encoder()
    model = RefEncoder(cfg, tokenizer=None, transformer_cls=BertModel).eval()
    sd = random_phrase_state_dict(geo, seed)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all(not m.startswith(('phrase_encoder.encoder', 'phrase_encoder.embeddings', 'filter_linear')) for m in missing), missing
    out = {}
    for name, (B, S, type_split) in CASES.items():
        ids, mask, tt = synthetic_context_batch(B, S, vocab, seed + S, type_split=type_split)
        with torch.no_grad():
            start, end, fs, fe = model(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
        assert end is start
        rs, _, rfs, rfe = phrase_ref.embed_phrase(sd, ids, mask, tt)
        d = max((start - rs).abs().max().item(), (fs - rfs).abs().max().item(), (fe - rfe).abs().max().item())
        print(name, 'reference class vs torch restatement: max abs diff', d, '| out scale', start.abs().mean().item(),
              '| filter scale', fs.abs().mean().item())
        assert d < 2e-4, d
        rows = stored_rows(mask.numpy())
        out[f'{name}_ids'], out[f'{name}_mask'], out[f'{name}_tt'] = ids.numpy(), mask.numpy(), tt.numpy()
        out[f'{name}_rows'] = rows
        out[f'{name}_vec'] = start.reshape(B * S, -1)[torch.from_numpy(rows)].numpy()
        out[f'{name}_filter_start'], out[f'{name}_filter_end'] = fs.numpy(), fe.numpy()
    out['seed'] = np.array(seed)
    out['vocab'] = np.array(vocab)
    path = os.path.join(ROOT, 'tests', 'golden', 'encoder_phrase.npz')
    np.savez_compressed(path, **out)
    print('wrote tests/golden/encoder_phrase.npz', os.path.getsize(path), 'bytes')
