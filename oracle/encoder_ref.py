"""oracle/encoder_ref.py -- TEST INFRASTRUCTURE.  Plain PyTorch fp32 restatement of the query-tower forward
(HF BertModel, transformers 2.9.0 semantics, SURVEY.md Appendix B) used by Encoder.embed_query
(reference densephrases/encoder.py:101-118).  It is pinned against the reference class itself:
tests/golden/make_encoder_golden.py imports the reference densephrases/encoder.py, runs it on
seeded weights/inputs and stores the outputs; tests/test_encoder.py checks this restatement against those fixtures, so it
can stand in for the reference wherever the reference repository is not present."""
import math

import torch
import torch.nn.functional as F


def tower_forward(sd, prefix, ids, mask, tt, layers=12, heads=12):
    """-> hidden states [B,S,768] of one tower, fp32, on ids.device."""
    def w(name):
        return sd[f'{prefix}.{name}'].to(ids.device, torch.float32)
    B, S = ids.shape
    x = F.embedding(ids, w('embeddings.word_embeddings.weight')) + w('embeddings.position_embeddings.weight')[:S][None] \
        + F.embedding(tt, w('embeddings.token_type_embeddings.weight'))
    x = F.layer_norm(x, (x.shape[-1],), w('embeddings.LayerNorm.weight'), w('embeddings.LayerNorm.bias'), eps=1e-12)
    bias_mask = (1.0 - mask.to(torch.float32))[:, None, None, :] * -10000.0
    H = x.shape[-1]
    dh = H // heads
    for l in range(layers):
        p = f'encoder.layer.{l}'
        def lin(t, name):
            return F.linear(t, w(f'{p}.{name}.weight'), w(f'{p}.{name}.bias'))
        q = lin(x, 'attention.self.query').view(B, S, heads, dh).transpose(1, 2)
        k = lin(x, 'attention.self.key').view(B, S, heads, dh).transpose(1, 2)
        v = lin(x, 'attention.self.value').view(B, S, heads, dh).transpose(1, 2)
        probs = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh) + bias_mask, dim=-1)
        ctx = (probs @ v).transpose(1, 2).reshape(B, S, H)
        a = F.layer_norm(lin(ctx, 'attention.output.dense') + x, (H,), w(f'{p}.attention.output.LayerNorm.weight'),
                         w(f'{p}.attention.output.LayerNorm.bias'), eps=1e-12)
        h = lin(a, 'intermediate.dense')
        h = 0.5 * h * (1.0 + torch.erf(h / math.sqrt(2.0)))
        x = F.layer_norm(lin(h, 'output.dense') + a, (H,), w(f'{p}.output.LayerNorm.weight'), w(f'{p}.output.LayerNorm.bias'), eps=1e-12)
    return x


def embed_query(sd, ids, mask, tt):
    """== Encoder.embed_query: (query_start [B,1,768], query_end [B,1,768])."""
    with torch.no_grad():
        s = tower_forward(sd, 'query_start_encoder', ids, mask, tt)[:, :1, :]
        e = tower_forward(sd, 'query_end_encoder', ids, mask, tt)[:, :1, :]
    return s, e
