"""TEST INFRASTRUCTURE.  Plain PyTorch fp32 restatement of the phrase side of the reference Encoder
(densephrases/encoder.py:92-99 embed_phrase, :137-144 filter_linear): the phrase tower over every token, built on the query
restatement's `oracle.encoder_ref.tower_forward`, plus the 768 -> 2 filter head.  tests/golden/make_phrase_golden.py pins it
against the unmodified reference class (tests/golden/encoder_phrase.npz)."""
import torch
import torch.nn.functional as F

from oracle.encoder_ref import tower_forward


def embed_phrase(sd, ids, mask, tt, dtype=torch.float32):
    """-> (start [B,S,768], end (the same tensor), filter_start_logits [B,S], filter_end_logits [B,S]) in `dtype` (fp32: the
    restatement; fp64: the high-precision truth) on ids.device."""
    with torch.no_grad():
        x = tower_forward(sd, 'phrase_encoder', ids, mask, tt, dtype=dtype)
        logits = F.linear(x, sd['filter_linear.weight'].to(ids.device, dtype), sd['filter_linear.bias'].to(ids.device, dtype))
    return x, x, logits[..., 0], logits[..., 1]
