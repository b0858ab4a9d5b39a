"""TEST INFRASTRUCTURE.  Plain PyTorch restatement of Encoder.forward with a context and a question (reference
densephrases/encoder.py:120-153, 206-208, 260): the two query towers' [CLS] vectors (oracle.encoder_ref), the phrase tower and
filter head (tests/phrase_ref), and the join start . q_start, end . q_end.  tests/golden/make_rc_golden.py pins it against the
unmodified reference class (tests/golden/encoder_rc.npz)."""
import torch

from densephrases_b200.encoder import random_phrase_state_dict, random_state_dict
from oracle import encoder_ref
from tests import phrase_ref


def rc_state_dict(config, seed):
    """Seeded random weights of all three towers and the filter head, in the reference's naming."""
    sd = random_state_dict(config, seed)
    sd.update(random_phrase_state_dict(config, seed + 7))
    return sd


def read(sd, ids, mask, tt, qids, qmask, qtt, dtype=torch.float32):
    """-> (start_logits, end_logits, filter_start_logits, filter_end_logits), each [B,S] in `dtype`, on ids.device."""
    with torch.no_grad():
        qs, qe = encoder_ref.embed_query(sd, qids, qmask, qtt, dtype=dtype)
        x, _, fs, fe = phrase_ref.embed_phrase(sd, ids, mask, tt, dtype=dtype)
        return x.matmul(qs.transpose(1, 2)).squeeze(-1), x.matmul(qe.transpose(1, 2)).squeeze(-1), fs, fe
