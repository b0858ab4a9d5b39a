"""Encoder: forward of the DensePhrases encoder on the H100 tensor cores.

Mirror of reference densephrases/encoder.py (class Encoder):
- query side: `embed_query` (:101-118) and `forward(input_ids_=..., attention_mask_=..., token_type_ids_=..., return_query=True)`
  (:146-152) -> (query_start, query_end), each [B,1,768], computed by two independent BERT-base towers whose weights come from the
  `query_start_encoder.*` / `query_end_encoder.*` entries of the reference state dict;
- phrase side: `embed_phrase` (:92-99) and `forward(input_ids=..., attention_mask=..., token_type_ids=..., return_phrase=True)`
  (:130-144) -> (start, end, filter_start_logits, filter_end_logits): the `phrase_encoder.*` tower over every token (start and end
  are the same [B,S,768] tensor) and the `filter_linear` head (768 -> 2) on it.
Legacy names `bert_start.*` / `bert_q_start.*` / `bert_q_end.*` are accepted like single_utils.backward_compat (:36-56).  Training
losses are out of scope (SURVEY.md 8a).  Compute: libdph_b200 (wgmma TF32 / bf16 GEMMs, tensor-core attention, fp32 everything else)."""
import ctypes as C

import numpy as np
import torch

from . import _lib as L

LEGACY = {'bert_q_start': 'query_start_encoder', 'bert_q_end': 'query_end_encoder', 'bert_start': 'phrase_encoder'}
TOWERS = ('query_start_encoder', 'query_end_encoder')
PHRASE_TOWER = 'phrase_encoder'              # tower 2 of libdph_b200
MAX_PHRASE_LEN = 512                         # longest context the phrase path runs (also bounded by max_position_embeddings)


class BertGeometry(object):
    """The subset of HF BertConfig this path needs (SpanBERT-base-cased defaults, options.py:23)."""

    def __init__(self, vocab_size=28996, max_position_embeddings=512, type_vocab_size=2, hidden_size=768, num_hidden_layers=12,
                 num_attention_heads=12, intermediate_size=3072, **_):
        assert (hidden_size, num_hidden_layers, num_attention_heads, intermediate_size) == (768, 12, 12, 3072), \
            'only the BERT-base geometry of the released DensePhrases models is built'
        self.vocab_size, self.max_position_embeddings, self.type_vocab_size = vocab_size, max_position_embeddings, type_vocab_size
        self.hidden_size, self.num_hidden_layers = hidden_size, num_hidden_layers
        self.num_attention_heads, self.intermediate_size = num_attention_heads, intermediate_size


def tower_blob(sd, prefix, config):
    """Pack one tower's tensors into the flat fp32 blob libdph_b200 expects (layout documented in csrc/encoder.cu)."""
    def t(name):
        return sd[f'{prefix}.{name}'].detach().to(torch.float32).cpu().contiguous().view(-1)
    parts = [t('embeddings.word_embeddings.weight'), t('embeddings.position_embeddings.weight'), t('embeddings.token_type_embeddings.weight'),
             t('embeddings.LayerNorm.weight'), t('embeddings.LayerNorm.bias')]
    for l in range(config.num_hidden_layers):
        p = f'encoder.layer.{l}'
        parts += [t(f'{p}.attention.self.query.weight'), t(f'{p}.attention.self.key.weight'), t(f'{p}.attention.self.value.weight'),
                  t(f'{p}.attention.self.query.bias'), t(f'{p}.attention.self.key.bias'), t(f'{p}.attention.self.value.bias'),
                  t(f'{p}.attention.output.dense.weight'), t(f'{p}.attention.output.dense.bias'),
                  t(f'{p}.attention.output.LayerNorm.weight'), t(f'{p}.attention.output.LayerNorm.bias'),
                  t(f'{p}.intermediate.dense.weight'), t(f'{p}.intermediate.dense.bias'),
                  t(f'{p}.output.dense.weight'), t(f'{p}.output.dense.bias'), t(f'{p}.output.LayerNorm.weight'), t(f'{p}.output.LayerNorm.bias')]
    return torch.cat(parts).numpy()


def canonical_state_dict(sd):
    """Legacy tower names (bert_start / bert_q_start / bert_q_end) -> the current ones, like single_utils.backward_compat."""
    return {next((k.replace(old, new, 1) for old, new in LEGACY.items() if k.startswith(old)), k): v for k, v in sd.items()}


def check_phrase_shape(config, shape):
    """-> (B, S) of a phrase-path batch, or ValueError: 2-D, 1 <= S <= min(512, max_position_embeddings) and 1 <= B <= 65535
    (the attention kernels put the batch on grid.y)."""
    if len(shape) != 2:
        raise ValueError(f'input_ids must be [B, S], got {tuple(shape)}')
    B, S = int(shape[0]), int(shape[1])
    limit = min(MAX_PHRASE_LEN, config.max_position_embeddings)
    if not 1 <= S <= limit:
        raise ValueError(f'sequence length {S} outside 1..{limit} (the phrase path runs up to min(512, max_position_embeddings))')
    if not 1 <= B <= 65535:
        raise ValueError(f'batch size {B} outside 1..65535')
    return B, S


class Encoder(object):
    """phrase_only: the encoder carries only the phrase tower and the filter head (runtime.load_encoder(phrase_only=True));
    otherwise the two query towers are required and the phrase tower and filter head are loaded when the state dict has them."""

    def __init__(self, config, tokenizer=None, state_dict=None, device=0, precise='bf16x3', phrase_only=False):
        self.config = config if isinstance(config, BertGeometry) else BertGeometry(**{k: getattr(config, k) for k in
                                                                                     ('vocab_size', 'max_position_embeddings', 'type_vocab_size', 'hidden_size',
                                                                                      'num_hidden_layers', 'num_attention_heads', 'intermediate_size')})
        self.tokenizer = tokenizer
        self.device_index = device
        self.device = torch.device('cuda', device)
        self._h = C.c_void_p()
        L.check(L.lib().dph_encoder_create(C.byref(self._h), device, self.config.vocab_size, self.config.max_position_embeddings,
                                           self.config.type_vocab_size))
        self.training = False
        self.phrase_only = phrase_only
        self.has_query = self.has_phrase = self.has_filter = False
        self.set_precision(precise)
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def __del__(self):
        h, self._h = getattr(self, '_h', None), None
        if h and L is not None and L._lib is not None:
            L._lib.dph_encoder_free(h)

    MODES = {'tf32': 0, '3xtf32': 1, 'bf16x3': 2}      # name -> dph_encoder_set_precision argument

    def set_precision(self, precise):
        """'bf16x3' (default of this class): meets the north star's 1e-3 tolerance on the query vectors at nearly the speed of 'tf32';
        'tf32' / False: 1xTF32 GEMMs (== torch 1.9's default for fp32 matmuls on Ampere+), fastest, ~2e-2;
        '3xtf32' / True: 3xTF32 split, fp32-accurate; 'bf16x3': bf16 (hi, lo) planes, three bf16 MMAs per product -- both meet
        the 1e-3 tolerance of the north star, bf16x3 at the speed of 'tf32'."""
        mode = precise if isinstance(precise, str) else ('3xtf32' if precise else 'tf32')
        if mode not in self.MODES:
            raise ValueError(f'unknown precision mode {mode!r}; choose one of {sorted(self.MODES)}')
        self.mode = mode
        self.precise = mode != 'tf32'
        L.check(L.lib().dph_encoder_set_precision(self._h, self.MODES[mode]))

    def precision_modes(self):
        return list(self.MODES)

    @staticmethod
    def mma_multiplier(mode):
        """Tensor-core work issued per algorithmic flop, in TF32-MMA equivalents (a bf16 MMA costs half a TF32 one)."""
        return {'tf32': 1.0, '3xtf32': 3.0, 'bf16x3': 1.5}[mode]

    def default_mode(self):
        """The fastest mode that meets the north star's 1e-3 tolerance on the [CLS] vectors (tests/test_encoder.py)."""
        return 'bf16x3' if 'bf16x3' in self.MODES else '3xtf32'

    def set_attention(self, tensor_core=True):
        """True (default): tensor-core attention for S <= 64, and on the phrase path at every S; False: fp32 SIMT attention always
        (S <= 384)."""
        L.check(L.lib().dph_encoder_set_attention(self._h, int(bool(tensor_core))))

    # -- torch.nn.Module-style surface the callers touch (embed_utils.py:393, single_utils.py:116) --
    def eval(self):
        self.training = False
        return self

    def to(self, device):
        return self

    def load_state_dict(self, sd, strict=False):
        sd = canonical_state_dict(sd)
        need = L.lib().dph_encoder_tower_floats(self._h)

        def load(tower, prefix):
            blob = np.ascontiguousarray(tower_blob(sd, prefix, self.config), dtype=np.float32)
            assert blob.size == need, f'{prefix}: {blob.size} floats, expected {need}'
            L.check(L.lib().dph_encoder_load_tower(self._h, tower, blob.ctypes.data_as(C.c_void_p), L.MEM_HOST))
        if not self.phrase_only:
            for tower, prefix in enumerate(TOWERS):
                load(tower, prefix)
            self.has_query = True
        has_phrase = any(k.startswith(PHRASE_TOWER + '.') for k in sd)
        if self.phrase_only and not has_phrase:
            raise KeyError(f'phrase-only encoder: the state dict has no {PHRASE_TOWER}.* (or legacy bert_start.*) weights')
        if has_phrase:
            load(len(TOWERS), PHRASE_TOWER)
            self.has_phrase = True
        if 'filter_linear.weight' in sd:
            W = np.ascontiguousarray(sd['filter_linear.weight'].detach().to(torch.float32).cpu().numpy())
            b = np.ascontiguousarray(sd['filter_linear.bias'].detach().to(torch.float32).cpu().numpy())
            assert W.shape == (2, self.config.hidden_size) and b.shape == (2,), f'filter_linear: {W.shape}, {b.shape}'
            L.check(L.lib().dph_encoder_load_filter(self._h, W.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), L.MEM_HOST))
            self.has_filter = True
        return self

    def _check_ids(self, input_ids, token_type_ids):
        if not input_ids.is_cuda:       # ids normally come from the CPU tokenizer: range check before the copy (torch.nn.Embedding raises IndexError)
            if int(input_ids.min()) < 0 or int(input_ids.max()) >= self.config.vocab_size:
                raise IndexError(f'input_ids outside [0, {self.config.vocab_size})')
            if int(token_type_ids.min()) < 0 or int(token_type_ids.max()) >= self.config.type_vocab_size:
                raise IndexError(f'token_type_ids outside [0, {self.config.type_vocab_size})')

    def embed_query(self, input_ids_, attention_mask_, token_type_ids_):
        """int64 [B,S] tensors (cuda or cpu) -> (query_start, query_end) float32 [B,1,768] on the GPU."""
        if not self.has_query:
            raise NotImplementedError('this encoder has no query towers (phrase-only)')
        B, S = input_ids_.shape
        self._check_ids(input_ids_, token_type_ids_)
        ids, mask, tt = (x.to(self.device, dtype=torch.int64).contiguous() for x in (input_ids_, attention_mask_, token_type_ids_))
        start = torch.empty((B, 1, self.config.hidden_size), dtype=torch.float32, device=self.device)
        end = torch.empty_like(start)
        L.check(L.lib().dph_encoder_set_stream(self._h, C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))
        L.check(L.lib().dph_encoder_embed_query(self._h, ids.data_ptr(), mask.data_ptr(), tt.data_ptr(), B, S, start.data_ptr(), end.data_ptr(),
                                                L.MEM_DEVICE))
        return start, end

    def _phrase(self, input_ids, attention_mask, token_type_ids, with_filter):
        if not self.has_phrase:
            raise NotImplementedError('this encoder has no phrase tower: load a state dict with phrase_encoder.* weights')
        if with_filter and not self.has_filter:
            raise NotImplementedError('this encoder has no filter head: load a state dict with filter_linear.{weight,bias}')
        B, S = check_phrase_shape(self.config, input_ids.shape)
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        self._check_ids(input_ids, token_type_ids)
        ids, mask, tt = (x.to(self.device, dtype=torch.int64).contiguous() for x in (input_ids, attention_mask, token_type_ids))
        out = torch.empty((B, S, self.config.hidden_size), dtype=torch.float32, device=self.device)
        filt = torch.empty((B, S, 2), dtype=torch.float32, device=self.device) if with_filter else None
        L.check(L.lib().dph_encoder_set_stream(self._h, C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))
        L.check(L.lib().dph_encoder_embed_phrase(self._h, ids.data_ptr(), mask.data_ptr(), tt.data_ptr(), B, S, out.data_ptr(),
                                                 filt.data_ptr() if with_filter else None, L.MEM_DEVICE))
        return out, filt

    def embed_phrase(self, input_ids, attention_mask, token_type_ids):
        """int64 [B,S] tensors (cuda or cpu), S <= 512 -> (start, end) float32 [B,S,768] on the GPU; `end` is `start` (encoder.py:92-99)."""
        out, _ = self._phrase(input_ids, attention_mask, token_type_ids, with_filter=False)
        return out, out

    def forward(self, input_ids=None, attention_mask=None, token_type_ids=None, input_ids_=None, attention_mask_=None, token_type_ids_=None,
                return_phrase=False, return_query=False, **unused):
        if input_ids is not None and return_phrase:
            out, filt = self._phrase(input_ids, attention_mask, token_type_ids, with_filter=True)
            return out, out, filt[..., 0], filt[..., 1]
        if input_ids is not None or not return_query:
            raise NotImplementedError('on the GPU: the phrase side with return_phrase=True (encoder.py:130-144) and the query side with '
                                      'return_query=True (encoder.py:146-152)')
        assert len(input_ids_.size()) == 2
        return self.embed_query(input_ids_, attention_mask_, token_type_ids_)

    __call__ = forward


def random_state_dict(config, seed, prefixes=TOWERS, std=0.02):
    """Seeded random weights in the reference's state-dict naming (no checkpoint is reachable offline).  LayerNorm gains
    are 1 + noise and biases are noise so every parameter matters in parity tests."""
    g = torch.Generator().manual_seed(seed)
    H, FF = config.hidden_size, config.intermediate_size

    def rn(*shape, s=std):
        return torch.randn(*shape, generator=g) * s

    sd = {}
    for prefix in prefixes:
        sd[f'{prefix}.embeddings.word_embeddings.weight'] = rn(config.vocab_size, H)
        sd[f'{prefix}.embeddings.position_embeddings.weight'] = rn(config.max_position_embeddings, H)
        sd[f'{prefix}.embeddings.token_type_embeddings.weight'] = rn(config.type_vocab_size, H)
        sd[f'{prefix}.embeddings.LayerNorm.weight'] = 1.0 + rn(H, s=0.1)
        sd[f'{prefix}.embeddings.LayerNorm.bias'] = rn(H, s=0.1)
        for l in range(config.num_hidden_layers):
            p = f'{prefix}.encoder.layer.{l}'
            for name, shape in (('attention.self.query', (H, H)), ('attention.self.key', (H, H)), ('attention.self.value', (H, H)),
                                ('attention.output.dense', (H, H)), ('intermediate.dense', (FF, H)), ('output.dense', (H, FF))):
                sd[f'{p}.{name}.weight'] = rn(*shape, s=0.04)
                sd[f'{p}.{name}.bias'] = rn(shape[0], s=0.05)
            for name in ('attention.output.LayerNorm', 'output.LayerNorm'):
                sd[f'{p}.{name}.weight'] = 1.0 + rn(H, s=0.1)
                sd[f'{p}.{name}.bias'] = rn(H, s=0.1)
    return sd


def random_phrase_state_dict(config, seed, std=0.02):
    """Seeded random phrase-tower (`phrase_encoder.*`) and `filter_linear` weights in the reference's naming; the tower follows
    random_state_dict, the filter head draws from its own generator after it."""
    sd = random_state_dict(config, seed, prefixes=(PHRASE_TOWER,), std=std)
    g = torch.Generator().manual_seed(seed + 1)
    sd['filter_linear.weight'] = torch.randn(2, config.hidden_size, generator=g) * std
    sd['filter_linear.bias'] = torch.randn(2, generator=g) * 0.05
    return sd


def synthetic_query_batch(B, S, vocab_size, seed):
    """SURVEY 8d: uniform token ids, 6-20 real tokens + [CLS]/[SEP] (ids 101/102), zero padding to S, all token types 0."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros((B, S), dtype=torch.int64)
    mask = torch.zeros((B, S), dtype=torch.int64)
    for b in range(B):
        n = int(torch.randint(6, 21, (1,), generator=g))
        n = min(n, S - 2)
        ids[b, 0] = 101
        ids[b, 1:1 + n] = torch.randint(1000, vocab_size, (n,), generator=g)
        ids[b, 1 + n] = 102
        mask[b, :n + 2] = 1
    return ids, mask, torch.zeros_like(ids)


def synthetic_context_batch(B, S, vocab_size, seed, type_split=False):
    """Contexts padded to S: [CLS] + uniform token ids + [SEP] (ids 101/102) over a real length drawn uniformly from [S/2, S]
    (at least 2), so a batch has ragged masks.  type_split: the tokens after the first third get token type 1."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros((B, S), dtype=torch.int64)
    mask = torch.zeros((B, S), dtype=torch.int64)
    tt = torch.zeros((B, S), dtype=torch.int64)
    for b in range(B):
        n = max(2, int(torch.randint(max(1, S // 2), S + 1, (1,), generator=g)))
        ids[b, 0] = 101
        ids[b, 1:n - 1] = torch.randint(1000, vocab_size, (n - 2,), generator=g)
        ids[b, n - 1] = 102
        mask[b, :n] = 1
        if type_split:
            tt[b, n // 3:n] = 1
    return ids, mask, tt
