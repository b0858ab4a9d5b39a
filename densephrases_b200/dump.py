"""Phrase dump: documents -> the reference's HDF5 phrase dump (generate_phrase_vecs.py --do_dump, `dump_phrases` :45-147, with
embed_utils.py `write_phrases` / `write_filter` :40-382).

Pipeline per predict file:
1. context examples from the reference's JSON input (`_create_examples(context_only=True)`, squad_utils.py:811-865) and
   context-only features (`squad_convert_example_to_features(context_only=True)`, :143-300) with this repo's WordPieceTokenizer:
   the title takes at most 10 tokens, windows start doc_stride apart (transformers 2.9 `encode_plus` overflow), token types are 1;
2. the phrase tower (`Encoder.forward(return_phrase=True)`) per batch of per_gpu_eval_batch_size features;
3. on the GPU (csrc/dump.cu): the rows each document keeps (filter_start or filter_end above filter_threshold), their start2end
   re-indexed to the kept rows, int8 quantisation, compaction into one page-locked buffer -- only kept rows leave the device, 768 B
   each, instead of the reference's fp32 start and end vectors of every token;
4. on the host: each document's character offsets (`word2char_start` / `word2char_end`, get_metadata :84-105) and the file.

A document is the run of features from one with par_idx == 0 and span_idx == 0 to the next (write_phrases :266-285); documents
span forward batches, and the device step carries each open document's row and kept counts.  A document none of whose rows passes
the filter keeps its first row with filter_start > -999999 (filter_metadata :125-128).

The character offsets are pure-Python text alignment (two get_final_text calls per token, as in the reference) and run in this
process; at the gen-vecs shape they are most of a dump's time (DESIGN.md 4.6).

Limits: S <= 512 and max_answer_length <= 64.  The whole dump file is built in host memory (an existing file is read once and kept)
and rewritten by artifacts.write_hdf5 after each input file."""
import json
import logging
import os
import timeit

import numpy as np
import torch

from . import _lib as L
from . import artifacts
from .rc import final_text_span, tokens_to_string
from .tokenization import CLS, SEP

logger = logging.getLogger(__name__)

MAX_ANSWER_LENGTH = 64
MAX_TITLE_TOKENS = 10


# ---- examples and features ----------------------------------------------------------------------------------------------------------
def _is_whitespace(c):
    return c == " " or c == "\t" or c == "\r" or c == "\n" or ord(c) == 0x202F


def create_tokens(text):
    """SquadExample.create_tokens: whitespace-separated words (squad_utils.py:1096-1111)."""
    tokens, prev_ws = [], True
    for c in text or '':
        if _is_whitespace(c):
            prev_ws = True
        else:
            if prev_ws:
                tokens.append(c)
            else:
                tokens[-1] += c
            prev_ws = False
    return tokens


class ContextExample(object):
    def __init__(self, context_text, title, doc_idx, par_idx):
        self.context_text, self.title, self.doc_idx, self.par_idx = context_text, title, doc_idx, par_idx
        self.doc_tokens = create_tokens(context_text)
        self.title_tokens = create_tokens(title)


def read_examples(input_data):
    """The `data` list of a SQuAD-style JSON file -> context examples (_create_examples(context_only=True)): '\\xa0' becomes ' ',
    paragraphs with is_paragraph false are skipped, par_idx counts the kept paragraphs of a document."""
    examples = []
    for doc_idx, entry in enumerate(input_data):
        title = entry["title"]
        par_idx = 0
        for paragraph in entry["paragraphs"]:
            context_text = paragraph["context"].replace('\xa0', ' ')
            if type(title) == list:
                title = title[0]
            title = title.strip().replace('_', ' ')
            if 'is_paragraph' in paragraph and not paragraph['is_paragraph']:
                continue
            examples.append(ContextExample(context_text, title, doc_idx, par_idx))
            par_idx += 1
    return examples


class ContextFeature(object):
    def __init__(self, **kw):
        self.__dict__.update(kw)


def convert_examples_to_features(examples, tokenizer, max_seq_length, doc_stride, append_title):
    """Context-only features (squad_convert_examples_to_features(context_only=True)): one feature per window of the example's
    word pieces; unique ids from 1000000000, example_index counts only examples that have a feature (as the reference's does)."""
    features, unique_id, example_index = [], 1000000000, 0
    title_extra = 3 if append_title else 2                # [CLS] title [SEP] ... [SEP] / [CLS] ... [SEP]
    for ex in examples:
        title = [p for w in ex.title_tokens for p in tokenizer.tokenize(w)][:MAX_TITLE_TOKENS] if append_title else []
        tok_to_orig, doc = [], []
        for i, w in enumerate(ex.doc_tokens):
            for p in tokenizer.tokenize(w):
                tok_to_orig.append(i)
                doc.append(p)
        title_offset = len(title) + 2 if append_title else 1
        cap = max_seq_length - (len(title) + title_extra if append_title else title_extra)
        head = [CLS] + (title + [SEP] if append_title else [])
        made = []
        while len(made) * doc_stride < len(doc):
            lo = len(made) * doc_stride
            plen = min(len(doc) - lo, cap)
            tokens = head + doc[lo:lo + plen] + [SEP]
            ids = [tokenizer.vocab.get(t, tokenizer.unk_token_id) for t in tokens]
            tokens = [tokenizer.ids_to_tokens[i] for i in ids]
            pad = max_seq_length - len(ids)
            made.append(ContextFeature(
                input_ids=ids + [tokenizer.pad_token_id] * pad, attention_mask=[1] * len(ids) + [0] * pad,
                token_type_ids=[1] * max_seq_length, tokens=tokens,
                token_to_orig_map={title_offset + i: tok_to_orig[lo + i] for i in range(plen)}, paragraph_len=plen,
                title_offset=title_offset, span_idx=len(made), doc_idx=ex.doc_idx, par_idx=ex.par_idx))
            if len(doc) - lo <= cap:                        # encode_plus returned no overflowing tokens
                break
        if not made:
            continue
        for f in made:
            f.example_index, f.unique_id = example_index, unique_id
            unique_id += 1
        example_index += 1
        features.extend(made)
    return features


# ---- character offsets (get_metadata :84-105, get_final_text_ squad_metrics.py:354-371) ----------------------------------------
def _final_pos(example, feature, s, e, do_lower_case, tokenizer, word_off):
    ods, ode = feature.token_to_orig_map[s], feature.token_to_orig_map[e]
    tok_text = ' '.join(tokens_to_string(tokenizer, feature.tokens[s:e + 1]).strip().split())
    lo, hi = final_text_span(tok_text, ' '.join(example.doc_tokens[ods:ode + 1]), do_lower_case)
    return word_off[ods] + lo, word_off[ods] + hi


def document_offsets(examples, features, toffs, do_lower_case, tokenizer):
    """-> (context, word2char_start int32, word2char_end int32) of one document's features: positions in the paragraphs joined by
    ' [PAR] ', each paragraph appended when the next paragraph's first feature starts."""
    full_text, prev, w2s, w2e = '', None, [], []
    for feature, to in zip(features, toffs):
        example = examples[feature.example_index]
        if prev is not None and feature.span_idx == 0:
            full_text = full_text + ' '.join(prev.doc_tokens) + ' [PAR] '
        word_off = np.concatenate([[0], np.cumsum([len(w) + 1 for w in example.doc_tokens])]).tolist()
        n, base = len(feature.tokens), len(full_text)
        for i in range(to + 1, n - 1):
            w2s.append(base + _final_pos(example, feature, i, min(n - 2, i + 1), do_lower_case, tokenizer, word_off)[0])
            w2e.append(base + _final_pos(example, feature, max(to + 1, i - 1), i, do_lower_case, tokenizer, word_off)[1])
        prev = example
    return full_text + ' '.join(prev.doc_tokens), np.array(w2s, np.int32), np.array(w2e, np.int32)


def documents(examples, features):
    """write_phrases' grouping (:266-285): lists of consecutive feature indices, a new one at par_idx == 0 and span_idx == 0."""
    groups = []
    for i, f in enumerate(features):
        if groups and examples[f.example_index].par_idx == 0 and f.span_idx == 0:
            groups.append([i])
        elif groups:
            groups[-1].append(i)
        else:
            groups.append([i])
    return groups


def title_offsets(features, tokenizer, has_title):
    return [f.input_ids.index(tokenizer.sep_token_id) * int(has_title) for f in features]


# ---- device step ----------------------------------------------------------------------------------------------------------------
class DumpSelect(object):
    """The binding of dph_dump_select with a reusable page-locked output buffer."""

    def __init__(self, max_answer_length, filter_threshold, dense_offset, dense_scale):
        if not 1 <= int(max_answer_length) <= MAX_ANSWER_LENGTH:
            raise ValueError(f'max_answer_length {max_answer_length} outside 1..{MAX_ANSWER_LENGTH}')
        self.L, self.thr, self.offset, self.scale = int(max_answer_length), float(filter_threshold), float(dense_offset), float(dense_scale)
        self.buf = None
        self.d2h_bytes = 0
        self.device_ms = 0.0                 # CUDA events around the two kernels (their writes into the pinned buffer included)
        self.copy_s = 0.0                    # host copies out of the pinned buffer
        self._events = None

    def __call__(self, start, filt, feat, doc):
        """start fp32 [B,S,768] and filt fp32 [B,S,2] CUDA tensors; feat int32 [B,4] (row_lo, row_hi, document slot, document-level
        row of row_lo); doc int32 [n_doc,2] (rows kept before this batch, fallback still needed) -> dict of numpy arrays (copies):
        n_kept, doc_kept [n_doc], rows int8 [K,768], f2o int64 [K], start2end int32 [K,L], fb_f2o int64 [n_doc], fb_rows [n_doc,768]."""
        if start.dtype != torch.float32 or filt.dtype != torch.float32 or not start.is_cuda or not filt.is_cuda:
            raise ValueError('start and filter logits must be fp32 CUDA tensors')
        B, S = int(start.shape[0]), int(start.shape[1])
        if tuple(start.shape) != (B, S, 768) or tuple(filt.shape) != (B, S, 2):
            raise ValueError(f'start {tuple(start.shape)} / filter logits {tuple(filt.shape)} must be [B,S,768] / [B,S,2]')
        start, filt = start.contiguous(), filt.contiguous()
        feat = np.ascontiguousarray(feat, np.int32)
        doc = np.ascontiguousarray(doc, np.int32)
        if feat.shape != (B, 4) or doc.ndim != 2 or doc.shape[1] != 2:
            raise ValueError('feat must be [B,4] and doc [n_doc,2]')
        R, n_doc = int(np.maximum(feat[:, 1] - feat[:, 0], 0).sum()), int(doc.shape[0])
        offs = np.zeros(7, np.int64)
        need = int(L.lib().dph_dump_layout(R, n_doc, self.L, offs.ctypes.data))
        if need < 0:
            raise ValueError('bad dump layout arguments')
        if self.buf is None or self.buf.numel() < need:
            self.buf = torch.empty(max(need, 1 << 20), dtype=torch.uint8, pin_memory=True)
        dev = start.device
        stream = torch.cuda.current_stream(dev)
        if self._events is None:
            self._events = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        self._events[0].record(stream)
        L.check(L.lib().dph_dump_select(start.data_ptr(), filt.data_ptr(), B, S, feat.ctypes.data, n_doc, doc.ctypes.data, self.L,
                                        self.thr, self.offset, self.scale, self.buf.data_ptr(), self.buf.numel(), stream.cuda_stream))
        self._events[1].record(stream)
        self._events[1].synchronize()
        self.device_ms += self._events[0].elapsed_time(self._events[1])
        t0 = timeit.default_timer()
        raw = self.buf.numpy()
        at = lambda i, dt, n: raw[offs[i]:offs[i] + n * np.dtype(dt).itemsize].view(dt)      # noqa: E731
        K = int(at(0, np.int64, 1)[0])
        self.d2h_bytes += 8 + n_doc * 12 + K * (768 + 8 + 4 * self.L)
        out = dict(n_kept=K, doc_kept=at(1, np.int32, n_doc).copy(), fb_f2o=at(2, np.int64, n_doc).copy(),
                   rows=at(3, np.int8, K * 768).reshape(K, 768).copy(), f2o=at(4, np.int64, K).copy(),
                   start2end=at(5, np.int32, K * self.L).reshape(K, self.L).copy())
        fb = out['fb_f2o'] >= 0
        self.d2h_bytes += int(fb.sum()) * 768
        out['fb_rows'] = at(6, np.int8, n_doc * 768).reshape(n_doc, 768)[fb].copy() if fb.any() else np.zeros((0, 768), np.int8)
        out['fb_slot'] = np.cumsum(fb) - 1                   # fb_rows row of each document slot that got a fallback
        self.copy_s += timeit.default_timer() - t0
        return out


def filter_pairs(fs, fe):
    """(filter_start, filter_end) [B,S] views of Encoder's [B,S,2] filter output -> that [B,S,2] tensor (no copy when they are)."""
    B, S = fs.shape
    if fs.stride() == (2 * S, 2) and fe.stride() == (2 * S, 2) and fe.data_ptr() == fs.data_ptr() + 4:
        return fs.as_strided((B, S, 2), (2 * S, 2, 1))
    return torch.stack((fs, fe), -1).contiguous()


def phrase_outputs(model, features, batch_size):
    """-> per batch (first feature index, start fp32 [B,S,768], filt fp32 [B,S,2]) from model(..., return_phrase=True)."""
    for b0 in range(0, len(features), batch_size):
        fb = features[b0:b0 + batch_size]
        ids, mask, tt = (torch.tensor([getattr(f, k) for f in fb], dtype=torch.int64) for k in ('input_ids', 'attention_mask', 'token_type_ids'))
        with torch.no_grad():
            start, _, fs, fe = model(input_ids=ids, attention_mask=mask, token_type_ids=tt, return_phrase=True)
        yield b0, start, filter_pairs(fs, fe)


# ---- dumping ------------------------------------------------------------------------------------------------------------------------
class _Doc(object):
    def __init__(self, feats):
        self.feats = feats
        self.rows = 0                     # valid rows seen so far
        self.kept = 0
        self.parts = []                   # (rows int8, f2o, start2end) per batch
        self.fallback = None              # (row int8 [768], f2o)
        self.filters = []                 # filter-only mode: (filter_start, filter_end) per feature


def dump_documents(examples, features, outputs, tokenizer, max_answer_length, do_lower_case, filter_threshold, dense_offset,
                   dense_scale, has_title, filter_only=False, timings=None):
    """Features and their phrase outputs (phrase_outputs) -> {did: (group datasets dict, group attrs dict)} as write_phrases
    (or write_filter) fills them.  timings, when a dict, accumulates: 'forward' and 'select' (host seconds around the forward and
    the device step), 'select_device_ms' (CUDA events around the device step), 'copy' (host copies out of the pinned buffer),
    'offsets' (seconds), 'd2h_bytes'."""
    groups = documents(examples, features)
    group_of = np.empty(len(features), np.int64)
    for g, idxs in enumerate(groups):
        group_of[idxs] = g
    toffs = title_offsets(features, tokenizer, has_title)
    row_lo = np.array([to + 1 for to in toffs], np.int64)
    row_hi = np.array([len(f.tokens) - 1 for f in features], np.int64)
    docs = {}
    out = {}
    sel = None if filter_only else DumpSelect(max_answer_length, filter_threshold, dense_offset, dense_scale)
    tm = timings if timings is not None else {}

    def close(g):
        d = docs.pop(g)
        fidx = d.feats
        ex = examples[features[fidx[-1]].example_index]
        did = str(ex.doc_idx)
        if filter_only:
            fs = np.concatenate([x[0] for x in d.filters])
            fe = np.concatenate([x[1] for x in d.filters])
            out[did] = ({'filter_start': fs, 'filter_end': fe}, {'title': ex.title})
            return
        if d.kept:
            start = np.concatenate([p[0] for p in d.parts])
            f2o = np.concatenate([p[1] for p in d.parts])
            s2e = np.concatenate([p[2] for p in d.parts])
        elif d.fallback is not None:
            start, f2o = d.fallback[0][None], np.array([d.fallback[1]], np.int64)
            s2e = np.full((1, max_answer_length), -1, np.int32)
            s2e[0, 0] = 0
        else:
            start, f2o, s2e = np.zeros((0, 768), np.int8), np.zeros(0, np.int64), np.zeros((0, max_answer_length), np.int32)
        t0 = timeit.default_timer()
        fl = [features[i] for i in fidx]
        context, w2s, w2e = document_offsets(examples, fl, [toffs[i] for i in fidx], do_lower_case, tokenizer)
        tm['offsets'] = tm.get('offsets', 0.0) + timeit.default_timer() - t0
        lpp = np.array([max(0, int(row_hi[i] - row_lo[i])) for i in fidx], np.int64)
        out[did] = ({'start': start, 'len_per_para': lpp, 'start2end': s2e, 'word2char_start': w2s, 'word2char_end': w2e, 'f2o_start': f2o},
                    {'context': context, 'title': ex.title, 'offset': float(dense_offset), 'scale': float(dense_scale)})

    it = iter(outputs)
    while True:
        t0 = timeit.default_timer()
        try:
            b0, start, filt = next(it)
        except StopIteration:
            break
        B = int(start.shape[0])
        gs = group_of[b0:b0 + B]
        if filter_only:
            f = filt.cpu().numpy()
            tm['forward'] = tm.get('forward', 0.0) + timeit.default_timer() - t0
            for k in range(B):
                i, g = b0 + k, int(gs[k])
                if g not in docs:
                    docs[g] = _Doc(groups[g])
                docs[g].filters.append((f[k, row_lo[i]:row_hi[i], 0], f[k, row_lo[i]:row_hi[i], 1]))
        else:
            torch.cuda.current_stream(start.device).synchronize()
            t1 = timeit.default_timer()
            tm['forward'] = tm.get('forward', 0.0) + t1 - t0
            g0 = int(gs[0])
            n_doc = int(gs[-1]) - g0 + 1
            feat = np.zeros((B, 4), np.int32)
            doc = np.zeros((n_doc, 2), np.int32)
            for s in range(n_doc):
                g = g0 + s
                if g not in docs:
                    docs[g] = _Doc(groups[g])
                doc[s] = (docs[g].kept, int(docs[g].kept == 0 and docs[g].fallback is None))
            rows = {g: docs[g].rows for g in range(g0, g0 + n_doc)}
            for k in range(B):
                i, g = b0 + k, int(gs[k])
                n = max(0, int(row_hi[i] - row_lo[i]))
                feat[k] = (row_lo[i], row_lo[i] + n, g - g0, rows[g])
                rows[g] += n
            r = sel(start, filt, feat, doc)
            tm['select'] = tm.get('select', 0.0) + timeit.default_timer() - t1
            at = 0
            for s in range(n_doc):
                d, n = docs[g0 + s], int(r['doc_kept'][s])
                if n:
                    d.parts.append((r['rows'][at:at + n], r['f2o'][at:at + n], r['start2end'][at:at + n]))
                at += n
                d.kept += n
                d.rows = rows[g0 + s]
                if doc[s, 1] and r['fb_f2o'][s] >= 0:
                    d.fallback = (r['fb_rows'][r['fb_slot'][s]], int(r['fb_f2o'][s]))
        for g in sorted(docs):                          # documents whose last feature has been seen
            if groups[g][-1] < b0 + B:
                close(g)
    for g in sorted(docs):
        close(g)
    if sel is not None:
        tm['d2h_bytes'] = tm.get('d2h_bytes', 0) + sel.d2h_bytes
        tm['select_device_ms'] = tm.get('select_device_ms', 0.0) + sel.device_ms
        tm['copy'] = tm.get('copy', 0.0) + sel.copy_s
    return out


def read_dump(path):
    """An existing dump file -> {did: (datasets, attrs)}."""
    h = artifacts.open_hdf5(path)
    out = {}
    for did, addr in h.children(h.root_addr).items():
        members = h.children(addr)
        out[did] = ({k: h.dataset(a) for k, a in members.items()}, h.attributes(addr))
    return out


def write_dump(path, groups, existing=None):
    """{did: (datasets, attrs)} -> the HDF5 file, merged into an existing one (its other groups kept, re-dumped ones replaced).
    existing: the file's groups when the caller already holds them (read_dump), else the file is read.  -> the merged groups."""
    merged = existing if existing is not None else (read_dump(path) if os.path.exists(path) else {})
    merged.update(groups)
    artifacts.write_hdf5(path, {did: g[0] for did, g in merged.items()}, attrs={did: g[1] for did, g in merged.items()})
    return merged


def dump_phrases(args, model, tokenizer, filter_only=False):
    """generate_phrase_vecs.py's dump_phrases: args.predict_file (a JSON file under args.data_dir, or `<dir>/<start>:<end>` for the
    files <dir>/0000, ... with doc_idx += 1000 * file) -> args.output_dir/dump/phrase/<name>.hdf5 (dump/filter with filter_only).
    Each file is built in host memory before it is written."""
    output_path = 'dump/phrase' if not filter_only else 'dump/filter'
    os.makedirs(os.path.join(args.output_dir, output_path), exist_ok=True)
    if ':' not in args.predict_file:
        predict_files, offsets = [args.predict_file], [0]
        output_dump_file = os.path.join(args.output_dir, f"{output_path}/{os.path.splitext(os.path.basename(args.predict_file))[0]}.hdf5")
    else:
        dirname, basename = os.path.dirname(args.predict_file), os.path.basename(args.predict_file)
        start, end = list(map(int, basename.split(':')))
        output_dump_file = os.path.join(args.output_dir, f"{output_path}/{start}-{end}.hdf5")
        if os.path.exists(output_dump_file):
            h = artifacts.open_hdf5(output_dump_file)
            start = int(max(map(int, h.children(h.root_addr))) / 1000)
            logger.info('%s exists; starting from %d' % (output_dump_file, start))
        names = [str(i).zfill(4) for i in range(start, end)]
        predict_files = [os.path.join(dirname, name) for name in names]
        offsets = [int(each) * 1000 for each in names]
    batch_size = args.per_gpu_eval_batch_size * max(1, getattr(args, 'n_gpu', 1))
    merged = read_dump(output_dump_file) if os.path.exists(output_dump_file) else {}     # read once, kept across input files
    for offset, predict_file in zip(offsets, predict_files):
        args.predict_file = predict_file
        t0 = timeit.default_timer()
        with open(os.path.join(getattr(args, 'data_dir', None) or '', predict_file), encoding='utf-8') as f:
            examples = read_examples(json.load(f)['data'])
        for ex in examples:
            ex.doc_idx += offset
        features = convert_examples_to_features(examples, tokenizer, args.max_seq_length, args.doc_stride, args.append_title)
        logger.info(f'***** Dumping phrases from {predict_file}: {len(features)} features, batch size {batch_size} *****')
        groups = dump_documents(examples, features, phrase_outputs(model, features, batch_size), tokenizer,
                                None if filter_only else args.max_answer_length, args.do_lower_case, args.filter_threshold,
                                args.dense_offset, args.dense_scale, args.append_title, filter_only=filter_only)
        merged = write_dump(output_dump_file, groups, merged)
        logger.info('Dumped %d documents in %.1f s', len(groups), timeit.default_timer() - t0)
    return output_dump_file


def main(argv=None):
    from .options import Options
    from .runtime import load_encoder
    options = Options()
    options.add_model_options()
    options.add_data_options()
    options.add_rc_options()
    args = options.parse(argv)
    logging.basicConfig(format='%(asctime)s - %(levelname)s - %(name)s -   %(message)s', level=logging.INFO)
    if args.do_dump:
        assert args.load_dir
        args.n_gpu = 1
        model, tokenizer, _ = load_encoder(torch.device('cuda', 0), args, phrase_only=True)
        dump_phrases(args, model, tokenizer, filter_only=args.filter_only)


if __name__ == '__main__':
    main()
