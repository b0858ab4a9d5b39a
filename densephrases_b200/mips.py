"""MIPS -- the phrase-index runtime of DensePhrases on the H100-native IVF-PQ index.

API mirror of the reference class `MIPS` (reference densephrases/index.py:23-482): same constructor and
`search(...)` signature, same result dictionaries, same tolerance of missing ids / out-of-range labels, so the
reference's callers (eval_phrase_retrieval.evaluate :57-77, DensePhrases.search model.py:82-87,
train_query.get_top_phrases :187-201) work on top of it.  The internals are written for batches, not items:

  reference                                            here
  ---------------------------------------------------  -------------------------------------------------------------
  faiss index.search(x, k)            (index.py:200)   IvfPqIndex.search -> libdph_b200 CUDA path
  2*B*k*L python reconst_fn(id) calls (:282-300)       one reconstruct_batch([2*B*k*L]) call (missing id -> zero row)
  per-hit python valid_phrase closures (:305-331)      one vectorised validity matrix per direction over a packed f2o table
  per-label dict lookups in get_idxs   (:124-141)      grouped fancy indexing
  spaCy sentencizer                    (:65-66,178)    rule-based stand-in (spaCy is not in this image)

On-disk artefacts: `MIPS(...)` takes the reference's paths.  It prefers this repo's containers when they sit next to them
(`index.dph.npz`, `idx2id.npz`, `meta_dph.pkl`) and otherwise parses the reference's own files -- `index.faiss` (+ the
`.ivfdata` payload of a merged index), `idx2id.hdf5`, `meta_compressed.pkl` with its blosc blobs -- with the pure-Python
readers of densephrases_b200/artifacts.py (no faiss / h5py / blosc; see that module's STATUS note).
`MIPS.from_components` wraps in-memory objects.  Without in-RAM metadata the phrase stage falls back to the phrase dump
(phrase_dump.py: metadata and int8 token vectors per document, index.py:246-273) -- functional, not accelerated.
"""
import json
import logging
import os
import pickle
import re
import string
from time import time

import numpy as np
import torch

from .artifacts import decode_meta_field

logger = logging.getLogger(__name__)
_PUNCT = set(string.punctuation)
_ARTICLES = re.compile(r'\b(a|an|the)\b')
_MASKED = -1e9        # additive mask for invalid phrase ends/starts (index.py:328,357)
_DROPPED = -1e8       # score of dummy / deduplicated results (index.py:404,441)
_KEEP_ABOVE = -1e5    # results below this are filtered out (index.py:419,446)


def normalize_answer(text):
    """SQuAD answer normalisation as used by agg_strat 'opt4' (index.py:435 -> eval_utils.normalize_answer)."""
    text = ''.join(ch for ch in text.lower() if ch not in _PUNCT)
    return ' '.join(_ARTICLES.sub(' ', text).split())


class RuleSentencizer(object):
    """[(sentence_text, first_char_offset)] -- what `[(X.text, X[0].idx) for X in nlp(text).sents]` gives the reference
    (index.py:179).  A sentence ends after a run of . ! ? (optionally followed by closing quotes/brackets) + whitespace."""
    _boundary = re.compile(r'[.!?]+["\')\]]*\s+')

    def __call__(self, text):
        cuts = [0] + [m.end() for m in self._boundary.finditer(text)] + [len(text)]
        out = []
        for a, b in zip(cuts[:-1], cuts[1:]):
            piece = text[a:b]
            if piece.strip():
                out.append((piece.strip(), a + len(piece) - len(piece.lstrip())))
        return out or [(text, 0)]


class _PackedDocs(object):
    """f2o_start of all documents touched by one batch, packed into one array for vectorised validity checks."""

    def __init__(self, metas):
        self.slot = {d: i for i, d in enumerate(metas)}
        lens = np.array([len(metas[d]['f2o_start']) for d in metas] + [0], dtype=np.int64)
        self.base = np.concatenate([[0], np.cumsum(lens[:-1])])
        self.len = lens
        self.f2o = np.concatenate([np.asarray(metas[d]['f2o_start'], dtype=np.int64) for d in metas] + [np.zeros(1, np.int64)])

    def windows(self, doc, first, last, max_len):
        """doc [Q]; first/last [Q,L] candidate (start word, end word) pairs -> bool [Q,L] valid_phrase (index.py:305-321)."""
        slot = np.array([self.slot.get(d, len(self.len) - 1) for d in doc.tolist()], dtype=np.int64)
        n, b = self.len[slot][:, None], self.base[slot][:, None]
        ok = (doc[:, None] >= 0) & (first >= 0) & (first < n) & (last >= 0) & (last < n)
        span = self.f2o[b + np.clip(last, 0, np.maximum(n - 1, 0))] - self.f2o[b + np.clip(first, 0, np.maximum(n - 1, 0))]
        return ok & (span >= 0) & (span <= max_len)


def distributed_context():
    """(rank, world, local_rank) of a one-process-per-GPU job (torchrun exports RANK / WORLD_SIZE / LOCAL_RANK); the NCCL process
    group is created on first use so that the reference's drivers, which know nothing about ranks, can simply be launched with
    `python -m torch.distributed.run --nproc-per-node N eval_phrase_retrieval.py ...` (SURVEY.md 8b: all ranks enter search together)."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world <= 1:
        return 0, 1, torch.cuda.current_device() if torch.cuda.is_available() else 0
    import torch.distributed as dist
    rank, local_rank = int(os.environ.get('RANK', '0')), int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local_rank)
    if not dist.is_initialized():
        dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
    return rank, world, local_rank


class MIPS(object):
    def __init__(self, phrase_dump_dir, index_path, idx2id_path, cuda=False, logging_level=logging.INFO):
        from .sharded import ShardedIvfPq
        from . import artifacts, synthetic_dump
        rank, world, dev = distributed_context()
        index_dir = os.path.dirname(index_path)
        container, spec = os.path.join(index_dir, 'index.dph.npz'), os.path.join(index_dir, 'index.dph.json')
        if os.path.exists(spec):                                         # synthetic index generated on the GPU(s) (synthetic_dump.py)
            sp = json.load(open(spec))['synthetic_index']
            logger.info(f'Generating the synthetic index of {spec}: {sp}')
            rng = np.random.default_rng(sp['opq_seed'])
            A = np.linalg.qr(rng.standard_normal((768, 768)))[0].astype(np.float32)
            index = ShardedIvfPq(sp['nlist'], rank=rank, world=world, device=dev)
            index.build_synthetic(A, synthetic_dump.uniform_list_lengths(sp['N'], sp['nlist']), sp['seed'])
        else:
            if os.path.exists(container):
                logger.info(f'Reading {container}')
                z = np.load(container)
                parts = {k: z[k] for k in z.files}
            elif os.path.exists(index_path):
                logger.info(f'Reading {index_path} (FAISS container, parsed natively)')
                parts = artifacts.read_faiss_index(index_path, ondisk_same_dir=True)      # faiss.IO_FLAG_ONDISK_SAME_DIR, index.py:30
                if not parts['by_residual'] or parts['metric'] != 0 or parts['quantizer_metric'] != 0:
                    raise RuntimeError('only the inner-product, by-residual IVF-PQ index of build_phrase_index.py:113-116 is supported')
            else:
                raise RuntimeError(f'neither {container}, {spec} nor {index_path} found')
            index = ShardedIvfPq.from_arrays(parts['A'], parts['centroids'], parts['pq'], parts['list_len'], parts['codes'], parts.get('ids'),
                                             rank=rank, world=world, device=dev)
        dump_root = phrase_dump_dir[:phrase_dump_dir.index('/phrase')] if '/phrase' in phrase_dump_dir else phrase_dump_dir
        doc_groups = None
        if 'PQ' in index_path:                                          # in-RAM metadata only with PQ indexes (index.py:69-74)
            if os.path.exists(os.path.join(dump_root, 'meta_dph.json')):
                sp = json.load(open(os.path.join(dump_root, 'meta_dph.json')))['synthetic_meta']
                doc_groups = synthetic_dump.LazyDocs(sp['tokens_per_doc'], sp['seed'])
            else:
                for name in ('meta_dph.pkl', 'meta_compressed.pkl'):
                    if os.path.exists(os.path.join(dump_root, name)):
                        doc_groups = artifacts.read_meta(os.path.join(dump_root, name))
                        break
        self.phrase_dump_dir = phrase_dump_dir
        self._attach(index, self.load_idx_f(idx2id_path), doc_groups, index_path, cuda, logging_level)
        if doc_groups is None:                     # index.py:75-76: "Will read metadata directly from hdf5 files"
            from .phrase_dump import PhraseDump
            logger.info('Will read metadata and token vectors directly from the phrase dump (not accelerated)')
            self.phrase_dump = PhraseDump(phrase_dump_dir)

    @classmethod
    def from_components(cls, index, idx_f, doc_groups, index_path='synthetic_PQ', cuda=True, logging_level=logging.INFO, phrase_dump=None):
        """index: IvfPqIndex-like (search / reconstruct_batch / opq_matrix / ntotal / d / nprobe);
        idx_f: {str(offset): {'doc','word'}} (idx2id.hdf5 layout, build_phrase_index.py:268-276);
        doc_groups: {str(doc_idx): {'word2char_start','word2char_end','f2o_start','context','title'}} (meta_compressed.pkl)."""
        self = cls.__new__(cls)
        self.phrase_dump_dir = None
        self._attach(index, idx_f, doc_groups, index_path, cuda, logging_level)
        self.phrase_dump = phrase_dump            # object with .get(doc_idx) -> record (phrase_dump.py); used when doc_groups is None
        return self

    def _attach(self, index, idx_f, doc_groups, index_path, cuda, logging_level):
        logger.setLevel(logging_level)
        self.index, self.idx_f, self.doc_groups = index, idx_f, doc_groups
        self.reconst_batch = index.reconstruct_batch                   # batched form of reconst_fn (index.py:31)
        self.is_pq = 'PQ' in index_path
        self.max_idx = 1e9 if self.is_pq else 1e8                      # label = offset + row (index.py:33)
        self.cuda = cuda
        if cuda and not torch.cuda.is_available():
            raise AssertionError(f'Cuda availability {torch.cuda.is_available()}')
        self.device = torch.device('cuda' if cuda else 'cpu')
        self.R = torch.from_numpy(np.ascontiguousarray(index.opq_matrix(), dtype=np.float32)).to(self.device)   # index.py:32,57
        self.index.nprobe = 256                                        # fixed at load time in the reference (index.py:53,62)
        self.num_docs_list = []
        self.stage_seconds = {'mips': 0.0, 'get_idxs': 0.0, 'phrase_vectors': 0.0, 'phrase_select': 0.0, 'metadata': 0.0, 'batches': 0}
        self.sentencizer = RuleSentencizer()
        self.offset = self.scale = None
        self.phrase_dump = None
        logger.info(f'index ntotal: {self.index.ntotal} | PQ: {self.is_pq} | nprobe: {self.index.nprobe}')

    # ---- loading helpers -------------------------------------------------------------------------------
    def load_idx_f(self, idx2id_path):
        """{offset_key: {'doc': int32[], 'word': int32[]}} like index.py:78-88; read from `idx2id.npz` (members '<offset>/<type>')
        when it exists next to idx2id_path, else from the HDF5 file itself."""
        npz = os.path.splitext(idx2id_path)[0] + '.npz'
        spec = os.path.splitext(idx2id_path)[0] + '.dph.json'
        if os.path.exists(spec):
            from . import synthetic_dump
            sp = json.load(open(spec))['synthetic_idx2id']
            return synthetic_dump.synthetic_idx2id(sp['ntotal'], sp['tokens_per_doc'])
        if not os.path.exists(npz):
            from . import artifacts
            return artifacts.read_idx2id(idx2id_path)
        z = np.load(npz)
        table = {}
        for member in z.files:
            key, kind = member.split('/')
            table.setdefault(key, {})[kind] = z[member]
        return table

    def decompress_meta(self, doc_idx):
        """Per-document metadata record (index.py:106-122).  Array fields may be stored raw, zlib-compressed (this repo's
        converter) or as the reference's blosc frames (compress_metadata.py:32-53), the latter two with a 'dtypes' entry."""
        rec = self.doc_groups[doc_idx]
        dt = rec.get('dtypes', {})

        def field(name):
            v = rec[name]
            return decode_meta_field(v, dt[name]) if isinstance(v, (bytes, bytearray)) else np.asarray(v)

        ctx = rec['context']
        if isinstance(ctx, (bytes, bytearray)):
            ctx = decode_meta_field(ctx).decode('utf-8')
        return {'word2char_start': field('word2char_start'), 'word2char_end': field('word2char_end'), 'f2o_start': field('f2o_start'),
                'context': ctx, 'title': rec['title'], 'offset': -2, 'scale': 20}

    # ---- dense stage -------------------------------------------------------------------------------------
    def get_idxs(self, I):
        """labels [.,k] -> (doc_idx, word_idx) through idx2id; labels outside [0, ntotal) are clipped after a log line
        (index.py:128-133: that is how the reference survives the -1 padding of short result lists)."""
        I = np.asarray(I)
        if ((I < 0) | (I >= self.index.ntotal)).any():
            logger.info('index out of range!')
            I = np.clip(I, 0, self.index.ntotal - 1)
        step = int(self.max_idx)
        group = (I / self.max_idx).astype(np.int64) * step
        row = I % step
        doc = np.empty(I.shape, dtype=np.int64)
        word = np.empty(I.shape, dtype=np.int64)
        for g in np.unique(group):
            sel = group == g
            doc[sel] = self.idx_f[str(g)]['doc'][row[sel]]
            word[sel] = self.idx_f[str(g)]['word'][row[sel]]
        return doc, word

    def search_dense(self, query, q_texts, nprobe=256, top_k=10):
        """Start and end halves of `query [B, 2d]` are stacked into one [2B, d] search (index.py:195-202).
        `nprobe` is accepted and ignored, like the reference (its assignment is commented out at index.py:191)."""
        B = query.shape[0]
        tic = time()
        if isinstance(query, torch.Tensor) and query.is_cuda and hasattr(self.index, 'search_device'):
            # device-resident queries (DensePhrases.search hands over the encoder's output): no host round trip before the index
            d = query.shape[1] // 2
            x = torch.cat([query[:, :d], query[:, d:]], 0).float().contiguous()
            Dd, Id = self.index.search_device(x, top_k)
            scores, labels = Dd.cpu().numpy(), Id.cpu().numpy()
        else:
            if isinstance(query, torch.Tensor):
                query = query.detach().cpu().numpy()
            halves = np.split(query.astype(np.float32), 2, axis=1)
            scores, labels = self.index.search(np.concatenate(halves, axis=0), top_k)
        self.stage_seconds['mips'] += time() - tic
        self.stage_seconds['batches'] += 1
        logger.debug(f'1) {time()-tic:.3f}s: MIPS')
        tic = time()
        s_doc, s_word = self.get_idxs(labels[:B])
        e_doc, e_word = self.get_idxs(labels[B:])
        self.num_docs_list.append(sum(len(set(a.tolist()) | set(b.tolist())) for a, b in zip(s_doc, e_doc)) / B)
        self.stage_seconds['get_idxs'] += time() - tic
        logger.debug(f'2) {time()-tic:.3f}s: get index')
        return s_doc, s_word, labels[:B], e_doc, e_word, labels[B:], scores[:B], scores[B:]

    # ---- phrase stage ------------------------------------------------------------------------------------
    def _unrotated_scores(self, window_vecs, qvec):
        """window_vecs [Q,L,d] (rotated space) -> un-rotate with R (index.py:340,365) and dot with the query [Q,d]."""
        with torch.no_grad():
            w = torch.from_numpy(window_vecs).to(self.device).matmul(self.R)
            q = torch.from_numpy(np.ascontiguousarray(qvec, dtype=np.float32)).to(self.device)
            return (q.unsqueeze(1) * w).sum(2).cpu().numpy(), w.cpu().numpy()

    def _windows_from_dump(self, docs, s_doc, s_word, e_doc, e_word, L):
        """The phrase-dump branch of the reference (index.py:246-273,330-336,356-361): metadata straight from the dump's document
        groups; for a start hit the int8 rows [start, min(start + L, T)) of the document's `start` dataset, left-aligned in an L-row
        window, for an end hit the rows [max(0, end - L + 1), end], right-aligned; filled rows are dequantised x / 20 - 2, padding
        rows stay 0.  Also returns the RAW first / last rows: the reference hands those, not the dequantised ones, to the
        `return_idxs` vectors (index.py:381-389)."""
        recs = {d: self.phrase_dump.get(d) for d in docs}
        meta = {d: {'word2char_start': np.asarray(r['word2char_start']), 'word2char_end': np.asarray(r['word2char_end']),
                    'f2o_start': np.asarray(r['f2o_start']), 'context': r['context'], 'title': r['title'], 'offset': -2, 'scale': 20}
                for d, r in recs.items()}
        H, dim = len(s_doc), self.index.d
        raw_f, raw_b = np.zeros((H, L, dim), dtype=np.float32), np.zeros((H, L, dim), dtype=np.float32)
        fwd, bwd = np.zeros((H, L, dim), dtype=np.float32), np.zeros((H, L, dim), dtype=np.float32)

        def dequant(rows):                                   # int8_to_float(num, offset=-2, factor=20) = num / factor + offset
            return np.asarray(rows).astype(np.float64) / 20.0 + (-2.0)
        for h in range(H):
            if s_doc[h] in recs:
                vec = recs[s_doc[h]]['start']
                a = int(s_word[h])
                rows = np.asarray(vec[a:min(a + L, len(vec))]) if a >= 0 else np.zeros((0, dim))
                n = len(rows)
                if n:
                    raw_f[h, :n], fwd[h, :n] = rows, dequant(rows)
            if e_doc[h] in recs:
                vec = recs[e_doc[h]]['start']
                b = int(e_word[h])
                rows = np.asarray(vec[max(0, b - L + 1):b + 1]) if b >= 0 else np.zeros((0, dim))
                n = len(rows)
                if n:
                    raw_b[h, L - n:], bwd[h, L - n:] = rows, dequant(rows)
        return meta, fwd, bwd, raw_f[:, 0], raw_b[:, -1]

    def search_phrase(self, query, start_doc_idxs, start_idxs, orig_start_idxs, end_doc_idxs, end_idxs, orig_end_idxs,
                      start_scores, end_scores, top_k=10, max_answer_length=10, return_idxs=False, return_sent=False):
        """For every start hit pick the best end within L tokens and vice versa (index.py:220-422).  Token vectors come from the
        index (`reconstruct`, PQ + in-RAM metadata: the accelerated branch) or -- when there is no `meta_compressed.pkl` -- from the
        int8 `start` rows of the phrase dump together with the dump's own metadata (index.py:246-273; functional, not accelerated)."""
        from_dump = self.doc_groups is None or orig_start_idxs is None
        if from_dump and self.phrase_dump is None:
            raise NotImplementedError('no in-RAM metadata (meta_compressed.pkl / meta_dph.pkl) and no phrase dump to read token vectors '
                                      'and metadata from (index.py:246-273)')
        L, B = max_answer_length, query.shape[0]
        q_rep = np.repeat(query, top_k, axis=0)                         # row h = hit h of query h // top_k
        q_start, q_end = np.split(q_rep, 2, axis=1)
        owner = np.repeat(np.arange(B), 2 * top_k)
        s_doc, s_word, s_sc = (np.reshape(a, [-1]) for a in (start_doc_idxs, start_idxs, start_scores))
        e_doc, e_word, e_sc = (np.reshape(a, [-1]) for a in (end_doc_idxs, end_idxs, end_scores))
        assert len(s_doc) == len(s_word) == len(e_word) == len(s_sc)
        H = len(s_doc)

        tic = time()
        docs = [d for d in dict.fromkeys(s_doc.tolist() + e_doc.tolist()) if d >= 0]
        span = np.arange(L, dtype=np.int64)
        if from_dump:
            meta, fwd, bwd, fwd_first, bwd_last = self._windows_from_dump(docs, s_doc, s_word, e_doc, e_word, L)
            fused = False
        else:
            meta = {d: self.decompress_meta(str(d)) for d in docs}
            s_lab, e_lab = np.reshape(orig_start_idxs, [-1]), np.reshape(orig_end_idxs, [-1])
            fwd_labels = s_lab.astype(np.int64)[:, None] + span              # [start, start+L)        (index.py:284)
            bwd_labels = e_lab.astype(np.int64)[:, None] - (L - 1) + span    # (end-L, end]            (index.py:294)
            fused = (not return_idxs) and hasattr(self.index, 'window_scores')
        packed = _PackedDocs(meta)
        if from_dump:
            pass
        elif fused:   # one CUDA call per direction: reconstruct + un-rotate + dot fused (libdph_b200: dph_index_window_scores)
            end_sc = self.index.window_scores(q_end, fwd_labels[:, 0], L)
            start_sc = self.index.window_scores(q_start, bwd_labels[:, 0], L)
        else:
            vecs, _ = self.reconst_batch(np.concatenate([fwd_labels.ravel(), bwd_labels.ravel()]))   # missing label -> zeros
            vecs = np.asarray(vecs, dtype=np.float32)
            fwd, bwd = vecs[:H * L].reshape(H, L, -1), vecs[H * L:].reshape(H, L, -1)
            fwd_first, bwd_last = fwd[:, 0], bwd[:, -1]
        self.stage_seconds['phrase_vectors'] += time() - tic
        logger.debug(f'1) {time()-tic:.3f}s: reconstruct vecs')

        tic = time()
        cand_end = s_word[:, None] + span                                # end word candidates for each start hit
        ok_end = packed.windows(s_doc, np.broadcast_to(s_word[:, None], cand_end.shape), cand_end, L)
        if not fused:
            end_sc, fwd_unrot = self._unrotated_scores(fwd, q_end)
        score_se = s_sc[:, None] + end_sc + np.where(ok_end, 0.0, _MASKED)
        pick_e = score_se.argmax(1)
        best_end = np.where(ok_end, cand_end, -1)[np.arange(H), pick_e]
        self.stage_seconds['phrase_select'] += time() - tic
        logger.debug(f'2) {time()-tic:.3f}s: find end')

        tic = time()
        cand_start = e_word[:, None] - (L - 1) + span                    # start word candidates for each end hit
        ok_start = packed.windows(e_doc, cand_start, np.broadcast_to(e_word[:, None], cand_start.shape), L)
        if not fused:
            start_sc, bwd_unrot = self._unrotated_scores(bwd, q_start)
        score_es = start_sc + e_sc[:, None] + np.where(ok_start, 0.0, _MASKED)
        pick_s = score_es.argmax(1)
        best_start = np.where(ok_start, cand_start, -1)[np.arange(H), pick_s]
        self.stage_seconds['phrase_select'] += time() - tic
        logger.debug(f'3) {time()-tic:.3f}s: find start')

        # interleave (start-anchored, end-anchored) results per hit (index.py:375-378)
        tic = time()
        doc_of = np.stack([s_doc, e_doc], 1).ravel()
        first = np.stack([s_word, best_start], 1).ravel()
        last = np.stack([best_end, e_word], 1).ravel()
        score = np.stack([score_se.max(1), score_es.max(1)], 1).ravel()
        if return_idxs:   # un-rotated start/end vectors for query-side fine-tuning (index.py:381-389): R is applied once more
            R = self.R.cpu().numpy()
            svec = np.stack([fwd_first, bwd_unrot[np.arange(H), pick_s]], 1).reshape(2 * H, -1).dot(R)
            evec = np.stack([fwd_unrot[np.arange(H), pick_e], bwd_last], 1).reshape(2 * H, -1).dot(R)

        results = [[] for _ in range(B)]
        for h, (d, a, b, sc) in enumerate(zip(doc_of.tolist(), first.tolist(), last.tolist(), score.tolist())):
            if d < 0:
                rec = {'score': _DROPPED, 'context': 'dummy', 'start_pos': 0, 'end_pos': 0, 'title': ['']}
            else:
                m = meta[d]
                w2c_s, w2c_e, f2o = m['word2char_start'], m['word2char_end'], m['f2o_start']
                c0 = w2c_s[f2o[a]].item()
                c1 = w2c_e[f2o[b]].item() if (len(w2c_e) > 0 and b >= 0) else c0 + 1
                rec = {'context': m['context'], 'title': [m['title']], 'doc_idx': d, 'start_pos': c0, 'end_pos': c1,
                       'start_idx': a, 'end_idx': b, 'score': sc,
                       'start_vec': svec[h] if return_idxs else None, 'end_vec': evec[h] if return_idxs else None}
            rec['answer'] = rec['context'][rec['start_pos']:rec['end_pos']]
            rec = self.adjust(rec)
            if return_sent:
                rec = self.adjust_sent(rec)
            results[owner[h]].append(rec)
        results = [[r for r in sorted(rs, key=lambda r: -r['score']) if r['score'] > _KEEP_ABOVE] for rs in results]
        self.stage_seconds['metadata'] += time() - tic
        logger.debug(f'4) {time()-tic:.3f}s: get metadata')
        return results

    def adjust(self, each, delimiter=' [PAR] '):
        """Crop the document context to the paragraph holding the answer (index.py:167-176)."""
        ctx = each['context']
        lo = ctx.rfind(delimiter, 0, each['start_pos'])
        lo = 0 if lo < 0 else lo + len(delimiter)
        hi = ctx.find(delimiter, each['end_pos'])
        hi = len(ctx) if hi < 0 else hi
        if delimiter == '. ':
            hi += 1
        each['context'] = ctx[lo:hi]
        each['start_pos'] -= lo
        each['end_pos'] -= lo
        return each

    def adjust_sent(self, each):
        """Crop the context to the sentence(s) covering the answer (index.py:178-187)."""
        sents = self.sentencizer(each['context'])
        begins = np.array([b for _, b in sents])
        a = max(int((begins <= each['start_pos']).sum()) - 1, 0)
        b = max(int((begins <= each['end_pos'] - 1).sum()) - 1, 0)
        a, b = min(a, b), max(a, b)
        each['context'] = ' '.join(s for s, _ in sents[a:b + 1])
        each['start_pos'] -= sents[a][1]
        each['end_pos'] -= sents[a][1]
        return each

    def aggregate_results(self, results, top_k=10, q_text=None, agg_strat='opt1'):
        """Deduplicate one query's results: later duplicates get score -1e8 and are filtered (index.py:424-448)."""
        keyfn = {'opt1': lambda r: f'{r["title"]}_{r["start_pos"]}_{r["end_pos"]}',      # phrase retrieval
                 'opt2': lambda r: f'{r["context"]}',                                   # sentence / paragraph retrieval
                 'opt3': lambda r: f'{r["title"]}',                                     # document retrieval
                 'opt4': lambda r: f'{normalize_answer(r["answer"])}'}.get(agg_strat)  # answer-level merge (KILT)
        if keyfn is None:
            raise NotImplementedError('wrong aggregation strategy')
        seen = {}
        for pos, r in enumerate(results):
            key = keyfn(r)
            if key not in seen:
                seen[key] = pos
                continue
            r['score'] = _DROPPED
            keeper = results[seen[key]]
            if agg_strat == 'opt4' and r['title'][0] not in keeper['title']:
                keeper['title'] += r['title']
        return [r for r in sorted(results, key=lambda r: -r['score']) if r['score'] > _KEEP_ABOVE]

    def search(self, query, q_texts=None,
               nprobe=256, top_k=10,
               aggregate=False, return_idxs=False,
               max_answer_length=10, agg_strat='opt1', return_sent=False):
        """query [B, 2*768] (start || end) -> list[B] of result dicts sorted by score (index.py:450-482)."""
        tic = time()
        dense = self.search_dense(query, q_texts=q_texts, nprobe=nprobe, top_k=top_k)
        s_doc, s_word, s_lab, e_doc, e_word, e_lab, s_sc, e_sc = dense
        if isinstance(query, torch.Tensor):          # the phrase stage and the result dicts work on host arrays
            query = query.detach().cpu().numpy()
        logger.debug(f'Top-{top_k} MIPS: {time()-tic:.3f}s')
        tic = time()
        outs = self.search_phrase(query, s_doc, s_word, s_lab, e_doc, e_word, e_lab, s_sc, e_sc, top_k=top_k,
                                  max_answer_length=max_answer_length, return_idxs=return_idxs, return_sent=return_sent)
        logger.debug(f'Top-{top_k} phrase search: {time()-tic:.3f}s')
        if aggregate:
            outs = [self.aggregate_results(rs, top_k, qt, agg_strat) for rs, qt in zip(outs, q_texts)]
        if s_doc.shape[1] != top_k:
            logger.info(f'Warning.. {s_doc.shape[1]} only retrieved')
        return outs


MIPSIndex = MIPS   # the name BASELINE.json's north_star uses
