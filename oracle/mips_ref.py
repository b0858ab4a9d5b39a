"""oracle/mips_ref.py -- TEST INFRASTRUCTURE.  Item-by-item restatement of the reference's phrase stage
(reference densephrases/index.py:220-448: search_phrase + aggregate_results) over the oracle IVF-PQ index,
written the way the reference runs it (one reconstruct per id, one validity test per candidate, python sorting) so the
batched product implementation (densephrases_b200/mips.py) can be compared result-by-result.
PINNED against the reference itself: tests/golden/mips_search.json holds the outputs of the UNMODIFIED reference `MIPS.search`
(run in the build container by tests/golden/make_mips_golden.py over the same synthetic corpus and oracle index);
tests/test_mips.py::test_phrase_stage_matches_reference_golden checks this restatement and the product mirror against it.
(The IVF-PQ search underneath stays "parity unpinned" at the FAISS boundary, see oracle/ivfpq_ref.c.)"""
import numpy as np


def ref_get_idxs(I, idx_f, ntotal, max_idx=1e9):
    I = np.clip(np.asarray(I), 0, ntotal - 1)                                   # index.py:128-133
    doc = np.zeros(I.shape, dtype=np.int64)
    word = np.zeros(I.shape, dtype=np.int64)
    for pos in np.ndindex(I.shape):
        off = int(I[pos] / max_idx) * int(max_idx)
        row = int(I[pos]) % int(max_idx)
        doc[pos] = idx_f[str(off)]['doc'][row]
        word[pos] = idx_f[str(off)]['word'][row]
    return doc, word


def _reconstruct_or_zero(ref, label, d):
    v, found = ref.reconstruct(np.array([label], dtype=np.int64))               # faiss reconstruct raises on a miss; the reference
    return v[0] if found[0] else np.zeros(d, dtype=np.float32)                  # catches it and substitutes zeros (index.py:285-288)


def ref_search(ref, idx_f, doc_groups, query, top_k=10, nprobe=256, max_answer_length=10, aggregate=False, agg_strat='opt1',
               return_idxs=False, normalize_answer=None):
    """== MIPS.search (index.py:450-482) on the oracle index `ref`."""
    L = max_answer_length
    B = query.shape[0]
    q = query.astype(np.float32)
    qs, qe = q[:, :q.shape[1] // 2], q[:, q.shape[1] // 2:]
    D, I = ref.search(np.concatenate([qs, qe], 0), top_k, nprobe)
    s_doc, s_word = ref_get_idxs(I[:B], idx_f, ref.ntotal)
    e_doc, e_word = ref_get_idxs(I[B:], idx_f, ref.ntotal)
    R = ref.A.reshape(ref.d, ref.d)
    outs = []
    for b in range(B):
        hits = []
        for h in range(top_k):
            for anchor in ('start', 'end'):
                doc = int(s_doc[b, h] if anchor == 'start' else e_doc[b, h])
                meta = doc_groups[str(doc)]
                f2o = meta['f2o_start']

                def valid(si, ei):
                    if doc < 0 or si < 0 or si >= len(f2o) or ei < 0 or ei >= len(f2o):
                        return False
                    return 0 <= f2o[ei] - f2o[si] <= L

                if anchor == 'start':
                    label, word, base = int(I[b, h]), int(s_word[b, h]), float(D[b, h])
                    labels = [label + i for i in range(L)]
                    cands = [(word, word + i) if valid(word, word + i) else None for i in range(L)]
                    qvec = qe[b]
                else:
                    label, word, base = int(I[B + b, h]), int(e_word[b, h]), float(D[B + b, h])
                    labels = [label - i for i in range(L - 1, -1, -1)]
                    cands = [(word - i, word) if valid(word - i, word) else None for i in range(L - 1, -1, -1)]
                    qvec = qs[b]
                raw = np.stack([_reconstruct_or_zero(ref, lb, ref.d) for lb in labels]).astype(np.float32)
                unrot = raw @ R                                                  # index.py:340,365 (fp32)
                sc = np.float32(base) + (qvec[None, :] * unrot).sum(1).astype(np.float32) + np.array([0.0 if c else -1e9 for c in cands])
                j = int(np.argmax(sc))
                si, ei = cands[j] if cands[j] else ((word, -1) if anchor == 'start' else (-1, word))
                c0 = int(meta['word2char_start'][f2o[si]])
                c1 = int(meta['word2char_end'][f2o[ei]]) if (len(meta['word2char_end']) > 0 and ei >= 0) else c0 + 1
                rec = {'context': meta['context'], 'title': [meta['title']], 'doc_idx': doc, 'start_pos': c0, 'end_pos': c1,
                       'start_idx': si, 'end_idx': ei, 'score': float(sc[j]), 'start_vec': None, 'end_vec': None}
                if return_idxs:
                    if anchor == 'start':
                        rec['start_vec'], rec['end_vec'] = raw[0] @ R, unrot[j] @ R
                    else:
                        rec['start_vec'], rec['end_vec'] = unrot[j] @ R, raw[-1] @ R
                rec['answer'] = rec['context'][c0:c1]
                ctx = rec['context']                                              # adjust(), index.py:167-176
                lo = ctx.rfind(' [PAR] ', 0, c0)
                lo = 0 if lo == -1 else lo + len(' [PAR] ')
                hi = ctx.find(' [PAR] ', c1)
                hi = len(ctx) if hi == -1 else hi
                rec['context'], rec['start_pos'], rec['end_pos'] = ctx[lo:hi], c0 - lo, c1 - lo
                hits.append(rec)
        hits = [r for r in sorted(hits, key=lambda r: -r['score']) if r['score'] > -1e5]
        if aggregate:
            seen = {}
            for pos, r in enumerate(hits):
                key = {'opt1': f'{r["title"]}_{r["start_pos"]}_{r["end_pos"]}', 'opt2': r['context'], 'opt3': f'{r["title"]}',
                       'opt4': normalize_answer(r['answer']) if normalize_answer else r['answer']}[agg_strat]
                if key in seen:
                    r['score'] = -1e8
                    if agg_strat == 'opt4' and r['title'][0] not in hits[seen[key]]['title']:
                        hits[seen[key]]['title'] += r['title']
                else:
                    seen[key] = pos
            hits = [r for r in sorted(hits, key=lambda r: -r['score']) if r['score'] > -1e5]
        outs.append(hits)
    return outs
