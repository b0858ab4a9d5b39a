"""tests/merge_ref.py -- the definition of merging indexes (DESIGN.md 3.4), on list-major arrays.

faiss InvertedLists::merge_from as the merge stage of build_phrase_index.py:282-338 uses it: for every list l the result holds the
first index's rows of l, then each source's rows of l, in argument order, each in its stored order.  A source row's label is its
stored label plus add_id; an index without labels (None) has the sequential labels 0 .. ntotal - 1 (its list-major row).  numpy
concatenation per list, nothing else.
"""
import numpy as np


def arrays(ref):
    """(list_len, codes, ids) of an oracle RefIndex, sequential labels and synthetic codes materialised."""
    codes = ref.codes if ref.codes is not None else np.concatenate(
        [ref.list_codes(l) for l in range(ref.nlist)] + [np.zeros((0, ref.code_size), np.uint8)])
    ids = ref.ids if ref.ids is not None else np.arange(ref.ntotal, dtype=np.int64)
    return np.asarray(ref.list_len, np.int64), codes, ids


def np_merge(dest, sources, add_id=0):
    """dest, sources: (list_len [nlist], codes [n, M], ids [n] or None), list-major -> the merged (list_len, codes, ids)."""
    parts = [dest] + list(sources)
    nlist = len(dest[0])
    lists, part, codes, ids = [], [], [], []
    for k, (ln, c, i) in enumerate(parts):
        ln = np.asarray(ln, np.int64)
        assert ln.shape == (nlist,)
        n = int(ln.sum())
        lab = np.arange(n, dtype=np.int64) if i is None else np.asarray(i, np.int64)
        assert lab.shape == (n,) and len(c) == n
        lists.append(np.repeat(np.arange(nlist, dtype=np.int64), ln))
        part.append(np.full(n, k, np.int64))
        codes.append(np.asarray(c, np.uint8).reshape(n, np.shape(dest[1])[1]))
        ids.append(lab if k == 0 else lab + add_id)
    order = np.lexsort((np.concatenate(part), np.concatenate(lists)))        # by list, then by part; stored order inside a part
    lens = sum(np.asarray(p[0], np.int64) for p in parts)
    return lens, np.concatenate(codes)[order], np.concatenate(ids)[order]
