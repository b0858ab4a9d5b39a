"""tests/query_filter_ref.py -- per-query filters (DESIGN.md 3.7), restated in numpy.

A per-query filter holds selectors and the selector of every query of a batch (-1: none).  Row i of the batch's search is the filtered
search of query i alone with its selector's row mask (tests/filter_ref.py), or the unfiltered search for -1.  A selector is held as a
CSR over the shard's lists: for list lo + j, entries off[j] .. off[j + 1] of (blk, word) -- the list's blocks that hold a selected row,
ascending, and their mask words.
"""
import numpy as np

from oracle import filter_ref as FR
from tests.filter_ref import np_mask


def np_csr(list_len, selected, lo=0, hi=None):
    """selected [ntotal] (list-major rows of ALL lists) -> (off u32 [hi - lo + 1], blk u32 [m], word u32 [m]) of the shard [lo, hi)."""
    list_len = np.asarray(list_len, dtype=np.int64)
    hi = len(list_len) if hi is None else hi
    mask = np_mask(list_len, selected, lo, hi)
    nb = (list_len[lo:hi] + 31) // 32
    first = np.concatenate([[0], np.cumsum(nb)])
    off, blk, word = [0], [], []
    for j in range(hi - lo):
        w = mask[first[j]:first[j + 1]]
        b = np.flatnonzero(w)
        blk.append(b)
        word.append(w[b])
        off.append(off[-1] + len(b))
    cat = lambda a: np.concatenate(a + [np.zeros(0, np.int64)]).astype(np.uint32)   # noqa: E731
    return np.asarray(off, dtype=np.uint32), cat(blk), cat(word)


def csr_mask(list_len, off, blk, word, lo=0, hi=None):
    """The row mask of tests/filter_ref.py expanded from a CSR."""
    list_len = np.asarray(list_len, dtype=np.int64)
    hi = len(list_len) if hi is None else hi
    nb = (list_len[lo:hi] + 31) // 32
    first = np.concatenate([[0], np.cumsum(nb)])[:-1]
    out = np.zeros(int(nb.sum()), dtype=np.uint32)
    lists = np.repeat(np.arange(hi - lo), np.diff(np.asarray(off, dtype=np.int64)))
    out[first[lists] + np.asarray(blk, dtype=np.int64)] = word
    return out


def query_filtered_search(ref, x, k, nprobe, selected, assign, search=FR.search):
    """The definition: selected [F] row selections (uint8 [ntotal]), assign [n] in [-1, F) -> (D [n,k], I [n,k]).  Each query is searched
    with its own selection (every row for -1) by `search` (the C oracle, or tests/filter_ref.np_filtered_search); queries are
    independent, so the queries of one selection are searched together."""
    n = len(x)
    D = np.empty((n, k), dtype=np.float32)
    I = np.empty((n, k), dtype=np.int64)
    assign = np.asarray(assign)
    for s in np.unique(assign):
        rows = np.flatnonzero(assign == s)
        sel = np.ones(ref.ntotal, np.uint8) if s < 0 else selected[s]
        D[rows], I[rows], _ = search(ref, x[rows], k, nprobe, sel)
    return D, I
