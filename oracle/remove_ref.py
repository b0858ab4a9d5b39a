"""oracle/remove_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The removal half of the faiss boundary: IndexIVF::remove_ids of faiss 1.6.x without a direct map (DirectMap::NoMap) [3P], on the
list-major arrays of an index (DESIGN.md 3.2).

1. ``ref_remove`` / ``RemovableRefIndex.remove_ids``: ctypes binding of ``oracle/remove_ref.c:ref_remove``, the literal faiss loop
   per list, and a GrowableRefIndex that can also shrink.
2. ``np_remove``: a vectorised restatement of the loop's closed form (kept rows below L' = len - |S| stay; the h-th hole below L'
   takes the h-th kept row at or above L' counted from the end).  tests/test_remove_cpu.py holds the two to equality.

A selector is a label set (any int64 array: order, duplicates and absent or negative labels do not matter) or a step-1 ``range``.

Only tests/, __graft_entry__.smoke() and tools/bench_remove.py's host baseline may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import encode_ref as E

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libremove_ref.so")
_lib = None


def build(force=False):
    src = os.path.join(_HERE, "remove_ref.c")
    if (not force) and os.path.exists(_SO) and os.path.getmtime(_SO) >= os.path.getmtime(src):
        return _SO
    subprocess.check_call(["gcc", "-O3", "-fPIC", "-shared", "-fvisibility=hidden", "-o", _SO, src])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.ref_remove.restype = C.c_int64
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def selector(sel):
    """-> (sorted unique labels or None, lo, hi); a range selects [lo, hi)."""
    if isinstance(sel, range):
        assert sel.step == 1
        return None, sel.start, sel.stop
    return np.unique(np.asarray(sel, dtype=np.int64)), 0, 0


def is_empty(sel):
    s, lo, hi = selector(sel)
    return len(s) == 0 if s is not None else lo >= hi


def ref_remove_inplace(lens, codes, ids, s, lo, hi, per):
    """ref_remove on C-contiguous int64 lens / ids, uint8 codes (modified in place) and a selector() triple -> rows removed."""
    return lib().ref_remove(C.c_int64(len(lens)), _p(lens), _p(codes), _p(ids), C.c_int(codes.shape[1]), None if s is None else _p(s),
                            C.c_int64(0 if s is None else len(s)), C.c_int64(lo), C.c_int64(hi), _p(per))


def ref_remove(list_len, codes, ids, sel):
    """The literal loop: (list_len, codes [n,M], ids [n]) list-major -> (new list_len, codes, ids, removed per list)."""
    lens = np.array(list_len, dtype=np.int64)
    codes = np.array(codes, dtype=np.uint8, order="C")
    ids = np.array(ids, dtype=np.int64)
    s, lo, hi = selector(sel)
    per = np.zeros(len(lens), dtype=np.int64)
    n = ref_remove_inplace(lens, codes, ids, s, lo, hi, per)
    keep = int(lens.sum())
    assert n == int(per.sum()) and keep + n == len(ids)
    return lens, codes[:keep], ids[:keep], per


def np_remove(list_len, codes, ids, sel):
    """The closed form, vectorised over all lists; same outputs as ref_remove."""
    lens = np.asarray(list_len, dtype=np.int64)
    ids = np.asarray(ids, dtype=np.int64)
    s, lo, hi = selector(sel)
    hit = np.isin(ids, s) if s is not None else (ids >= lo) & (ids < hi)
    li = np.repeat(np.arange(len(lens)), lens)
    j = np.arange(len(ids)) - np.repeat(np.cumsum(lens) - lens, lens)
    per = np.bincount(li, weights=hit, minlength=len(lens)).astype(np.int64)
    Lp = (lens - per)[li]
    holes = np.flatnonzero(hit & (j < Lp))                                  # by list, ascending j
    donors = np.flatnonzero(~hit & (j >= Lp))
    donors = donors[np.lexsort((-j[donors], li[donors]))]                    # by list, descending j
    assert np.array_equal(li[holes], li[donors])                            # as many donors as holes in every list
    src = np.arange(len(ids))
    src[holes] = donors
    src = src[j < Lp]
    return lens - per, np.asarray(codes, dtype=np.uint8)[src], ids[src], per


class RemovableRefIndex(E.GrowableRefIndex):
    """GrowableRefIndex that can also shrink like faiss' index.remove_ids."""

    def remove_ids(self, sel, fn=ref_remove):
        """== index.remove_ids(IDSelectorBatch(sel) | IDSelectorRange(lo, hi)) -> (rows removed, removed per list).  A non-empty
        selector makes the index an explicit one (synthetic codes materialised, implicit labels become list_off[l] + j), as append does."""
        if is_empty(sel):
            return 0, np.zeros(self.nlist, dtype=np.int64)
        assert self.code_off is None
        codes = self.codes if self.codes is not None else np.concatenate(
            [self.list_codes(l) for l in range(self.nlist)] + [np.zeros((0, self.code_size), np.uint8)])
        ids = self.ids if self.ids is not None else np.arange(self.ntotal, dtype=np.int64)
        lens, codes, ids, per = fn(self.list_len, codes, ids, sel)
        self.__init__(self.A, self.pq, lens, centroids=self.C, codes=codes, ids=ids, seed=self.seed, centroid_sigma=self.centroid_sigma)
        return int(per.sum()), per
