"""oracle/encode_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The encoding half of the faiss boundary: IndexPreTransform(OPQ) -> IndexIVFPQ::add_with_ids (faiss 1.6.x, by_residual) [3P], as
reference build_phrase_index.py:145-150,156-279 calls it, with the fixed floating-point order of DESIGN.md 3.1.

1. ``encode`` / ``GrowableRefIndex``: ctypes binding of ``oracle/encode_ref.c:ref_encode`` (which compiles in ivfpq_ref.c, so the
   rotation and the coarse quantizer are the search oracle's own code), and a RefIndex that can grow like faiss' add_with_ids.
2. ``np_encode``: the numpy restatement, built on ivfpq_ref's np_rotate / np_coarse / fma32 (small cases only).
tests/test_add_cpu.py holds the two to bit-equality, the lists to ref_coarse top-1 and the codes to the fp64 argmin.

Only tests/, __graft_entry__.smoke() and tools/bench_add.py's host baseline may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ivfpq_ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libencode_ref.so")
_lib = None


def build(force=False):
    """Same flags as ivfpq_ref.build (no fast-math, no fp contraction beyond the explicit fmaf)."""
    srcs = [os.path.join(_HERE, f) for f in ("encode_ref.c", "ivfpq_ref.c")]
    if (not force) and os.path.exists(_SO) and all(os.path.getmtime(_SO) >= os.path.getmtime(s) for s in srcs):
        return _SO
    cmd = ["gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-shared",
           "-fvisibility=hidden", "-o", _SO, srcs[0], "-lm"]
    subprocess.check_call(cmd)
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.ref_num_threads.restype = C.c_int
        _lib = L
    return _lib


def encode(A, Cm, pq, x):
    """ref_encode: x [n,d] -> (list_no [n] i64, codes [n,M] u8)."""
    x, A, Cm, pq = R._f32(x), R._f32(A), R._f32(Cm), R._f32(pq)
    n, d = x.shape
    M, ksub, dsub = pq.shape
    list_no = np.empty(n, dtype=np.int64)
    codes = np.empty((n, M), dtype=np.uint8)
    lib().ref_encode(R._p(x), C.c_int64(n), C.c_int(d), R._p(A), R._p(Cm), C.c_int64(len(Cm)), R._p(pq), C.c_int(M), C.c_int(ksub),
                     C.c_int(dsub), R._p(list_no), R._p(codes))
    return list_no, codes


def np_encode(x, A, Cm, pq):
    """numpy restatement of ref_encode: rotation, top-1 coarse (heap tie rule), fp32 residual, per sub-quantizer fmaf chain
    acc = fma(d_t, d_t, acc) over t, argmin with the lowest codeword winning a tie."""
    xr = R.np_rotate(x, A)
    Cm, pq = R._f32(Cm), R._f32(pq)
    _, key = R.np_coarse(xr, Cm, 1)
    list_no = key[:, 0]
    r = xr - Cm[list_no]                                             # fp32 - fp32 -> one correctly rounded fp32 subtraction
    M, ksub, dsub = pq.shape
    codes = np.empty((len(xr), M), dtype=np.uint8)
    for m in range(M):
        acc = np.zeros((len(xr), ksub), dtype=np.float32)
        for t in range(dsub):
            diff = r[:, m * dsub + t][:, None] - pq[m][None, :, t]
            acc = R.fma32(diff, diff, acc)
        codes[:, m] = np.argmin(acc, axis=1)                          # first minimum == strict-< scan, j ascending
    return list_no, codes


class GrowableRefIndex(R.RefIndex):
    """RefIndex that can be filled like faiss' index.add_with_ids."""

    def encode(self, x):
        """IndexPreTransform(OPQ) -> IndexIVFPQ encoding of add_with_ids (ref_encode): x [n,d] -> (list_no [n] i64, codes [n,M] u8)."""
        return encode(self.A, self.centroids(), self.pq, x)

    def add_with_ids(self, x, ids=None):
        """== faiss index.add_with_ids(x, ids) (build_phrase_index.py:145-150); ids None -> ntotal + arange(n) like IndexIVF::add.
        Returns the (list_no, codes) of the new rows."""
        list_no, codes = self.encode(x)
        self.append(list_no, codes, self.ntotal + np.arange(len(list_no), dtype=np.int64) if ids is None else ids)
        return list_no, codes

    def append(self, list_no, codes, ids):
        """Append encoded rows to their lists in input order (ArrayInvertedLists::add_entry). The index becomes an explicit one:
        synthetic codes are materialised and implicit labels become their values (list_off[l] + j)."""
        assert self.code_off is None
        list_no = np.asarray(list_no, dtype=np.int64)
        ids = np.asarray(ids, dtype=np.int64)
        assert len(ids) == len(list_no) == len(codes) and (ids >= 0).all() and ((list_no >= 0) & (list_no < self.nlist)).all()
        old_codes = self.codes if self.codes is not None else np.concatenate(
            [self.list_codes(l) for l in range(self.nlist)] + [np.zeros((0, self.code_size), np.uint8)])
        old_ids = self.ids if self.ids is not None else np.arange(self.ntotal, dtype=np.int64)
        lists = np.concatenate([np.repeat(np.arange(self.nlist, dtype=np.int64), self.list_len), list_no])
        order = np.argsort(lists, kind="stable")
        self.__init__(self.A, self.pq, self.list_len + np.bincount(list_no, minlength=self.nlist), centroids=self.C,
                      codes=np.concatenate([old_codes, np.asarray(codes, np.uint8)])[order], ids=np.concatenate([old_ids, ids])[order],
                      seed=self.seed, centroid_sigma=self.centroid_sigma)
