"""oracle/filter_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The filtered search (DESIGN.md 3.6): faiss index.search(x, k, params=SearchParametersIVF(sel=IDSelectorBatch | IDSelectorRange |
IDSelectorNot)) (faiss >= 1.7.3) [3P].

1. ``selected_rows``: the selector's rows of an oracle RefIndex, one byte per list-major row -- a row is selected exactly when its
   label is (the label set or range of remove_ids; exclude inverts it).
2. ``search``: ctypes binding of ``oracle/filter_ref.c:ref_search_preassigned_filtered`` after the oracle's own rotation and coarse
   quantizer.
tests/test_filter_cpu.py holds (2) to tests/filter_ref.py's numpy restatement bit for bit.

Only tests/ and tools/bench_filter.py may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ivfpq_ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfilter_ref.so")
_lib = None


def build(force=False):
    """Same flags as ivfpq_ref.build (no fast-math, no fp contraction beyond the explicit fmaf)."""
    srcs = [os.path.join(_HERE, f) for f in ("filter_ref.c", "ivfpq_ref.c")]
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
        _lib = C.CDLL(_SO)
    return _lib


def labels(ref):
    """The list-major labels of a RefIndex (sequential 0 .. ntotal - 1 when it has none)."""
    return ref.ids if ref.ids is not None else np.arange(ref.ntotal, dtype=np.int64)


def selected_rows(ref, sel, exclude=False):
    """sel: an int64 label array (any order, duplicates, absent or negative labels match nothing) or a step-1 range -> uint8 [ntotal]."""
    lab = labels(ref)
    if isinstance(sel, range):
        assert sel.step == 1
        hit = (lab >= sel.start) & (lab < sel.stop)
    else:
        hit = np.isin(lab, np.asarray(sel, dtype=np.int64))
    return (hit != bool(exclude)).astype(np.uint8)


def search(ref, x, k, nprobe, selected):
    """The filtered search of RefIndex ref: x [n,d] -> (D [n,k] f32, I [n,k] i64, key [n,nprobe])."""
    xr = ref.rotate(x)
    _, key = ref.coarse(xr, nprobe)
    selected = np.ascontiguousarray(selected, dtype=np.uint8)
    assert selected.shape == (ref.ntotal,)
    n = len(xr)
    D = np.empty((n, k), dtype=np.float32)
    I = np.empty((n, k), dtype=np.int64)
    lib().ref_search_preassigned_filtered(C.byref(ref.s), R._p(xr), C.c_int64(n), R._p(key), C.c_int(nprobe), C.c_int(k), R._p(selected),
                                          R._p(D), R._p(I))
    return D, I, key
