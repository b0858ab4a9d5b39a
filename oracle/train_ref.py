"""oracle/train_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The training half of the faiss boundary: the spherical k-means coarse quantizer and the residual PQ codebooks of
IndexPreTransform(OPQMatrix, IndexIVFPQ(IndexFlatIP)) (faiss 1.6.x Clustering / ProductQuantizer::train) [3P], as reference
build_phrase_index.py:96-142 trains them, with the fixed floating-point order and draws of DESIGN.md 3.3.

1. ``train_coarse`` / ``train_pq`` / ``sample`` / ``init_rows`` / ``split_clusters``: ctypes bindings of ``oracle/train_ref.c``
   (which compiles in ivfpq_ref.c, so rotation, coarse top-1 and rnd64 are the search oracle's own code).
2. ``np_train_coarse`` / ``np_train_pq``: the numpy restatement, built on ivfpq_ref's np_rotate / np_coarse / fma32 (small cases).
tests/test_train_cpu.py holds the two to bit-equality.

Only tests/, __graft_entry__.smoke() and tools/bench_train.py may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ivfpq_ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libtrain_ref.so")
_lib = None
STREAM_SAMPLE, STREAM_INIT, STREAM_SPLIT = 4, 5, 6
SPLIT_EPS = np.float32(1.0 / 1024.0)


def build(force=False):
    """Same flags as ivfpq_ref.build (no fast-math, no fp contraction beyond the explicit fmaf)."""
    srcs = [os.path.join(_HERE, f) for f in ("train_ref.c", "ivfpq_ref.c")]
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
        L.ref_train_sample.restype = C.c_int64
        L.ref_split_clusters.restype = C.c_int64
        L.ref_train_coarse.restype = C.c_int
        L.ref_train_pq.restype = C.c_int
        _lib = L
    return _lib


def sample(n, cap, seed, which):
    """Row numbers of the training sample (ascending): which 0 = coarse quantizer, 1 = PQ."""
    idx = np.empty(min(n, cap), dtype=np.int64)
    ns = lib().ref_train_sample(C.c_int64(n), C.c_int64(cap), C.c_uint64(seed), C.c_uint64(which), R._p(idx))
    return idx[:ns]


def init_rows(ns, k, seed, s):
    """Sample positions of the k initial centroids of k-means run s (0 coarse, 1 + m sub-quantizer m)."""
    out = np.empty(k, dtype=np.int64)
    lib().ref_train_init_rows(C.c_int64(ns), C.c_int64(k), C.c_uint64(seed), C.c_uint64(s), R._p(out))
    return out


def split_clusters(Cm, h, ns, seed, s, it):
    """ref_split_clusters on copies -> (C, h, nsplit)."""
    Cm = np.array(Cm, dtype=np.float32, order="C")
    h = np.array(h, dtype=np.float32)
    k, dd = Cm.shape
    nsplit = lib().ref_split_clusters(R._p(Cm), C.c_int64(k), C.c_int(dd), R._p(h), C.c_int64(ns), C.c_uint64(seed), C.c_uint64(s),
                                      C.c_uint64(it))
    return Cm, h, int(nsplit)


def train_coarse(x, A, k, niter, seed, max_points_per_centroid=256, C0=None):
    """ref_train_coarse -> (centroids [k, d], obj [niter] f64, nsplit [niter] i64).  C0: hot start."""
    x, A = R._f32(x), R._f32(A)
    n, d = x.shape
    Cm = np.zeros((k, d), np.float32) if C0 is None else np.array(C0, dtype=np.float32, order="C")
    obj = np.zeros(niter, np.float64)
    nsplit = np.zeros(niter, np.int64)
    rc = lib().ref_train_coarse(R._p(x), C.c_int64(n), C.c_int(d), R._p(A), C.c_int64(k), C.c_int(niter), C.c_uint64(seed),
                                C.c_int64(max_points_per_centroid), C.c_int(C0 is not None), R._p(Cm), R._p(obj), R._p(nsplit))
    if rc:
        raise ValueError(f"train_coarse: n = {n} < k = {k}")
    return Cm, obj, nsplit


def train_pq(x, A, Cm, niter, seed, max_points_per_centroid=256, pq0=None, M=96, ksub=256):
    """ref_train_pq -> pq [M, ksub, d // M].  Cm None: no residual (OPQ).  pq0: hot start."""
    x, A = R._f32(x), R._f32(A)
    n, d = x.shape
    dsub = d // M
    pq = np.zeros((M, ksub, dsub), np.float32) if pq0 is None else np.array(pq0, dtype=np.float32, order="C")
    Cm = None if Cm is None else R._f32(Cm)
    rc = lib().ref_train_pq(R._p(x), C.c_int64(n), C.c_int(d), R._p(A), R._p(Cm), C.c_int64(0 if Cm is None else len(Cm)), C.c_int(M),
                            C.c_int(ksub), C.c_int(dsub), C.c_int(niter), C.c_uint64(seed), C.c_int64(max_points_per_centroid),
                            C.c_int(pq0 is not None), R._p(pq))
    if rc:
        raise ValueError(f"train_pq: n = {n} < ksub = {ksub}")
    return pq


# ================================================================================================
# numpy restatement
# ================================================================================================
def _rank(keys, take):
    return np.lexsort((np.arange(len(keys)), keys))[:take]            # key ascending, then position


def np_sample(n, cap, seed, which):
    if n <= cap:
        return np.arange(n, dtype=np.int64)
    keys = np.array([R.lib().ref_rnd64(seed, STREAM_SAMPLE, i, which) for i in range(n)], dtype=np.uint64)
    return np.sort(_rank(keys, cap)).astype(np.int64)


def np_init_rows(ns, k, seed, s):
    keys = np.array([R.lib().ref_rnd64(seed, STREAM_INIT, s, p) for p in range(ns)], dtype=np.uint64)
    return _rank(keys, k).astype(np.int64)


def np_split_clusters(Cm, h, ns, seed, s, it):
    Cm, h = Cm.copy(), h.copy()
    k = len(Cm)
    draw, nsplit = 0, 0
    up, dn = np.float32(1) + SPLIT_EPS, np.float32(1) - SPLIT_EPS
    even = (np.arange(Cm.shape[1]) % 2) == 0
    for ci in range(k):
        if h[ci] != 0:
            continue
        cj = 0
        while True:
            with np.errstate(divide="ignore", invalid="ignore"):         # ns == k: +-inf or nan, as in C
                p = (h[cj] - np.float32(1)) / np.float32(ns - k)
            u =np.float32(R.lib().ref_rnd64(seed, STREAM_SPLIT, (s << 32) | it, draw) >> 40) * np.float32(2.0 ** -24)
            draw += 1
            if u < p:
                break
            cj = (cj + 1) % k
        Cm[ci] = Cm[cj]
        Cm[ci] = np.where(even, Cm[ci] * up, Cm[ci] * dn)
        Cm[cj] = np.where(even, Cm[cj] * dn, Cm[cj] * up)
        h[ci] = h[cj] / np.float32(2)
        h[cj] = h[cj] - h[ci]
        nsplit += 1
    return Cm, h, nsplit


def np_update(xs, assign, Cm):
    """sum in ascending row order with plain fp32 adds, times the fp32 reciprocal of the count; empty clusters keep their row."""
    Cm = Cm.copy()
    k = len(Cm)
    h = np.zeros(k, np.float32)
    for c in range(k):
        rows = xs[assign == c]
        h[c] = np.float32(len(rows))
        if len(rows) == 0:
            continue
        s = np.zeros(xs.shape[1], np.float32)
        for r in rows:
            s = s + r
        Cm[c] = s * (np.float32(1) / np.float32(len(rows)))
    return Cm, h


def np_renorm(Cm):
    Cm = Cm.copy()
    for c in range(len(Cm)):
        nr = np.float32(0)
        for t in range(Cm.shape[1]):
            nr = R.fma32(Cm[c, t], Cm[c, t], nr)
        if nr > 0:
            Cm[c] = Cm[c] * (np.float32(1) / np.sqrt(np.float32(nr)))
    return Cm


def np_train_coarse(x, A, k, niter, seed, max_points_per_centroid=256, C0=None):
    n = len(x)
    if n < k:
        raise ValueError("n < k")
    idx = np_sample(n, max_points_per_centroid * k, seed, 0)
    xs = R.np_rotate(R._f32(x)[idx], A)
    if C0 is None:
        Cm = np_renorm(xs[np_init_rows(len(xs), k, seed, 0)])
    else:
        Cm = R._f32(C0).copy()
    obj, nsplit = np.zeros(niter), np.zeros(niter, np.int64)
    for it in range(niter):
        cd, key = R.np_coarse(xs, Cm, 1)
        obj[it] = sum(float(v) for v in cd[:, 0])
        Cm, h = np_update(xs, key[:, 0], Cm)
        Cm, h, nsplit[it] = np_split_clusters(Cm, h, len(xs), seed, 0, it)
        Cm = np_renorm(Cm)
    return Cm, obj, nsplit


def np_train_pq(x, A, Cm, niter, seed, max_points_per_centroid=256, pq0=None, M=96, ksub=256):
    n, d = x.shape
    dsub = d // M
    if n < ksub:
        raise ValueError("n < ksub")
    idx = np_sample(n, max_points_per_centroid * ksub, seed, 1)
    xs = R.np_rotate(R._f32(x)[idx], A)
    if Cm is not None:
        Cm = R._f32(Cm)
        _, key = R.np_coarse(xs, Cm, 1)
        xs = xs - Cm[key[:, 0]]
    pq = np.zeros((M, ksub, dsub), np.float32) if pq0 is None else R._f32(pq0).copy()
    for m in range(M):
        sub = np.ascontiguousarray(xs[:, m * dsub:(m + 1) * dsub])
        cb = sub[np_init_rows(len(xs), ksub, seed, 1 + m)].copy() if pq0 is None else pq[m].copy()
        for it in range(niter):
            acc = np.zeros((len(sub), ksub), np.float32)
            for t in range(dsub):
                diff = sub[:, t][:, None] - cb[None, :, t]
                acc = R.fma32(diff, diff, acc)
            assign = np.argmin(acc, axis=1)                            # first minimum == strict-< scan, j ascending
            cb, h = np_update(sub, assign, cb)
            cb, h, _ = np_split_clusters(cb, h, len(sub), seed, 1 + m, it)
        pq[m] = cb
    return pq
