"""oracle/ivfpq_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Two things live here:

1. ``CRef`` / ``RefIndex``: ctypes binding of ``oracle/ivfpq_ref.c`` (the primary, OpenMP, bit-exact
   CPU restatement of the FAISS ``IndexPreTransform(OPQ) -> IndexIVFPQ(IP, by_residual)`` search that
   reference densephrases/index.py:200 calls, and of ``reconstruct`` at index.py:31,286,296).
2. A *numpy* restatement of the same algorithm (``np_*`` functions; pure-Python heap loops, small cases
   only) plus an exhaustive fp64 scorer. tests/test_oracle.py holds the C and numpy versions to
   bit-equality and both to the fp64 brute force.

PARITY UNPINNED at the FAISS boundary: the reference holds no golden vectors for this path and faiss
(faiss-gpu==1.6.5, requirements.txt:2) cannot be installed here; see the header of ivfpq_ref.c.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libivfpq_ref.so")
NEUTRAL = np.float32(-np.finfo(np.float32).max)


def build(force=False):
    """gcc -O3 -march=x86-64-v3 -fopenmp (AVX2+FMA, portable across the build container and the GPU box; no fast-math, no fp contraction beyond the explicit fmaf)."""
    src = os.path.join(_HERE, "ivfpq_ref.c")
    if (not force) and os.path.exists(_SO) and os.path.getmtime(_SO) >= os.path.getmtime(src):
        return _SO
    cmd = ["gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-shared",
           "-fvisibility=hidden", "-o", _SO, src, "-lm"]
    subprocess.check_call(cmd)
    return _SO


class _RefIndexStruct(C.Structure):
    _fields_ = [("d", C.c_int), ("M", C.c_int), ("ksub", C.c_int), ("dsub", C.c_int), ("code_size", C.c_int),
                ("nlist", C.c_int64), ("A", C.c_void_p), ("C", C.c_void_p), ("pq", C.c_void_p),
                ("list_len", C.c_void_p), ("list_off", C.c_void_p), ("codes", C.c_void_p), ("ids", C.c_void_p),
                ("seed", C.c_uint64), ("centroid_sigma", C.c_float), ("code_off", C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.ref_rnd64.restype = C.c_uint64
        L.ref_rnd64.argtypes = [C.c_uint64] * 4
        L.ref_num_threads.restype = C.c_int
        L.ref_sizeof_index.restype = C.c_int
        assert L.ref_sizeof_index() == C.sizeof(_RefIndexStruct)
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def gen_codes(seed, list_no, j0, n, code_size=96):
    out = np.empty((n, code_size), dtype=np.uint8)
    lib().ref_gen_codes(C.c_uint64(seed), C.c_int64(list_no), C.c_int64(j0), C.c_int64(n), C.c_int(code_size), _p(out))
    return out


def gen_centroids(seed, l0, n, d=768, sigma=0.5):
    out = np.empty((n, d), dtype=np.float32)
    lib().ref_gen_centroids(C.c_uint64(seed), C.c_int64(l0), C.c_int64(n), C.c_int(d), C.c_float(sigma), _p(out))
    return out


def gen_pq(seed, M=96, ksub=256, dsub=8, sigma=0.25):
    out = np.empty((M, ksub, dsub), dtype=np.float32)
    lib().ref_gen_pq(C.c_uint64(seed), C.c_int(M), C.c_int(ksub), C.c_int(dsub), C.c_float(sigma), _p(out))
    return out


class RefIndex:
    """Explicit (codes/ids arrays) or synthetic (codes, optionally centroids, regenerated from `seed`)."""

    def __init__(self, A, pq, list_len, centroids=None, codes=None, ids=None, seed=0, centroid_sigma=0.5, code_off=None):
        self.A = _f32(A)
        self.pq = _f32(pq)
        self.M, self.ksub, self.dsub = self.pq.shape
        self.d = self.A.shape[0]
        assert self.M * self.dsub == self.d
        self.code_size = self.M
        self.list_len = np.ascontiguousarray(list_len, dtype=np.int64)
        self.nlist = len(self.list_len)
        self.list_off = np.zeros(self.nlist, dtype=np.int64)
        np.cumsum(self.list_len[:-1], out=self.list_off[1:])
        self.ntotal = int(self.list_len.sum())
        self.C = None if centroids is None else _f32(centroids)
        self.codes = None if codes is None else np.ascontiguousarray(codes, dtype=np.uint8)
        self.ids = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64)
        self.seed, self.centroid_sigma = int(seed), float(centroid_sigma)
        self.code_off = None if code_off is None else np.ascontiguousarray(code_off, dtype=np.int64)
        self.s = _RefIndexStruct(self.d, self.M, self.ksub, self.dsub, self.code_size, self.nlist, _p(self.A).value,
                                 None if self.C is None else _p(self.C).value, _p(self.pq).value,
                                 _p(self.list_len).value, _p(self.list_off).value,
                                 None if self.codes is None else _p(self.codes).value,
                                 None if self.ids is None else _p(self.ids).value, self.seed, self.centroid_sigma,
                                 None if self.code_off is None else _p(self.code_off).value)

    def with_resident_lists(self, lists):
        """Copy of a synthetic index whose `lists` are materialised in RAM (like faiss' inverted lists); every other
        list stays virtual and must not be probed. Used by bench.py's CPU baseline so the timed scan reads resident codes."""
        assert self.codes is None
        lists = np.unique(np.asarray(lists, dtype=np.int64))
        lists = lists[lists >= 0]
        lens = self.list_len[lists]
        offs = np.zeros(len(lists), dtype=np.int64)
        np.cumsum(lens[:-1], out=offs[1:])
        codes = np.empty((int(lens.sum()), self.code_size), dtype=np.uint8)
        lib().ref_gen_codes_lists(C.c_uint64(self.seed), _p(lists), C.c_int64(len(lists)), _p(np.ascontiguousarray(lens)), _p(offs),
                                  C.c_int(self.code_size), _p(codes))
        code_off = np.full(self.nlist, -1, dtype=np.int64)
        code_off[lists] = offs
        return RefIndex(self.A, self.pq, self.list_len, centroids=self.C, codes=codes, ids=None, seed=self.seed,
                        centroid_sigma=self.centroid_sigma, code_off=code_off)

    # --- C restatement -------------------------------------------------------------------------
    def rotate(self, x):
        x = _f32(x)
        xr = np.empty_like(x)
        lib().ref_rotate(_p(x), C.c_int64(len(x)), C.c_int(self.d), _p(self.A), _p(xr))
        return xr

    def centroids(self):
        return self.C if self.C is not None else gen_centroids(self.seed, 0, self.nlist, self.d, self.centroid_sigma)

    def coarse(self, xr, nprobe):
        xr = _f32(xr)
        n = len(xr)
        cd = np.empty((n, nprobe), dtype=np.float32)
        key = np.empty((n, nprobe), dtype=np.int64)
        Cm = self.centroids()
        lib().ref_coarse(_p(xr), C.c_int64(n), C.c_int(self.d), _p(Cm), C.c_int64(self.nlist), C.c_int(nprobe), _p(cd), _p(key))
        return cd, key

    def search_preassigned(self, xr, key, k):
        xr = _f32(xr)
        key = np.ascontiguousarray(key, dtype=np.int64)
        n, nprobe = key.shape
        D = np.empty((n, k), dtype=np.float32)
        I = np.empty((n, k), dtype=np.int64)
        nsc = C.c_int64(0)
        lib().ref_search_preassigned(C.byref(self.s), _p(xr), C.c_int64(n), _p(key), C.c_int(nprobe), C.c_int(k), _p(D), _p(I),
                                     C.byref(nsc))
        self.last_ncodes = nsc.value
        return D, I

    def search(self, x, k, nprobe=256, return_key=False):
        """== faiss index.search(x, k) with index_ivf.nprobe = nprobe (index.py:53,62,200)."""
        x = _f32(x)
        n = len(x)
        D = np.empty((n, k), dtype=np.float32)
        I = np.empty((n, k), dtype=np.int64)
        key = np.empty((n, nprobe), dtype=np.int64)
        nsc = C.c_int64(0)
        lib().ref_search(C.byref(self.s), _p(x), C.c_int64(n), C.c_int(k), C.c_int(nprobe), _p(D), _p(I), _p(key), C.byref(nsc))
        self.last_ncodes = nsc.value
        return (D, I, key) if return_key else (D, I)

    def locate(self, ids):
        """direct map label -> (list_no, offset); missing -> (-1,-1). Sequential ids when self.ids is None."""
        ids = np.asarray(ids, dtype=np.int64)
        if self.ids is None:
            l = np.searchsorted(self.list_off, ids, side="right") - 1
            ok = (ids >= 0) & (ids < self.ntotal)
            l = np.where(ok, l, -1)
            off = np.where(ok, ids - self.list_off[np.clip(l, 0, None)], -1)
            return l.astype(np.int64), off.astype(np.int64)
        order = np.argsort(self.ids, kind="stable")
        pos = np.searchsorted(self.ids[order], ids)
        pos = np.clip(pos, 0, len(order) - 1)
        hit = self.ids[order][pos] == ids
        row = order[pos]
        l = np.searchsorted(self.list_off, row, side="right") - 1
        return np.where(hit, l, -1).astype(np.int64), np.where(hit, row - self.list_off[l], -1).astype(np.int64)

    def reconstruct(self, ids):
        """== reconst_fn(id) per id (index.py:286,296); missing id -> zeros + found 0 (index.py:287-288)."""
        l, off = self.locate(ids)
        out = np.empty((len(l), self.d), dtype=np.float32)
        found = np.empty(len(l), dtype=np.uint8)
        lib().ref_reconstruct_at(C.byref(self.s), _p(l), _p(off), C.c_int64(len(l)), _p(out), _p(found))
        return out, found

    def list_codes(self, l):
        if self.codes is not None:
            o = self.list_off[l] if self.code_off is None else self.code_off[l]
            return self.codes[o:o + self.list_len[l]]
        return gen_codes(self.seed, l, 0, int(self.list_len[l]), self.code_size)

    def list_ids(self, l):
        o = self.list_off[l]
        return self.ids[o:o + self.list_len[l]] if self.ids is not None else np.arange(o, o + self.list_len[l], dtype=np.int64)


# =================================================================================================
# numpy restatement (small cases). fp32 FMA is emulated exactly: the product of two fp32 is exact
# in fp64; the fp64 sum is corrected to round-to-odd with TwoSum so the final fp32 rounding is the
# single correct rounding of a*b+c.
# =================================================================================================
def fma32(a, b, c):
    a = np.asarray(a, dtype=np.float32).astype(np.float64)
    b = np.asarray(b, dtype=np.float32).astype(np.float64)
    c = np.asarray(c, dtype=np.float32).astype(np.float64)
    p = a * b                                    # exact (24+24 <= 53 bits)
    s = c + p
    bb = s - c
    e = (c - (s - bb)) + (p - bb)                # TwoSum error term, exact
    bits = s.view(np.int64).copy() if isinstance(s, np.ndarray) else np.array(s).view(np.int64).copy()
    s_arr = np.asarray(s)
    inexact = (e != 0) & ((bits & 1) == 0)
    away = (e > 0) == (s_arr > 0)                # error points away from zero -> magnitude + 1ulp
    bits = np.where(inexact & away, bits + 1, bits)
    bits = np.where(inexact & ~away, bits - 1, bits)
    return bits.view(np.float64).astype(np.float32)


def np_matmul_nt_seq(x, W):
    """out[i,o] = sequential fp32 FMA chain over t of x[i,t]*W[o,t]."""
    x = _f32(x)
    W = _f32(W)
    acc = np.zeros((x.shape[0], W.shape[0]), dtype=np.float32)
    for t in range(x.shape[1]):
        acc = fma32(x[:, t:t + 1], W[None, :, t], acc)
    return acc


def np_rotate(x, A):
    return np_matmul_nt_seq(x, A)


class _MinHeap:
    """faiss Heap.h CMin<float,int64>, literal 1-based sift-down/up on values only."""

    def __init__(self, k):
        self.k = k
        self.v = [NEUTRAL] * (k + 1)
        self.i = [-1] * (k + 1)

    def root(self):
        return self.v[1]

    def pop(self, k=None):
        k = self.k if k is None else k
        v, ids = self.v, self.i
        val = v[k]
        i = 1
        while True:
            i1 = i << 1
            i2 = i1 + 1
            if i1 > k:
                break
            if i2 == k + 1 or v[i1] < v[i2]:
                if val < v[i1]:
                    break
                v[i], ids[i] = v[i1], ids[i1]
                i = i1
            else:
                if val < v[i2]:
                    break
                v[i], ids[i] = v[i2], ids[i2]
                i = i2
        v[i], ids[i] = v[k], ids[k]

    def push(self, val, id_):
        v, ids = self.v, self.i
        i = self.k
        while i > 1:
            f = i >> 1
            if not (val < v[f]):
                break
            v[i], ids[i] = v[f], ids[f]
            i = f
        v[i], ids[i] = val, id_

    def reorder(self):
        k = self.k
        v, ids = self.v, self.i
        ii = 0
        for i in range(k):
            val, id_ = v[1], ids[1]
            self.pop(k - i)
            v[k - ii], ids[k - ii] = val, id_          # 0-based slot k-ii-1
            if id_ != -1:
                ii += 1
        outv = v[1 + k - ii:1 + k] + [NEUTRAL] * (k - ii)
        outi = ids[1 + k - ii:1 + k] + [-1] * (k - ii)
        return np.array(outv, dtype=np.float32), np.array(outi, dtype=np.int64)


def np_topk_heap(scores, k):
    h = _MinHeap(k)
    for j, s in enumerate(scores):
        if h.root() < s:
            h.pop()
            h.push(np.float32(s), j)
    return h.reorder()


def np_coarse(xr, Cm, nprobe):
    S = np_matmul_nt_seq(xr, Cm)
    cd = np.empty((len(xr), nprobe), dtype=np.float32)
    key = np.empty((len(xr), nprobe), dtype=np.int64)
    for i in range(len(xr)):
        cd[i], key[i] = np_topk_heap(S[i], nprobe)
    return cd, key


def np_lut(xr_row, pq):
    M, ksub, dsub = pq.shape
    lut = np.zeros((M, ksub), dtype=np.float32)
    q = _f32(xr_row).reshape(M, dsub)
    for t in range(dsub):
        lut = fma32(q[:, t:t + 1], pq[:, :, t], lut)
    return lut


def np_search(ix, x, k, nprobe):
    """Whole chain in numpy/python; ix is a RefIndex (used only as a data holder here)."""
    xr = np_rotate(x, ix.A)
    Cm = ix.centroids()
    _, key = np_coarse(xr, Cm, nprobe)
    n = len(xr)
    D = np.empty((n, k), dtype=np.float32)
    I = np.empty((n, k), dtype=np.int64)
    marange = np.arange(ix.M)
    for i in range(n):
        lut = np_lut(xr[i], ix.pq)
        h = _MinHeap(k)
        for r in range(nprobe):
            l = int(key[i, r])
            if l < 0 or ix.list_len[l] == 0:
                continue
            dis0 = np_matmul_nt_seq(xr[i:i + 1], Cm[l:l + 1])[0, 0]
            codes = ix.list_codes(l)
            ids = ix.list_ids(l)
            dis = np.full(len(codes), dis0, dtype=np.float32)
            for m in marange:                                   # sequential fp32 adds, m ascending
                dis = (dis + lut[m, codes[:, m]]).astype(np.float32)
            for j in range(len(codes)):
                if h.root() < dis[j]:
                    h.pop()
                    h.push(dis[j], int(ids[j]))
        D[i], I[i] = h.reorder()
    return D, I, key


def brute_force_fp64(ix, x, key, k):
    """Exhaustive fp64 <A x, centroid + decode(code)> over the probed lists; returns (D64, I) top-k."""
    xr = ix.A.astype(np.float64) @ np.asarray(x, dtype=np.float64).T        # [d, n]
    Cm = ix.centroids().astype(np.float64)
    pq = ix.pq.astype(np.float64)
    n = x.shape[0]
    D = np.full((n, k), -np.inf)
    I = np.full((n, k), -1, dtype=np.int64)
    for i in range(n):
        sc, idl = [], []
        for l in key[i]:
            l = int(l)
            if l < 0 or ix.list_len[l] == 0:
                continue
            codes = ix.list_codes(l)
            vec = pq[np.arange(ix.M)[None, :], codes.astype(np.int64)].reshape(len(codes), ix.d) + Cm[l][None, :]
            sc.append(vec @ xr[:, i])
            idl.append(ix.list_ids(l))
        if not sc:
            continue
        sc = np.concatenate(sc)
        idl = np.concatenate(idl)
        top = np.argsort(-sc, kind="stable")[:k]
        D[i, :len(top)] = sc[top]
        I[i, :len(top)] = idl[top]
    return D, I
