"""tests/filter_ref.py -- the definition of the filtered search (DESIGN.md 3.6), restated in numpy.

The filtered result is the unfiltered canonical ranking of every probed row -- score descending, then scan position ascending (probe
rank, then the row's place in its list) -- restricted to the selected rows and cut at k; missing slots are (-FLT_MAX, -1).  Scores use
the oracle's floating-point order (dis = dis0; for m ascending: dis += LUT[m][c[m]], fp32).  The row mask of a shard [lo, hi) holds one
uint32 per 32-row code block, the lists' blocks packed in list order, bit j % 32 of the list's block j // 32 = row j is selected.
"""
import numpy as np

from oracle import ivfpq_ref as R

NEG = np.float32(-3.4028234663852886e38)


def np_filtered_search(ref, x, k, nprobe, selected):
    """RefIndex ref, selected [ntotal] (list-major rows) -> (D [n,k] f32, I [n,k] i64, key [n,nprobe])."""
    xr = ref.rotate(x)
    _, key = ref.coarse(xr, nprobe)
    Cm = ref.centroids()
    lab = ref.ids if ref.ids is not None else np.arange(ref.ntotal, dtype=np.int64)
    n = len(xr)
    D = np.full((n, k), NEG, dtype=np.float32)
    I = np.full((n, k), -1, dtype=np.int64)
    for i in range(n):
        lut = R.np_lut(xr[i], ref.pq)
        scores, rows = [], []
        for l in key[i]:
            l = int(l)
            if l < 0 or ref.list_len[l] == 0:
                continue
            dis0 = R.np_matmul_nt_seq(xr[i:i + 1], Cm[l:l + 1])[0, 0]
            codes = ref.list_codes(l)
            dis = np.full(len(codes), dis0, dtype=np.float32)
            for m in range(ref.M):
                dis = (dis + lut[m, codes[:, m]]).astype(np.float32)
            scores.append(dis)
            rows.append(ref.list_off[l] + np.arange(len(codes)))
        if not scores:
            continue
        scores, rows = np.concatenate(scores), np.concatenate(rows)
        order = np.argsort(-scores.astype(np.float64), kind="stable")          # the canonical ranking of all probed rows
        order = order[np.asarray(selected, bool)[rows[order]]][:k]              # restricted, cut
        D[i, :len(order)] = scores[order]
        I[i, :len(order)] = lab[rows[order]]
    return D, I, key


def np_mask(list_len, selected, lo=0, hi=None):
    """selected [ntotal] (list-major rows of ALL lists) -> uint32 [blocks of lists lo..hi-1] (the shard's mask)."""
    list_len = np.asarray(list_len, dtype=np.int64)
    hi = len(list_len) if hi is None else hi
    off = np.concatenate([[0], np.cumsum(list_len)])
    words = []
    for l in range(lo, hi):
        nb = (int(list_len[l]) + 31) // 32
        bits = np.zeros(nb * 32, dtype=np.uint64)
        bits[:list_len[l]] = np.asarray(selected[off[l]:off[l + 1]], dtype=np.uint64) != 0
        words.append((bits.reshape(nb, 32) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32))
    return np.concatenate(words + [np.zeros(0, np.uint32)])
