"""The slicing rule of a search over codes in host memory (DESIGN.md 3.5), restated in numpy.

Within one search chunk, the probed lists of the shard [lo, hi) are the non-empty lists some query probes.  Walking them in ascending
id, a resident list costs 0 blocks and any other list its block count ceil(len / 32); a new slice starts when the next list would
overflow the stream region's blocks.  Slice s covers [first probed list of s, first probed list of s + 1), the first one from lo and the
last one up to hi, and fetches its non-resident probed lists.  A chunk that probes nothing in the shard is one empty slice over [lo, hi).
The search is rejected when the region is smaller than the shard's largest non-resident list."""
import numpy as np


def blocks(list_len):
    return (np.asarray(list_len, dtype=np.int64) + 31) // 32


def np_slices(keys, list_len, resident, region_blocks, lo, hi):
    """keys [n, nprobe] (probed lists, -1 = none), list_len [nlist], resident: lists kept in device memory -> (slices, counts):
    slices = [(first list, end list, [fetched lists])], counts = [slices, lists fetched, blocks fetched, resident lists scanned]."""
    list_len = np.asarray(list_len, dtype=np.int64)
    nb = blocks(list_len)
    res = np.zeros(len(list_len), dtype=bool)
    res[np.asarray(list(resident), dtype=np.int64)] = True
    shard = np.arange(lo, hi)
    stream = shard[~res[lo:hi]]
    if len(stream) and nb[stream].max() > region_blocks:
        raise ValueError(f"the stream region holds {region_blocks} blocks; list {stream[nb[stream].argmax()]} needs {nb[stream].max()}")
    k = np.unique(np.asarray(keys, dtype=np.int64).ravel())
    probed = k[(k >= lo) & (k < hi)]
    probed = probed[list_len[probed] > 0]
    starts, fetched, used = [], [], 0
    for l in probed:
        cost = 0 if res[l] else int(nb[l])
        if not starts or used + cost > region_blocks:
            starts.append(lo if not starts else int(l))
            fetched.append([])
            used = 0
        if cost:
            fetched[-1].append(int(l))
            used += cost
    if not starts:
        starts, fetched = [lo], [[]]
    ends = starts[1:] + [hi]
    slices = list(zip(starts, ends, fetched))
    all_fetched = [l for f in fetched for l in f]
    counts = [len(slices), len(all_fetched), int(nb[all_fetched].sum()) if all_fetched else 0, int(res[probed].sum())]
    return slices, counts
