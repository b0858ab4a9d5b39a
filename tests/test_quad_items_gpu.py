"""Quad-mode work items of up to eight queries: one code read runs through one packed table (<= 4 probing queries) or two
(5-8), and lists probed by more than eight queries are split into several items.  Results must equal the oracle bit for bit."""
import numpy as np
import pytest

from tests.helpers import assert_topk_equal, near_queries, uniform_lens
from tests.test_search_gpu import make_pair

pytestmark = pytest.mark.gpu

# probing queries per list: one-table items (1, 4), two-table items (5, 8), a list split into 8 + 1 (9) and into 8 + 8 + 1 (17)
COUNTS = (1, 4, 5, 8, 9, 17)


def queries_with_probe_counts(ref, nlist, counts, seed):
    """A batch whose top-1 lists (nprobe = 1) are probed by exactly `counts` queries; the most popular lists get the largest counts."""
    pool = near_queries(ref, 40 * nlist * max(counts), seed)
    _, key = ref.coarse(ref.rotate(pool), 1)
    top1 = key[:, 0]
    popular = np.argsort(-np.bincount(top1, minlength=nlist), kind="stable")
    picks = []
    for lst, c in zip(popular, sorted(counts, reverse=True)):
        rows = np.flatnonzero(top1 == lst)
        assert len(rows) >= c, "query pool too small for the probe counts"
        picks.append(rows[:c])
    return pool[np.sort(np.concatenate(picks))]


def test_quad_items_of_one_and_two_tables_and_split_lists(oracle):
    nlist = 8
    lens = uniform_lens(nlist * 4500, nlist)
    ref, gpu = make_pair(oracle, nlist, lens)
    gpu.nprobe = 1
    x = queries_with_probe_counts(ref, nlist, COUNTS, 77)
    n = len(x)
    for k in (10, 40):
        D, I = gpu.search(x, k)
        assert gpu.last_group_size() == 4
        counts = np.bincount(gpu.last_probes(n)[:, 0], minlength=nlist)
        assert sorted(counts[counts > 0].tolist()) == sorted(COUNTS)
        Dr, Ir = ref.search(x, k, 1)
        assert_topk_equal(D, I, Dr, Ir, f"quad items k={k}")
        assert not gpu.last_flags(n).any()
    D, I = gpu.search(x, 300)                  # k + slack no longer fits the quad buffers -> pair-packed
    assert gpu.last_group_size() == 2
    assert_topk_equal(D, I, *ref.search(x, 300, 1), "pair fallback")
