"""The quad scan streams across work items: a warp that runs out of blocks prefetches the next item's first blocks, every warp loads its
first block of the next item before the candidates of the current one are published, and the packed tables are built from the compact
8-bit table source.  Many short lists give every CTA a long chain of items of one and two packed tables, lists probed by more than
eight queries split into several items, a few long lists split into block segments, and list lengths are not multiples of 32.
Results must equal the oracle bit for bit."""
import numpy as np
import pytest

from tests.helpers import assert_topk_equal, near_queries
from tests.test_search_gpu import make_pair

pytestmark = pytest.mark.gpu

NLIST, NPROBE, BATCH = 4096, 32, 512
SEG_BLOCKS = 128                          # shortest block segment of a split list (DPH_GROUP_SEG_MIN)


def test_quad_item_chains_match_oracle(oracle):
    rng = np.random.default_rng(11)
    lens = rng.integers(1, 900, NLIST).astype(np.int64)
    lens[rng.choice(NLIST, 12, replace=False)] = rng.integers(2 * SEG_BLOCKS * 32 + 1, 3 * SEG_BLOCKS * 32, 12)   # three segments
    ref, gpu = make_pair(oracle, NLIST, lens)
    gpu.nprobe = NPROBE
    gpu.set_scan_mode(4)                  # quad-packed gathers although the lists are short
    x = near_queries(ref, BATCH, 2024)
    for k in (10, 40):
        D, I = gpu.search(x, k)
        assert gpu.last_group_size() == 4
        counts = np.bincount(gpu.last_probes(BATCH).ravel(), minlength=NLIST)
        assert (counts[(counts >= 1) & (counts <= 4)].size > 0 and counts[(counts >= 5) & (counts <= 8)].size > 0
                and counts[counts > 8].size > 0), "one-table, two-table and split items"
        assert (counts[lens > 2 * SEG_BLOCKS * 32] > 0).any(), "a list cut into block segments is probed"
        Dr, Ir = ref.search(x, k, NPROBE)
        assert_topk_equal(D, I, Dr, Ir, f"quad item chains k={k}")
        assert not gpu.last_flags(BATCH).any()
