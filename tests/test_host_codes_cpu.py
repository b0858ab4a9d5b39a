"""CPU: the slicing rule of a search over codes in host memory (tests/host_codes_ref.py, DESIGN.md 3.5) on hand examples."""
import numpy as np
import pytest

from tests.host_codes_ref import np_slices

# blocks per list: 0 (empty), 1, 2, 3, 1, 4, 0, 2
LENS = np.array([0, 32, 33, 96, 1, 128, 0, 64])


def test_every_probed_list_in_one_slice_in_order():
    keys = np.array([[1, 2, 3], [5, 7, -1]])
    slices, counts = np_slices(keys, LENS, [], 4, 0, 8)
    assert slices == [(0, 3, [1, 2]), (3, 5, [3]), (5, 7, [5]), (7, 8, [7])]
    assert counts == [4, 5, 12, 0]


def test_empty_lists_are_not_probed():
    slices, counts = np_slices(np.array([[0, 6, 4]]), LENS, [], 4, 0, 8)
    assert slices == [(0, 8, [4])] and counts == [1, 1, 1, 0]


def test_resident_lists_cost_nothing_inside_and_between_slices():
    keys = np.array([[1, 2, 3, 5, 7]])
    # 3 resident inside the first slice; 5 resident where a slice boundary would fall without it
    slices, counts = np_slices(keys, LENS, [3, 5], 4, 0, 8)
    assert slices == [(0, 7, [1, 2]), (7, 8, [7])]
    assert counts == [2, 3, 5, 2]
    # a slice made only of resident lists fetches nothing
    slices, counts = np_slices(np.array([[5, 3]]), LENS, [3, 5], 2, 0, 8)
    assert slices == [(0, 8, [])] and counts == [1, 0, 0, 2]


def test_list_exactly_the_region_size():
    slices, counts = np_slices(np.array([[5, 4]]), LENS, [], 4, 0, 8)
    assert slices == [(0, 5, [4]), (5, 8, [5])] and counts == [2, 2, 5, 0]


def test_list_larger_than_the_region_is_an_error():
    with pytest.raises(ValueError):
        np_slices(np.array([[1]]), LENS, [], 3, 0, 8)          # list 5 (4 blocks) is not resident, even though it is not probed
    np_slices(np.array([[1]]), LENS, [5], 3, 0, 8)              # resident: fine


def test_chunk_that_probes_nothing_in_the_shard():
    slices, counts = np_slices(np.array([[0, 1, 7], [-1, -1, -1]]), LENS, [], 4, 2, 6)
    assert slices == [(2, 6, [])] and counts == [1, 0, 0, 0]


def test_shard_range_first_and_last_slice():
    slices, _ = np_slices(np.array([[3, 4, 5, 1, 7]]), LENS, [], 4, 2, 6)
    assert slices == [(2, 5, [3, 4]), (5, 6, [5])]


def test_random_partition_properties():
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 300, 200) * (rng.random(200) < 0.7)
    for t in range(20):
        keys = rng.integers(-1, 200, (8, 16))
        res = rng.choice(200, 30, replace=False)
        region = int(((lens + 31) // 32).max()) + t
        slices, counts = np_slices(keys, lens, res, region, 0, 200)
        assert slices[0][0] == 0 and slices[-1][1] == 200
        assert all(a[1] == b[0] for a, b in zip(slices, slices[1:]))
        fetched = [l for s in slices for l in s[2]]
        assert fetched == sorted(set(fetched)) and not set(fetched) & set(res.tolist())
        for lo, hi, f in slices:
            assert all(lo <= l < hi for l in f) and sum((lens[l] + 31) // 32 for l in f) <= region
        assert counts[:2] == [len(slices), len(fetched)]
