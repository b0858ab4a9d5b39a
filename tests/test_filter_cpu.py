"""CPU: the filtered search's definition (DESIGN.md 3.6).  The C oracle (oracle/filter_ref.c) equals the numpy restatement
(tests/filter_ref.py) bit for bit; selecting every row gives the unfiltered oracle; the selectors follow remove_ids' rules; MIPS maps
documents to labels and never returns a hit outside its document filter."""
import numpy as np
import pytest

from oracle import filter_ref as FR
from oracle import remove_ref as RR
from tests.filter_ref import np_filtered_search, np_mask
from tests.helpers import assert_topk_equal, near_queries, opq_matrix

SEED = 31


def ragged_ref(oracle, nlist=12, explicit=True, dup=True, seed=SEED):
    """Lists with empty ones, short ones and one over two blocks; explicit labels (one label on two rows when dup) or sequential."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 70, nlist)
    lens[[1, 5]] = 0
    lens[3] = 1
    N = int(lens.sum())
    codes = rng.integers(0, 256, (N, 96)).astype(np.uint8)
    ids = None
    if explicit:
        ids = rng.permutation(10 * N)[:N].astype(np.int64) + 1000
        if dup:
            ids[-1] = ids[0]                     # one label on two rows of different lists
    return oracle.RefIndex(opq_matrix(seed), oracle.gen_pq(seed), lens, centroids=oracle.gen_centroids(seed, 0, nlist), codes=codes, ids=ids)


def selectors(ref):
    lab = FR.labels(ref)
    rng = np.random.default_rng(1)
    s = np.sort(lab)
    return {
        "half": rng.choice(lab, len(lab) // 2, replace=False),
        "tenth": np.concatenate([rng.choice(lab, max(len(lab) // 10, 1), replace=False), [-1, -7, 10**12]]),
        "one": lab[:1],
        "range": range(int(s[len(s) // 4]), int(s[3 * len(s) // 4])),
        "none": np.zeros(0, np.int64),
        "empty_range": range(5, 5),
    }


@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("nprobe", [1, 4, 12])
@pytest.mark.parametrize("k", [1, 10, 100])
def test_oracle_equals_numpy_restatement(oracle, explicit, nprobe, k):
    ref = ragged_ref(oracle, explicit=explicit)
    x = near_queries(ref, 6, SEED)
    for name, sel in selectors(ref).items():
        for exclude in (False, True):
            selected = FR.selected_rows(ref, sel, exclude)
            D, I, key = FR.search(ref, x, k, nprobe, selected)
            Dn, In, keyn = np_filtered_search(ref, x, k, nprobe, selected)
            assert np.array_equal(key, keyn)
            assert_topk_equal(D, I, Dn, In, f"{name} exclude={exclude}")
            lab = FR.labels(ref)
            assert np.isin(I[I >= 0], lab[selected.astype(bool)]).all(), name


@pytest.mark.parametrize("explicit", [True, False])
def test_selecting_everything_is_the_unfiltered_search(oracle, explicit):
    ref = ragged_ref(oracle, explicit=explicit)
    x = near_queries(ref, 8, SEED + 1)
    for k, nprobe in ((10, 4), (100, 12)):
        D0, I0 = ref.search(x, k, nprobe)
        everything = np.ones(ref.ntotal, np.uint8)
        Dn, In, _ = np_filtered_search(ref, x, k, nprobe, everything)
        D, I, _ = FR.search(ref, x, k, nprobe, everything)
        assert_topk_equal(Dn, In, D0, I0, "numpy, all selected")
        assert_topk_equal(D, I, D0, I0, "oracle, all selected")
        # the exclude form of an empty selector is everything, an empty selector nothing
        assert np.array_equal(FR.selected_rows(ref, np.zeros(0, np.int64), exclude=True), everything)
        Dz, Iz, _ = FR.search(ref, x, k, nprobe, FR.selected_rows(ref, range(0, 0)))
        assert (Iz == -1).all() and (Dz.view(np.int32) == np.float32(-3.4028234663852886e38).view(np.int32)).all()


def test_selected_rows_are_the_rows_remove_ids_removes(oracle):
    """A row is selected exactly when remove_ids would remove it (label set with duplicates, absent and negative labels; ranges)."""
    for explicit in (True, False):
        ref = ragged_ref(oracle, explicit=explicit)
        for name, sel in selectors(ref).items():
            rm = RR.RemovableRefIndex(ref.A, ref.pq, ref.list_len, centroids=ref.C, codes=ref.codes, ids=ref.ids)
            before = FR.labels(rm).copy()
            rm.remove_ids(sel)
            kept = FR.labels(rm)
            selected = FR.selected_rows(ref, sel).astype(bool)
            assert int(selected.sum()) == len(before) - len(kept), name
            assert sorted(before[~selected].tolist()) == sorted(kept.tolist()), name


def test_selector_rejections_match_remove_ids():
    """make_filter parses its selector with remove_ids' code: the same forms are accepted and the same ones rejected."""
    from densephrases_b200.ivfpq import IvfPqIndex
    ix = object.__new__(IvfPqIndex)          # the parser needs no device
    for what in ("remove_ids", "make_filter"):
        args, keep = ix._selector(range(3, 9), what)
        assert args[0] is None and args[1:4] == (0, 3, 9) and keep is None
        args, keep = ix._selector(range(-2**70, 2**70), what)
        assert args[2:4] == (-2**63, 2**63 - 1)
        args, keep = ix._selector(np.array([[5, 3], [3, -1]], np.int64), what)
        assert args[1] == 4 and keep.tolist() == [5, 3, 3, -1]
        with pytest.raises(ValueError, match=f"{what}: a range selector must have step 1"):
            ix._selector(range(0, 10, 2), what)
        with pytest.raises(TypeError, match=f"{what}: labels must be int64"):
            ix._selector(np.arange(3, dtype=np.int32), what)
        with pytest.raises(TypeError, match=what):
            ix._selector([1, 2, 3], what)


def test_mask_layout():
    lens = np.array([0, 33, 1, 64, 0, 5])
    selected = np.zeros(int(lens.sum()), np.uint8)
    selected[[0, 32, 33, 34, 97, 98, 102]] = 1      # list 1 rows 0 and 32, list 2 row 0, list 3 rows 0 and 63, list 5 rows 0, 4
    m = np_mask(lens, selected)
    assert m.tolist() == [1, 1, 1, 1, 1 << 31, 1 | (1 << 4)]
    assert np_mask(lens, selected, 3, 6).tolist() == [1, 1 << 31, 1 | (1 << 4)]


# ---- MIPS restricted to documents ------------------------------------------------------------------------------------------
def synthetic_idx2id(groups, rng, ndocs=9):
    """{str(offset): {'doc', 'word'}} with several offset groups (labels offset + row, offset a multiple of 1e9)."""
    return {str(int(g * 1e9)): {'doc': rng.integers(0, ndocs, n).astype(np.int32), 'word': rng.integers(0, 50, n).astype(np.int32)}
            for g, n in enumerate(groups)}


class FilterIndexStandIn:
    """The slice of the index API MIPS uses, over explicit labels: make_filter keeps the selected labels; search returns the best
    selected labels of a fixed score table, padding with (-FLT_MAX, -1) when fewer are selected (short results)."""

    def __init__(self, labels, seed):
        self.labels = np.asarray(labels, np.int64)
        self.ntotal = int(self.labels.max()) + 1
        self.d = 4
        self.nprobe = 256
        self.rng = np.random.default_rng(seed)

    def opq_matrix(self):
        return np.eye(self.d, dtype=np.float32)

    def reconstruct_batch(self, ids):
        return np.zeros((len(ids), self.d), np.float32), np.zeros(len(ids), np.uint8)

    def make_filter(self, sel, exclude=False):
        return np.isin(self.labels, np.asarray(sel, np.int64)) != exclude

    def search(self, x, k, filter=None):
        n = len(x)
        keep = np.ones(len(self.labels), bool) if filter is None else filter
        D = np.full((n, k), np.float32(-3.4028234663852886e38), np.float32)
        I = np.full((n, k), -1, np.int64)
        for i in range(n):
            cand = self.labels[keep]
            s = self.rng.standard_normal(len(cand)).astype(np.float32)
            top = np.argsort(-s, kind="stable")[:k]
            D[i, :len(top)], I[i, :len(top)] = s[top], cand[top]
        return D, I


def test_doc_filter_labels_match_brute_force():
    from densephrases_b200.mips import MIPS
    rng = np.random.default_rng(5)
    idx_f = synthetic_idx2id([40, 7, 0, 25], rng)
    labels = np.concatenate([int(g) + np.arange(len(t['doc'])) for g, t in idx_f.items()])
    mips = MIPS.from_components(FilterIndexStandIn(labels, 0), idx_f, None, cuda=False, index_path='synthetic_PQ')
    for docs in ([3], [0, 4, 4, 8], [], [100]):
        want = [int(g) + r for g, t in idx_f.items() for r in range(len(t['doc'])) if int(t['doc'][r]) in docs]
        for exclude in (False, True):
            got = mips.doc_filter(docs, exclude=exclude)
            assert np.array_equal(labels[got], np.sort([l for l in labels if (l in want) != exclude]).astype(np.int64)), (docs, exclude)


@pytest.mark.parametrize("exclude", [False, True])
def test_mips_doc_filter_never_returns_another_document(exclude):
    from densephrases_b200.mips import MIPS
    rng = np.random.default_rng(6)
    idx_f = synthetic_idx2id([60, 30], rng, ndocs=6)
    labels = np.concatenate([int(g) + np.arange(len(t['doc'])) for g, t in idx_f.items()])
    stand_in = FilterIndexStandIn(labels, 1)
    mips = MIPS.from_components(stand_in, idx_f, None, cuda=False, index_path='synthetic_PQ')
    docs = [1] if not exclude else [0, 2, 3, 4, 5]            # either way only document 1's phrases (few: short results)
    f = mips.doc_filter(docs, exclude=exclude)
    doc_of = {int(g) + r: int(t['doc'][r]) for g, t in idx_f.items() for r in range(len(t['doc']))}
    n1 = sum(1 for v in doc_of.values() if v == 1)
    top_k = n1 + 5                                             # more slots than selected phrases: padded slots
    query = rng.standard_normal((3, 2 * stand_in.d)).astype(np.float32)
    s_doc, s_word, s_lab, e_doc, e_word, e_lab, s_sc, e_sc = mips.search_dense(query, ['q'] * 3, top_k=top_k, doc_filter=f)
    for doc, lab in ((s_doc, s_lab), (e_doc, e_lab)):
        assert (lab < 0).any()
        assert (doc[lab < 0] == -1).all()
        assert (doc[lab >= 0] == 1).all()
        assert all(doc_of[int(l)] == 1 for l in lab[lab >= 0])
    # without the filter, get_idxs maps a padded slot to label 0's document, which the filter would not allow
    s_doc0, _ = mips.get_idxs(np.array([[-1]]))
    assert s_doc0[0, 0] == doc_of[0]
