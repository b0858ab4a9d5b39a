"""The search at its arithmetic limits, against the C oracle: saturated packed sums, worst-case LUT rounding, extreme query scales,
batches over several chunks, batch invariance at C2's list length and the k edges of the scan modes.  Scores are compared bit for
bit, labels up to exact-tie groups (tests/helpers.py)."""
import numpy as np
import pytest

from tests.helpers import assert_topk_equal, near_queries, uniform_lens
from tests.test_search_gpu import make_pair
from tests.test_search_limits_cpu import (QMAX, keep_pair, keep_quad, rounding_case, saturated_codes, saturating_codebooks,
                                          limit_query)

pytestmark = pytest.mark.gpu
EYE = np.eye(768, dtype=np.float32)


def assert_probes_equal(pr, cd, keyr, cdr, what=""):
    """Coarse scores bit for bit; probe lists equal as sets above the last score of each row, and as counts at that score (which
    lists tie at the nprobe boundary is heap-dependent in the oracle and canonical, smallest list id first, on the GPU)."""
    assert np.array_equal(cd.view(np.int32), cdr.view(np.int32)), f"{what}: coarse scores differ"
    for r in range(len(pr)):
        if np.array_equal(pr[r], keyr[r]):
            continue
        last = cd[r, -1]
        assert set(pr[r][cd[r] > last].tolist()) == set(keyr[r][cdr[r] > last].tolist()), f"{what}: row {r} probes differ"
        assert np.sum(cd[r] == last) == np.sum(cdr[r] == last), f"{what}: row {r} boundary tie size"


# ---- 1. saturated packed sums -------------------------------------------------------------------------------------------
SAT_NLIST, SAT_LEN, SAT_POS = 4, 4100, (7, 2100, 4099)      # long enough lists for the auto mode to pick the quad scan


def saturated_index(oracle, x, pq, seed=21):
    """IVF4 with A = I and random codes; every list holds the saturated code of x and its one- and two-byte variants."""
    from densephrases_b200 import IvfPqIndex
    lens = np.full(SAT_NLIST, SAT_LEN, dtype=np.int64)
    Cm = oracle.gen_centroids(seed, 0, SAT_NLIST)
    codes = np.concatenate([oracle.gen_codes(seed, l, 0, SAT_LEN) for l in range(SAT_NLIST)])
    sat = saturated_codes(x, pq)
    for l in range(SAT_NLIST):
        for row, p in zip(sat, SAT_POS):
            codes[l * SAT_LEN + p] = row
    ref = oracle.RefIndex(EYE, pq, lens, centroids=Cm, codes=codes)
    gpu = IvfPqIndex.from_arrays(EYE, Cm, pq, lens, codes)
    gpu.nprobe = 2
    return ref, gpu, {l * SAT_LEN + SAT_POS[0] for l in range(SAT_NLIST)}


@pytest.mark.parametrize("codebooks", ["equal_ranges", "generated"])
def test_saturated_codes_every_lane(oracle, codebooks):
    """4 and 8 copies of one query probe the same two lists: every byte lane of the quad words (one table, then two) and both u16
    lanes of the pair words carry the largest sum at once.  A carry across lanes would drop the saturated vector before the merge,
    where the proof cannot see it; the results must equal the oracle's, whose top-1 is the saturated vector."""
    x = limit_query(3)
    pq = saturating_codebooks(x, 4) if codebooks == "equal_ranges" else oracle.gen_pq(1234)
    ref, gpu, sat_labels = saturated_index(oracle, x, pq)
    k = 10
    for copies in (4, 8):
        q = np.repeat(x[None], copies, axis=0)
        Dr, Ir = ref.search(q, k, 2)
        assert set(Ir[:, 0].tolist()) <= sat_labels
        for mode in (2, 4, 0):
            gpu.set_scan_mode(mode)
            D, I = gpu.search(q, k)
            assert gpu.last_group_size() == (2 if mode == 2 else 4)
            assert_topk_equal(D, I, Dr, Ir, f"{codebooks} copies={copies} mode={mode}")


# ---- 2. worst-case LUT rounding -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dropped", [False, True])
@pytest.mark.parametrize("group,k", [(4, 1), (4, 10), (4, 85), (2, 86), (2, 300)])
def test_worst_case_rounding(oracle, group, k, dropped):
    """One list: a target whose exact score is 18 steps above that of its identical competitors, but whose quantised score is 74
    steps below theirs (tests/test_search_limits_cpu.py: rounding_case).
      * dropped: keep + 1 competitors push the target out of the scan's candidate buffer; the proof must flag the query, and the
        exact re-run finds it;
      * kept: k competitors; the target stays a candidate and eps must be large enough for the merge to re-score it.  The proof
        passes there (nothing was dropped), so the filter's own answer has to be right."""
    from densephrases_b200 import IvfPqIndex
    x, pq, target, comp = rounding_case(group)
    keep = keep_quad(k) if group == 4 else keep_pair(k)
    ncomp = keep + 1 if dropped else k
    pos = ncomp // 2
    codes = np.insert(np.repeat(comp[None], ncomp, axis=0), pos, target, axis=0)
    lens = np.array([len(codes)], dtype=np.int64)
    Cm = np.zeros((1, 768), dtype=np.float32)
    ref = oracle.RefIndex(EYE, pq, lens, centroids=Cm, codes=codes)
    gpu = IvfPqIndex.from_arrays(EYE, Cm, pq, lens, codes)
    gpu.nprobe = 1
    gpu.set_scan_mode(group)
    Dr, Ir = ref.search(x[None], k, 1)
    assert Ir[0, 0] == pos
    D, I = gpu.search(x[None], k)
    assert gpu.last_group_size() == group
    assert_topk_equal(D, I, Dr, Ir, f"group={group} k={k} dropped={dropped}")
    assert gpu.last_flags(1)[0] == (1 if dropped else 0)


# ---- 3. extreme and degenerate queries ----------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [-120, -100, -60, 0, 40, 100])
def test_extreme_query_scales(oracle, scale):
    """Queries scaled by 2^scale (every value stays finite; at 2^-120 the 3xTF32 split parts and products of the tensor-core coarse
    quantizer are subnormal), the all-zero query (every coarse and scan score ties), a query equal to a centroid and four copies of
    one query (one quad item): probes, coarse scores and top-k equal the oracle in every scan mode, on both coarse paths."""
    nlist, nprobe, k = 256, 16, 10
    ref, gpu = make_pair(oracle, nlist, np.full(nlist, 40, dtype=np.int64))
    gpu.nprobe = nprobe
    base = near_queries(ref, 34, 31)
    x = np.concatenate([base, np.zeros((1, 768), np.float32), ref.centroids()[5:6] @ ref.A, np.repeat(base[:1], 4, axis=0)])
    x = np.ldexp(x, scale).astype(np.float32)
    assert np.isfinite(x).all()
    n = len(x)
    Dr, Ir, keyr = ref.search(x, k, nprobe, return_key=True)
    cdr, _ = ref.coarse(ref.rotate(x), nprobe)
    for tc in (1, 0):
        gpu.set_coarse_tc(tc)
        for mode in (1, 3, 2, 4, 0):
            gpu.set_scan_mode(mode)
            D, I = gpu.search(x, k)
            what = f"2^{scale} tc={tc} mode={mode}"
            assert np.array_equal(gpu.last_xr(n).view(np.int32), ref.rotate(x).view(np.int32)), what
            assert_probes_equal(gpu.last_probes(n), gpu.last_coarse(n), keyr, cdr, what)
            assert_topk_equal(D, I, Dr, Ir, what)


@pytest.mark.parametrize("scale", [-100, -120])
def test_tensor_core_coarse_proof_at_tiny_scale(oracle, scale):
    """Near-identical centroids put the 3xTF32 candidate scores inside their error bound c |xr| max|C|, so the proof must send every
    query to the repair path, at any scale.  At |xr| ~ 2^-96 the squares of xr's elements underflow in fp32; a norm computed from
    them is 0, the bound collapses to 0 and the proof would accept candidates ranked by approximate scores."""
    from densephrases_b200 import IvfPqIndex
    from tests.helpers import opq_matrix
    nlist, nprobe = 256, 16
    rng = np.random.default_rng(4)
    lens = np.full(nlist, 30, dtype=np.int64)
    A, pq = opq_matrix(4), oracle.gen_pq(4)
    Cm = (oracle.gen_centroids(4, 0, 1) + 1e-6 * rng.standard_normal((nlist, 768))).astype(np.float32)
    codes = np.concatenate([oracle.gen_codes(4, l, 0, 30) for l in range(nlist)])
    ref = oracle.RefIndex(A, pq, lens, centroids=Cm, codes=codes)
    gpu = IvfPqIndex.from_arrays(A, Cm, pq, lens, codes)
    gpu.nprobe = nprobe
    x = np.ldexp(near_queries(ref, 48, 6), scale).astype(np.float32)
    out = {}
    for tc in (1, 0):
        gpu.set_coarse_tc(tc)
        D, I = gpu.search(x, 10)
        out[tc] = (gpu.last_probes(48).copy(), gpu.last_coarse(48).copy(), D, I)
    cdr, _ = ref.coarse(ref.rotate(x), nprobe)
    assert np.array_equal(out[0][1].view(np.int32), cdr.view(np.int32))
    assert np.array_equal(out[1][1].view(np.int32), out[0][1].view(np.int32)), "tensor-core coarse scores differ from the exact path"
    assert np.array_equal(out[1][0], out[0][0]), "tensor-core probes differ from the exact path"
    assert np.array_equal(out[1][2].view(np.int32), out[0][2].view(np.int32)) and np.array_equal(out[1][3], out[0][3])


# ---- 4. batches and chunks ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 4])
def test_batch_over_three_chunks(oracle, mode):
    """2 * 4096 + 17 queries on IVF64: the search runs three chunks of at most 4096 queries; every row equals the oracle, from host
    and from device memory."""
    import torch
    nlist, nprobe, k = 64, 8, 10
    ref, gpu = make_pair(oracle, nlist, uniform_lens(nlist * 300, nlist))
    gpu.nprobe = nprobe
    gpu.set_scan_mode(mode)
    x = near_queries(ref, 2 * 4096 + 17, 9)
    Dr, Ir = ref.search(x, k, nprobe)
    D, I = gpu.search(x, k)
    assert_topk_equal(D, I, Dr, Ir, f"host mode={mode}")
    Dd, Id = gpu.search(torch.from_numpy(x).cuda(), k)
    assert np.array_equal(Dd.cpu().numpy().view(np.int32), D.view(np.int32)) and np.array_equal(Id.cpu().numpy(), I)


def test_k_edges_in_every_mode(oracle):
    """k on both sides of the quad (85 / 86) and pair (683 / 684) limits and at the maximum, in every forced mode."""
    nlist, nprobe = 16, 4
    ref, gpu = make_pair(oracle, nlist, uniform_lens(nlist * 4500, nlist))
    gpu.nprobe = nprobe
    x = near_queries(ref, 12, 17)
    for k in (1, 85, 86, 683, 684, 1024):
        Dr, Ir = ref.search(x, k, nprobe)
        for mode in (1, 3, 2, 4):
            gpu.set_scan_mode(mode)
            D, I = gpu.search(x, k)
            if mode != 1:
                want = {3: 1, 2: 2 if k <= 683 else 1, 4: 4 if k <= 85 else (2 if k <= 683 else 1)}[mode]
                assert gpu.last_group_size() == want, f"k={k} mode={mode}"
            assert_topk_equal(D, I, Dr, Ir, f"k={k} mode={mode}")


def test_batch_invariance_at_c2_list_length(oracle):
    """IVF4096 over 20 M synthetic rows (C2's list length), nprobe 256: a batch of 1024 queries runs the quad scan, each of 32 of
    them searched alone runs the one-query scan; both orders are canonical, so scores and labels are byte-identical, tie order
    included; 16 rows are checked against the oracle."""
    import torch
    nlist, nprobe, k = 4096, 256, 10
    ref, gpu = make_pair(oracle, nlist, uniform_lens(20_000_000, nlist))
    gpu.nprobe = nprobe
    x = near_queries(ref, 1024, 41)
    xt = torch.from_numpy(x).cuda()
    D, I = gpu.search(xt, k)
    assert gpu.last_group_size() == 4
    D, I = D.cpu().numpy(), I.cpu().numpy()
    rng = np.random.default_rng(2)
    for r in rng.choice(1024, 32, replace=False):
        D1, I1 = gpu.search(xt[r:r + 1].contiguous(), k)
        assert gpu.last_group_size() == 1
        assert np.array_equal(D1.cpu().numpy()[0].view(np.int32), D[r].view(np.int32)) and np.array_equal(I1.cpu().numpy()[0], I[r]), f"row {r}"
    rows = np.sort(rng.choice(1024, 16, replace=False))
    Dr, Ir = ref.search(x[rows], k, nprobe)
    assert_topk_equal(D[rows], I[rows], Dr, Ir, "C2 lists")
