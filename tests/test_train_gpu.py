"""GPU: training a resident index (dph_index_train_coarse / dph_index_train_pq / IvfPqIndex.train) against the CPU oracle
(oracle/train_ref.c, DESIGN.md 3.3).  The coarse centroids and PQ codebooks are bit-identical after every iteration; a trained
index then adds, searches and round-trips through a faiss file like any other."""
import numpy as np
import pytest

from oracle import encode_ref as E
from oracle import train_ref as T
from tests.helpers import assert_topk_equal, opq_matrix

pytestmark = pytest.mark.gpu
SEED = 31


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def clustered_rows(n, groups, seed, A, spread=0.3):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((groups, 768)).astype(np.float32)
    return ((c[rng.integers(0, groups, n)] + spread * rng.standard_normal((n, 768))) @ A).astype(np.float32)


def handle(nlist, A, tc=True):
    from densephrases_b200 import IvfPqIndex
    ix = IvfPqIndex(nlist)
    ix.set_opq(A)
    ix.set_coarse_tc(tc)
    return ix


def check_coarse_chain(ix, x, A, nlist, niter, mppc=256, as_tensor=False):
    """niter hot-started one-iteration calls, each == the oracle's, then one full niter call == the oracle's full run."""
    import torch
    xin = torch.from_numpy(x).cuda() if as_tensor else x
    Cr = None
    for it in range(niter):
        obj, ns = ix.train_coarse(xin, niter=1, seed=SEED, max_points_per_centroid=mppc, hot_start=it > 0)
        Cr, objr, nsr = T.train_coarse(x, A, nlist, 1, SEED, mppc, C0=Cr)
        assert np.array_equal(bits(ix.centroids()), bits(Cr)), f"iteration {it}"
        assert np.array_equal(obj, objr) and np.array_equal(ns, nsr), f"iteration {it}: objective / splits"
    obj, ns = ix.train_coarse(xin, niter=niter, seed=SEED, max_points_per_centroid=mppc)
    Cf, objf, nsf = T.train_coarse(x, A, nlist, niter, SEED, mppc)
    assert np.array_equal(bits(ix.centroids()), bits(Cf)) and np.array_equal(obj, objf) and np.array_equal(ns, nsf), "full run"
    return nsf


@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("nlist", [1, 16, 256, 1024])              # 256, 1024: tensor-core candidates + exact re-rank when tc
def test_coarse_matches_oracle(nlist, tc):
    A = opq_matrix(SEED)
    x = clustered_rows(max(3 * nlist, 600), 40, nlist, A)
    ix = handle(nlist, A, tc)
    check_coarse_chain(ix, x, A, nlist, 3)
    check_coarse_chain(ix, x, A, nlist, 2, as_tensor=True)


def test_coarse_across_assignment_chunks_and_subsampled(monkeypatch):
    A = opq_matrix(SEED)
    x = clustered_rows(3000, 30, 5, A)
    monkeypatch.setenv("DPH_UPLOAD_CHUNK_ROWS", "97")              # 31 assignment / upload chunks
    check_coarse_chain(handle(256, A), x, A, 256, 2)
    monkeypatch.delenv("DPH_UPLOAD_CHUNK_ROWS")
    check_coarse_chain(handle(256, A), x, A, 256, 2, mppc=5)        # 3000 > 5 * 256: a ranked subsample of 1280 rows
    check_coarse_chain(handle(64, A), x, A, 64, 2, mppc=5, as_tensor=True)


def test_planted_split_matches_oracle():
    """Copies of a few rows make initial centroids coincide: empty clusters every side must split the same way."""
    A = opq_matrix(SEED)
    rng = np.random.default_rng(2)
    x = np.concatenate([np.repeat(rng.standard_normal((4, 768)), 150, 0), rng.standard_normal((40, 768))]).astype(np.float32)
    for tc in (True, False):
        nsplit = check_coarse_chain(handle(16, A, tc), x, A, 16, 3)
        assert nsplit.sum() > 0
    nsplit = check_coarse_chain(handle(256, A), np.concatenate([x, x[:200]]), A, 256, 2)
    assert nsplit.sum() > 0


@pytest.mark.parametrize("residual", [True, False])
def test_pq_matches_oracle(residual):
    import torch
    A = opq_matrix(SEED)
    x = clustered_rows(3000, 50, 9, A)
    ix = handle(64, A)
    ix.train_coarse(x, niter=2, seed=SEED)
    Cm = ix.centroids() if residual else None
    pqr = None
    for it, xin in enumerate((x, torch.from_numpy(x).cuda(), x)):      # init + 2 iterations, then hot-started single iterations
        ix.train_pq(xin, niter=2 if it == 0 else 1, seed=SEED, hot_start=it > 0, residual=residual)
        pqr = T.train_pq(x, A, Cm, 2 if it == 0 else 1, SEED, pq0=pqr)
        assert np.array_equal(bits(ix.pq_codebooks()), bits(pqr)), f"step {it}"
    ix.train_pq(x, niter=2, seed=SEED, max_points_per_centroid=4, residual=residual)        # 3000 > 4 * 256: subsampled
    assert np.array_equal(bits(ix.pq_codebooks()), bits(T.train_pq(x, A, Cm, 2, SEED, 4)))


def test_encode_pq_matches_oracle_argmin():
    import torch
    A = opq_matrix(SEED)
    x = clustered_rows(500, 10, 3, A)
    ix = handle(4, A)
    ix.train_pq(x, niter=2, seed=SEED, residual=False)
    pq = ix.pq_codebooks()
    _, ref = E.encode(A, np.zeros((1, 768), np.float32), pq, x)      # IVF1 with a zero centroid: the residual is xr itself
    assert np.array_equal(ix.encode_pq(x), ref)
    assert np.array_equal(ix.encode_pq(torch.from_numpy(x).cuda()).cpu().numpy(), ref)


@pytest.fixture(scope="module")
def trained():
    from tests.test_build_index import clustered
    x = clustered(6000, 1)
    from densephrases_b200 import IvfPqIndex
    ix = IvfPqIndex(16)
    info = ix.train(x[:3000], niter=6, niter_pq=8, opq_niter=2, seed=5)
    return x, ix, info


def test_full_train_properties_and_determinism(trained):
    from densephrases_b200 import IvfPqIndex
    x, ix, info = trained
    A = ix.opq_matrix()
    assert np.abs(A.astype(np.float64) @ A.T - np.eye(768)).max() < 1e-4
    assert ix.ntotal == 0 and len(info["obj"]) == 6
    again = IvfPqIndex(16)
    again.train(x[:3000], niter=6, niter_pq=8, opq_niter=2, seed=5)
    for a, b in ((A, again.opq_matrix()), (ix.centroids(), again.centroids()), (ix.pq_codebooks(), again.pq_codebooks())):
        assert np.array_equal(bits(a), bits(b))
    # everything downstream of A is the oracle's, bit for bit
    Cr, objr, _ = T.train_coarse(x[:3000], A, 16, 6, 5)
    assert np.array_equal(bits(ix.centroids()), bits(Cr)) and np.array_equal(info["obj"], objr)
    assert np.array_equal(bits(ix.pq_codebooks()), bits(T.train_pq(x[:3000], A, Cr, 8, 5)))


def test_train_add_search_and_faiss_file_round_trip(trained, tmp_path):
    from densephrases_b200 import IvfPqIndex, artifacts
    x, ix, _ = trained
    ix.add_with_ids(x, None)
    ix.nprobe = 8
    ref = E.GrowableRefIndex(ix.opq_matrix(), ix.pq_codebooks(), np.zeros(16, np.int64), centroids=ix.centroids())
    ref.add_with_ids(x)
    q = x[:48] + 0.05 * np.random.default_rng(9).standard_normal((48, 768)).astype(np.float32)
    D, I = ix.search(q, 10)
    Dr, Ir = ref.search(q, 10, 8)
    assert_topk_equal(D, I, Dr, Ir, "trained + added")
    lens, codes, ids = ix.lists()
    path = str(tmp_path / "trained.faiss")
    artifacts.write_faiss_index(path, ix.opq_matrix(), ix.centroids(), ix.pq_codebooks(), lens, codes, ids)
    back = artifacts.read_faiss_index(path)
    ix2 = IvfPqIndex.from_arrays(back["A"], back["centroids"], back["pq"], back["list_len"], back["codes"], back["ids"])
    ix2.nprobe = 8
    D2, I2 = ix2.search(q, 10)
    assert np.array_equal(bits(D2), bits(D)) and np.array_equal(I2, I)


def test_trained_recall_meets_torch_trainer(trained):
    """The clustered data of test_build_index: the GPU trainer meets that test's thresholds and is within 0.02 of the torch trainer's
    quality and recall on the same sample with the same iteration counts.  The torch trainer runs on one CPU thread: its QR and
    reductions round differently when split over threads, and on this sample that alone moves its recall by more than 0.01 (0.8275 on
    one thread, 0.84 on eight), so with the default thread count the reference would depend on the machine's core count."""
    import torch
    from densephrases_b200 import IvfPqIndex
    from densephrases_b200.build_index import build_index
    x, _, _ = trained
    rng = np.random.default_rng(3)
    q = x[rng.integers(0, len(x), 40)] + 0.05 * rng.standard_normal((40, 768)).astype(np.float32)
    ip = q.astype(np.float64) @ x.astype(np.float64).T
    exact = np.argsort(-ip, axis=1)[:, :10]

    def scores(I):
        top1 = np.mean([exact[i, 0] == I[i, 0] for i in range(40)])
        quality = np.mean([ip[i, I[i, :10]].mean() / ip[i, exact[i]].mean() for i in range(40)])
        recall = np.mean([len(set(I[i]) & set(exact[i])) / 10 for i in range(40)])
        return top1, quality, recall

    g = IvfPqIndex(16)
    g.train(x[:3000], niter=6, niter_pq=4, opq_niter=2, seed=5)
    g.add_with_ids(x, None)
    g.nprobe = 8
    gpu = scores(g.search(q, 50)[1])
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        t = build_index(x[:3000], x, nlist=16, seed=5, niter_opq=2, niter_km=6, niter_pq=4)
    finally:
        torch.set_num_threads(threads)
    ti = IvfPqIndex.from_arrays(t["A"], t["centroids"], t["pq"], t["list_len"], t["codes"], t["ids"])
    ti.nprobe = 8
    ref = scores(ti.search(q, 50)[1])
    assert gpu[0] > 0.9 and gpu[1] > 0.97 and gpu[2] > 0.6, gpu
    assert gpu[1] >= ref[1] - 0.02 and gpu[2] >= ref[2] - 0.02, (gpu, ref)


def test_refused_calls_leave_the_index_unchanged():
    import torch
    A = opq_matrix(SEED)
    x = clustered_rows(600, 10, 1, A)
    ix = handle(16, A)
    ix.train_coarse(x, niter=1, seed=SEED)
    ix.train_pq(x, niter=1, seed=SEED)

    def state():
        return ix.opq_matrix().tobytes(), ix.centroids().tobytes(), ix.pq_codebooks().tobytes()

    before = state()
    bad = x.copy()
    bad[7, 5] = np.nan
    for call in (lambda: ix.train_coarse(x[:10], niter=1),                        # n < nlist
                 lambda: ix.train_pq(x[:200], niter=1),                            # n < 256
                 lambda: ix.train_coarse(bad, niter=1),                            # non-finite
                 lambda: ix.train_pq(torch.from_numpy(bad).cuda(), niter=1),
                 lambda: ix.train_coarse(x[:0], niter=1)):
        with pytest.raises(RuntimeError):
            call()
        assert state() == before
    fresh = handle(16, A)
    from densephrases_b200 import IvfPqIndex
    no_opq = IvfPqIndex(16)
    with pytest.raises(RuntimeError):
        no_opq.train_coarse(x, niter=1)                                            # no OPQ matrix
    with pytest.raises(RuntimeError):
        fresh.train_pq(x, niter=1, residual=True)                                  # residuals without centroids
    ix.set_lists(np.array([1] + [0] * 15, np.int64), np.zeros((1, 96), np.uint8))
    with pytest.raises(RuntimeError):
        ix.train_coarse(x, niter=1)                                                # the index holds vectors
    assert state() == before
