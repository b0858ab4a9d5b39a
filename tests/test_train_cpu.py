"""CPU: the training definition of DESIGN.md 3.3 (oracle/train_ref.c) against its numpy restatement, a split checked by hand, and
the properties a trained quantizer must have (unit-norm coarse centroids, falling PQ distortion, a sample that depends only on
(seed, n))."""
import numpy as np
import pytest

from oracle import train_ref as T

D = 16                                   # small geometry: the oracle takes any d (PQ: M = 2 sub-quantizers of 8)


def rot(seed, d=D):
    return np.linalg.qr(np.random.default_rng(seed).standard_normal((d, d)))[0].astype(np.float32)


def data(n, seed, d=D, groups=6):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((groups, d))
    return (c[rng.integers(0, groups, n)] + 0.3 * rng.standard_normal((n, d))).astype(np.float32)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


@pytest.mark.parametrize("n,k,mppc", [(200, 8, 256), (300, 8, 20), (40, 40, 256)])     # all rows; a subsample; n == k
def test_coarse_c_equals_numpy(n, k, mppc):
    x, A = data(n, n), rot(1)
    Cc, oc, sc = T.train_coarse(x, A, k, 4, seed=3, max_points_per_centroid=mppc)
    Cn, on, sn = T.np_train_coarse(x, A, k, 4, seed=3, max_points_per_centroid=mppc)
    assert np.array_equal(bits(Cc), bits(Cn)) and np.array_equal(oc, on) and np.array_equal(sc, sn)
    # hot start continues from the given table: one more iteration on both sides
    Ch, _, _ = T.train_coarse(x, A, k, 1, seed=3, max_points_per_centroid=mppc, C0=Cc)
    Chn, _, _ = T.np_train_coarse(x, A, k, 1, seed=3, max_points_per_centroid=mppc, C0=Cn)
    assert np.array_equal(bits(Ch), bits(Chn))


@pytest.mark.parametrize("residual", [True, False])
def test_pq_c_equals_numpy(residual):
    x, A = data(400, 7), rot(2)
    Cm = T.train_coarse(x, A, 4, 2, seed=1)[0] if residual else None
    pc = T.train_pq(x, A, Cm, 3, seed=5, max_points_per_centroid=20, M=2, ksub=16)        # 400 > 20 * 16: subsampled
    pn = T.np_train_pq(x, A, Cm, 3, seed=5, max_points_per_centroid=20, M=2, ksub=16)
    assert np.array_equal(bits(pc), bits(pn))
    ph = T.train_pq(x, A, Cm, 2, seed=5, max_points_per_centroid=20, pq0=pc, M=2, ksub=16)
    phn = T.np_train_pq(x, A, Cm, 2, seed=5, max_points_per_centroid=20, pq0=pn, M=2, ksub=16)
    assert np.array_equal(bits(ph), bits(phn))


def test_split_rule_by_hand():
    # h = [0, 5, 1], ns - k = 3: cj = 0 has p = -1/3 (draw 0 fails), cj = 1 has p = 4/3 (draw 1 succeeds whatever u is)
    Cm = np.array([[9, 9], [1.0, 2.0], [3, 4]], np.float32)
    C2, h2, nsplit = T.split_clusters(Cm, [0, 5, 1], ns=6, seed=1, s=0, it=0)
    up, dn = np.float32(1 + 2 ** -10), np.float32(1 - 2 ** -10)
    assert nsplit == 1
    assert np.array_equal(C2[0], np.array([1.0 * up, 2.0 * dn], np.float32))
    assert np.array_equal(C2[1], np.array([1.0 * dn, 2.0 * up], np.float32))
    assert np.array_equal(C2[2], Cm[2]) and h2.tolist() == [2.5, 2.5, 1.0]
    C3, h3, n3 = T.np_split_clusters(Cm, np.array([0, 5, 1], np.float32), 6, 1, 0, 0)
    assert n3 == 1 and np.array_equal(bits(C3), bits(C2)) and np.array_equal(h3, h2)


def test_planted_duplicates_force_a_split():
    """Six copies of one row among eight: at least two initial centroids coincide, the lower list id takes all their members (the
    coarse tie rule) and the other cluster empties, so iteration 0 splits."""
    rng = np.random.default_rng(4)
    x = np.concatenate([np.repeat(rng.standard_normal((1, D)), 6, 0), rng.standard_normal((2, D))]).astype(np.float32)
    Cc, _, sc = T.train_coarse(x, rot(3), 4, 3, seed=9)
    Cn, _, sn = T.np_train_coarse(x, rot(3), 4, 3, seed=9)
    assert sc[0] > 0 and np.array_equal(sc, sn) and np.array_equal(bits(Cc), bits(Cn))


def test_coarse_centroids_have_unit_norm():
    x, A = data(2000, 11, d=32), rot(5, d=32)
    Cm, obj, _ = T.train_coarse(x, A, 16, 6, seed=2)
    assert np.abs(np.linalg.norm(Cm.astype(np.float64), axis=1) - 1).max() < 1e-6
    assert obj[-1] >= obj[0]                      # spherical k-means does not lower the summed inner product here


def pq_distortion(xr, pq):
    M, ksub, dsub = pq.shape
    tot = 0.0
    for m in range(M):
        sub = xr[:, m * dsub:(m + 1) * dsub].astype(np.float64)
        d2 = ((sub[:, None, :] - pq[m][None].astype(np.float64)) ** 2).sum(-1)
        tot += d2.min(1).sum()
    return tot


def test_pq_distortion_falls():
    x, A = data(3000, 13, d=32), rot(6, d=32)
    xr = x @ A.T.astype(np.float64)
    init = T.train_pq(x, A, None, 0, seed=4, M=4, ksub=32)           # niter 0: the init alone
    trained = T.train_pq(x, A, None, 10, seed=4, M=4, ksub=32)
    assert pq_distortion(xr, trained) < 0.9 * pq_distortion(xr, init)


def test_sample_and_init_depend_only_on_seed_and_n():
    a = T.sample(5000, 700, seed=21, which=0)
    assert len(a) == 700 and np.all(np.diff(a) > 0)
    assert np.array_equal(a, T.np_sample(5000, 700, 21, 0))
    assert not np.array_equal(a, T.sample(5000, 700, seed=22, which=0))
    assert not np.array_equal(a, T.sample(5000, 700, seed=21, which=1))           # the PQ draws its own sample
    assert np.array_equal(T.sample(300, 700, seed=21, which=0), np.arange(300))   # n <= cap: every row
    r = T.init_rows(700, 16, seed=21, s=0)
    assert len(set(r.tolist())) == 16 and np.array_equal(r, T.np_init_rows(700, 16, 21, 0))
    # two different inputs of the same size share sample and init: their first centroids are rows at the same positions
    x1, x2, A = data(300, 1), data(300, 2), np.eye(D, dtype=np.float32)
    c1 = T.train_coarse(x1, A, 8, 0, seed=5)[0]
    c2 = T.train_coarse(x2, A, 8, 0, seed=5)[0]
    r = T.init_rows(300, 8, 5, 0)
    for c, x in ((c1, x1), (c2, x2)):
        assert np.allclose(c, x[r] / np.linalg.norm(x[r], axis=1, keepdims=True), atol=1e-6)


def test_fewer_points_than_centroids_is_refused():
    x = data(10, 1)
    with pytest.raises(ValueError):
        T.train_coarse(x, rot(1), 16, 2, seed=1)
    with pytest.raises(ValueError):
        T.train_pq(x, rot(1), None, 2, seed=1, M=2, ksub=16)
