"""dph_sgemm_nt_seq (prep.cu) against the sequential-k FMA definition, through every tile kernel its shape rule picks (128x128,
64x64 with 32-deep k tiles, 32-row tiles, 16-row tiles).  The SGEMM carries the OPQ rotation, the coarse scores, encode and
training; every output must be the one fp32 FMA chain over k ascending from +0, bit for bit, at row and column counts on both sides
of every kernel's tile edges, widths that are not a multiple of 4 (the scalar store tail) and depths that are not a multiple of 64
(the row-tiled kernels step k by 64; those depths take the 64x64 kernel unless the 128x128 kernel is picked)."""
import ctypes as C
import itertools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NS = (1, 15, 16, 17, 63, 64, 65, 1000, 1024, 2047, 2048, 2049)
MS = (1, 5, 768, 1000, 1001, 1025, 3969, 4095, 4096, 20000, 65536)
TILES = {"128x128": (128, 128), "64x64": (64, 64), "32x64": (32, 64), "16x64": (16, 64)}     # rows x columns per CTA


def seq_matmul_ref(X, W):
    """out[i, o] = fmaf chain over t of X[i, t] * W[o, t] (oracle/ivfpq_ref.c: dot_seq), through the C oracle's coarse quantizer:
    with nprobe = the number of rows of W every score is returned once, and scattering by list id gives the full matrix."""
    from oracle import ivfpq_ref as R
    X = np.ascontiguousarray(X, dtype=np.float32)
    W = np.ascontiguousarray(W, dtype=np.float32)
    n, K = X.shape
    m = len(W)
    cd = np.empty((n, m), dtype=np.float32)
    key = np.empty((n, m), dtype=np.int64)
    R.lib().ref_coarse(R._p(X), C.c_int64(n), C.c_int(K), R._p(W), C.c_int64(m), C.c_int(m), R._p(cd), R._p(key))
    assert (key >= 0).all()
    out = np.empty((n, m), dtype=np.float32)
    np.put_along_axis(out, key, cd, axis=1)
    return out


def tile_kernel(n, m, K):
    """The tile kernel dph_launch_sgemm_nt_seq (prep.cu) picks for out [n, m] at depth K."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cdiv = lambda a, b: -(-a // b)
    if cdiv(m, 128) * cdiv(n, 128) >= 2 * sms:
        return "128x128"
    ct = cdiv(m, 64)
    if K % 64 or ct * cdiv(n, 64) >= 128:
        return "64x64"
    return "32x64" if ct * cdiv(n, 32) >= 128 else "16x64"


def assert_every_tile_edge(shapes, K):
    """Each kernel the rule can pick at depth K gets row and column counts one below, at and one above a multiple of its tile."""
    for kern in (TILES if K % 64 == 0 else ("128x128", "64x64")):
        tm, tn = TILES[kern]
        got = [(n, m) for n, m in shapes if tile_kernel(n, m, K) == kern]
        for side, tile, vals in (("rows", tm, [n for n, _ in got]), ("columns", tn, [m for _, m in got])):
            missing = {tile - 1, 0, 1} - {v % tile for v in vals}
            assert not missing, f"K={K}: no shape sends {side} = {sorted(missing)} mod {tile} to the {kern} kernel"


def shapes():
    """Every n with the small and mid widths, every width with small n; the largest n and m meet only mid partners."""
    out = set()
    for n in NS:
        for m in MS:
            if m >= 20000 and n > 65:
                continue
            if n >= 1000 and m > 4096:
                continue
            out.add((n, m))
    return sorted(out)


def run_gpu(X, W, K):
    import torch
    from densephrases_b200 import _lib as L
    n, m = X.shape[0], W.shape[0]
    out = torch.full((n, m), float("nan"), device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(L.lib().dph_sgemm_nt_seq(X.data_ptr(), n, W.data_ptr(), m, K, out.data_ptr(), st))
    torch.cuda.synchronize()
    return out


def test_sgemm_tiles_k768_all_shapes(oracle):
    import torch
    rng = np.random.default_rng(5)
    K = 768
    X = rng.standard_normal((max(NS), K)).astype(np.float32)
    W = rng.standard_normal((max(MS), K)).astype(np.float32)
    X[3, :7] = 0.0; X[3, 7] = -0.0; W[2, 100:] = -0.0            # signed zeros in the chains
    # every shape's reference is a corner of one of two blocks: (65 rows x all widths) and (all rows x 4096 widths)
    ref_wide = seq_matmul_ref(X[:65], W)
    ref_tall = seq_matmul_ref(X, W[:4096])
    Xd, Wd = torch.from_numpy(X).cuda(), torch.from_numpy(W).cuda()
    assert len(shapes()) >= 60
    assert_every_tile_edge(shapes(), K)
    for n, m in shapes():
        ref = ref_wide[:n, :m] if n <= 65 else ref_tall[:n, :m]
        refd = torch.from_numpy(np.ascontiguousarray(ref)).cuda()
        out = run_gpu(Xd[:n].contiguous(), Wd[:m].contiguous(), K)
        bad = (out.view(torch.int32) != refd.view(torch.int32))
        assert not bool(bad.any()), f"n={n} m={m} ({tile_kernel(n, m, K)}): {int(bad.sum())} outputs differ, first at {bad.nonzero()[0].tolist()}"


@pytest.mark.parametrize("K", [32, 64, 96, 128])
def test_sgemm_tiles_short_k(oracle, K):
    """K = 32 and 96 are not multiples of the row-tiled kernels' 64-deep k tile: every shape the 128x128 kernel does not take then
    runs the 64x64 kernel."""
    import torch
    shapes = sorted({(1, 1), (17, 5), (64, 1000), (65, 1001), (130, 768), (3, 129)} |
                    set(itertools.product((257, 2047, 2048, 2049), (63, 65, 1023, 1024, 2175, 2176, 2177))))
    assert_every_tile_edge(shapes, K)
    rng = np.random.default_rng(K)
    X = rng.standard_normal((2049, K)).astype(np.float32)
    W = rng.standard_normal((2177, K)).astype(np.float32)
    Xd, Wd = torch.from_numpy(X).cuda(), torch.from_numpy(W).cuda()
    ref = seq_matmul_ref(X, W)
    for n, m in shapes:
        refd = torch.from_numpy(np.ascontiguousarray(ref[:n, :m])).cuda()
        out = run_gpu(Xd[:n].contiguous(), Wd[:m].contiguous(), K)
        assert torch.equal(out.view(torch.int32), refd.view(torch.int32)), f"K={K} n={n} m={m} ({tile_kernel(n, m, K)})"
