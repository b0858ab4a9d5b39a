"""wgmma TF32 GEMM (densephrases_b200/csrc/gemm_tf32.cu) vs a plain PyTorch fp32 reference of the same op.
Tolerance: TF32 keeps 10 mantissa bits of each operand (rel. 2^-11 per product), accumulation is fp32; for K <= 3072 and
unit-scale operands |err| <= 2e-3 * sqrt(K) * scale is comfortably loose; we assert a relative Frobenius error < 1e-3."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def run_gemm(A, W, bias, resid, act, precise=0):
    import torch
    from densephrases_b200 import _lib as L
    out = torch.empty((A.shape[0], W.shape[0]), dtype=torch.float32, device=A.device)
    st = torch.cuda.current_stream().cuda_stream
    L.check(L.lib().dph_gemm_tf32_nt(A.data_ptr(), W.data_ptr(), bias.data_ptr() if bias is not None else None,
                                     resid.data_ptr() if resid is not None else None, out.data_ptr(), A.shape[0], W.shape[0], A.shape[1], act,
                                     precise, C.c_void_p(st)))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 128, 768), (4096, 768, 768), (4096, 2304, 768), (4096, 3072, 768), (4096, 768, 3072),
                                   (100, 256, 64), (1, 128, 96), (333, 768, 768)])
@pytest.mark.parametrize("variant", ["plain", "bias_gelu", "bias_resid"])
def test_gemm_tf32_matches_torch_fp32(M, N, K, variant):
    import torch
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A = torch.randn((M, K), generator=g, device="cuda")
    W = torch.randn((N, K), generator=g, device="cuda") * 0.05
    bias = torch.randn((N,), generator=g, device="cuda") if variant != "plain" else None
    resid = torch.randn((M, N), generator=g, device="cuda") if variant == "bias_resid" else None
    act = 1 if variant == "bias_gelu" else 0
    out = run_gemm(A, W, bias, resid, act)
    ref = A.double() @ W.double().T
    if bias is not None:
        ref = ref + bias.double()
    if act:
        ref = torch.nn.functional.gelu(ref)
    if resid is not None:
        ref = ref + resid.double()
    err = (out.double() - ref).norm() / ref.norm()
    assert torch.isfinite(out).all()
    assert err < 1e-3, f"relative error {err:.3e}"
    # 3xTF32 split mode: fp32-accurate
    outp = run_gemm(A, W, bias, resid, act, precise=1)
    errp = (outp.double() - ref).norm() / ref.norm()
    ref32 = torch.nn.functional.linear(A, W, bias)
    if act:
        ref32 = torch.nn.functional.gelu(ref32)
    if resid is not None:
        ref32 = ref32 + resid
    err32 = (ref32.double() - ref).norm() / ref.norm()
    assert errp < 5e-5, f"3xTF32 relative error {errp:.3e} (torch fp32: {err32:.3e})"
    # exactness of the data path: with operands exactly representable in TF32 the result must match fp32 to rounding
    A2 = (A * 8).round() / 8
    W2 = (W * 64).round() / 64
    out2 = run_gemm(A2.contiguous(), W2.contiguous(), None, None, 0)
    ref2 = (A2.double() @ W2.double().T)
    assert (out2.double() - ref2).abs().max() < 1e-3 * max(1.0, ref2.abs().max().item() * 1e-3)


@pytest.mark.parametrize("M,N,K", [(4096, 768, 768), (333, 2304, 768), (64, 3072, 768), (1000, 256, 3072), (20000, 768, 96), (1, 256, 32),
                                   (127, 512, 64), (129, 768, 3072), (4096, 2304, 768), (4097, 3072, 768)])
def test_gemm_schedules_are_bit_identical(M, N, K):
    """N % 256 == 0 runs persistent 128x256 tiles, one CTA per SM; the same problem with W, bias and residual padded by 128 output
    columns (N % 256 != 0) runs one 128x128 tile per CTA.  Both issue the same MMAs per output element in the same order."""
    import torch
    assert N % 256 == 0
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn((M, K), generator=g, device="cuda")
    W = torch.randn((N + 128, K), generator=g, device="cuda") * 0.05
    bias = torch.randn((N + 128,), generator=g, device="cuda")
    resid = torch.randn((M, N + 128), generator=g, device="cuda")
    persistent = run_gemm(A, W[:N], bias[:N], resid[:, :N].contiguous(), 1)
    per_tile = run_gemm(A, W, bias, resid, 1)[:, :N]
    assert torch.isfinite(persistent).all()
    assert torch.equal(persistent, per_tile), f"max|diff| {(persistent - per_tile).abs().max().item():.3e}"


@pytest.mark.parametrize("M,N,K", [(128, 256, 32), (4096, 768, 768), (4096, 2304, 768), (4096, 3072, 768), (4096, 768, 3072), (100, 256, 64), (1, 256, 96),
                                   (333, 768, 768)])
@pytest.mark.parametrize("variant", ["plain", "bias_gelu", "bias_resid"])
def test_gemm_bf16x3_matches_fp64(M, N, K, variant):
    """gemm_bf16x3.cu: fp32 operands carried as (hi, lo) bf16 planes, a_hi.b_lo + a_lo.b_hi + a_hi.b_hi in an fp32 register accumulator.
    Representation error 2^-18 per operand + the dropped lo.lo term 2^-18 -> relative Frobenius error well below 2e-5 (1xTF32: ~3e-4,
    torch fp32: ~1e-7); operands that are exact in two bf16 planes (16 mantissa bits) must reproduce the fp32 product to rounding."""
    import torch
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(M * 5 + N * 3 + K)
    A = torch.randn((M, K), generator=g, device="cuda")
    W = torch.randn((N, K), generator=g, device="cuda") * 0.05
    bias = torch.randn((N,), generator=g, device="cuda") if variant != "plain" else None
    resid = torch.randn((M, N), generator=g, device="cuda") if variant == "bias_resid" else None
    act = 1 if variant == "bias_gelu" else 0
    out = run_gemm(A, W, bias, resid, act, precise=2)
    ref = A.double() @ W.double().T
    if bias is not None:
        ref = ref + bias.double()
    if act:
        ref = torch.nn.functional.gelu(ref)
    if resid is not None:
        ref = ref + resid.double()
    assert torch.isfinite(out).all()
    err = (out.double() - ref).norm() / ref.norm()
    err1 = (run_gemm(A, W, bias, resid, act, precise=0).double() - ref).norm() / ref.norm() if N % 128 == 0 else 1.0
    print(f"bf16x3 {M}x{N}x{K} {variant}: rel err {err:.2e} (1xTF32 {err1:.2e})")
    assert err < 2e-5, f"relative error {err:.3e}"
    A2 = (A * 256).round() / 256            # <= 11 significant bits -> exact in (hi, lo)
    W2 = (W * 4096).round() / 4096
    out2 = run_gemm(A2.contiguous(), W2.contiguous(), None, None, 0, precise=2)
    ref2 = A2.double() @ W2.double().T
    assert (out2.double() - ref2).abs().max() < 2e-5 * max(1.0, ref2.abs().max().item())
