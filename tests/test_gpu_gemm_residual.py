"""GPU checks of the wgmma GEMM's residual epilogue at the sizes the encoder runs it (out_proj: N = 768, K = 1536;
linear2: N = 768, K = 1024; thousands of tiles, so persistent CTAs wrap many times and the residual prefetch of one tile
overlaps the epilogue of the previous one), in place as the encoder uses it and out of place as the VAE does.

Reference = PyTorch fp32 (TF32 off) on the same fp16 operands; the result must also be bit-identical between two runs.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ffi():
    from brepgen_b200 import _ffi
    return _ffi


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.cuda.synchronize()


def _operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, K, generator=g, device="cuda").half()
    W = (torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K)).half()
    bias = torch.randn(N, generator=g, device="cuda")
    resid = torch.randn(M, N, generator=g, device="cuda")
    return A, W, bias, resid


def _gemm(A, W, M, N, K, out, ldo, bias, resid_ptr, ldr):
    f = _ffi()
    f.check(f.lib().bg_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, out, ldo, 0, 0, bias.data_ptr(), resid_ptr,
                                   ldr, None, 1, N, f.current_stream()), "gemm")


@pytest.mark.parametrize("K", [1024, 1536])
def test_inplace_residual_gemm_production_size(K):
    """X += A W^T + b over 128 000 - 37 rows (3 000 tiles of 128 x 256, the last one partial), twice from the same input"""
    M, N = 128_000 - 37, 768
    A, W, bias, resid = _operands(M, N, K, seed=K)
    ref = (A.float() @ W.float().t() + bias) + resid
    runs = []
    for _ in range(2):
        X = resid.clone()
        _gemm(A, W, M, N, K, X.data_ptr(), N, bias, X.data_ptr(), N)
        torch.cuda.synchronize()
        runs.append(X)
    err = rel_l2(runs[0], ref)
    print(f"in-place residual gemm M={M} N={N} K={K} rel_l2={err:.3e}")
    assert torch.isfinite(runs[0]).all()
    assert err < 2e-6, err
    assert torch.equal(runs[0], runs[1])


@pytest.mark.parametrize("resid_offset_floats", [0, 2])
def test_out_of_place_residual_gemm(resid_offset_floats):
    """out = A W^T + b + resid with resid a different array of another pitch (as the VAE passes it); an offset of 2 floats
    makes the residual rows 8- but not 16-byte aligned"""
    M, N, K, ldr = 128 * 400 + 9, 768, 1024, 768 + 4
    A, W, bias, resid = _operands(M, N, K, seed=11)
    rbuf = torch.full((M * ldr + 8,), float("nan"), device="cuda")
    rview = rbuf[resid_offset_floats:resid_offset_floats + M * ldr].view(M, ldr)
    rview[:, :N] = resid
    out = torch.full((M, N), float("nan"), device="cuda")
    _gemm(A, W, M, N, K, out.data_ptr(), N, bias, rview.data_ptr(), ldr)
    torch.cuda.synchronize()
    ref = (A.float() @ W.float().t() + bias) + resid
    err = rel_l2(out, ref)
    print(f"out-of-place residual gemm M={M} ldr={ldr} offset={resid_offset_floats} rel_l2={err:.3e}")
    assert torch.isfinite(out).all()
    assert err < 2e-6, err
    assert torch.equal(rview[:, :N], resid), "the residual input was written"
