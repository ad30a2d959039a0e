"""GPU parity of the individual kernels, called through the C ABI (ctypes) exactly as the product path does.

Reference = plain PyTorch fp32 (TF32 off) on the same fp16-rounded operands, so the only differences are
accumulation order and the documented fp16 roundings (P in attention, fp16 outputs).
Tolerances (relative L2 unless stated): fp32-out GEMM 2e-6, fp16-out GEMM 1e-3 (one fp16 rounding = 2^-11),
attention 2e-3 (fp16 P and fp16 output), LayerNorm 1e-3 (fp16 output).
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
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.cuda.synchronize()


GEMM_CASES = [
    # M, N, K, out_f16, relu, bias, resid, rowvec_rpv
    (128, 256, 64, 0, 0, False, False, 0),
    (128, 128, 64, 0, 0, False, False, 0),
    (300, 768, 768, 0, 0, True, False, 0),
    (1000, 2304, 768, 1, 0, True, False, 0),
    (257, 1024, 768, 1, 1, True, False, 0),
    (513, 768, 1024, 0, 0, True, True, 0),
    (200, 128, 192, 0, 0, True, False, 7),
    (70, 768, 1536, 0, 0, True, False, 7),
    (384, 768, 2304, 0, 0, True, False, 3),
    (128 * 170, 2304, 768, 1, 0, True, False, 0),   # 1530 tiles > 132 CTAs: ring phases wrap across tiles
    (128 * 170 + 5, 768, 1024, 0, 0, True, True, 0),
    # N % 256 != 0 with many tiles: 128 x 128 tiles, persistent CTAs wrap (all three epilogues)
    (128 * 300, 128, 1152, 0, 0, True, False, 0),
    (128 * 300 + 7, 128, 576, 0, 0, True, True, 0),
    (128 * 300, 384, 256, 1, 1, True, False, 0),
]


@pytest.mark.parametrize("M,N,K,out_f16,relu,use_bias,use_resid,rpv", GEMM_CASES)
def test_gemm(M, N, K, out_f16, relu, use_bias, use_resid, rpv):
    f = _ffi()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A = (torch.randn(M, K, generator=g, device="cuda")).half()
    W = (torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K)).half()
    bias = torch.randn(N, generator=g, device="cuda") if use_bias else None
    resid = torch.randn(M, N, generator=g, device="cuda") if use_resid else None
    nvec = (M + rpv - 1) // rpv if rpv else 0
    rowvec = torch.randn(nvec, N, generator=g, device="cuda") if rpv else None
    ref = A.float() @ W.float().t()
    if bias is not None:
        ref = ref + bias
    if rowvec is not None:
        ref = ref + rowvec[torch.arange(M, device="cuda") // rpv]
    if resid is not None:
        ref = ref + resid
    if relu:
        ref = ref.relu()
    if use_resid:   # in-place residual like the encoder does
        out = resid.clone()
        resid_ptr = out.data_ptr()
    else:
        out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float16 if out_f16 else torch.float32)
        resid_ptr = None
    f.check(f.lib().bg_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, out.data_ptr(), N, out_f16, relu,
                                  f.ptr(bias), resid_ptr, N, f.ptr(rowvec), max(rpv, 1), N, f.current_stream()), "gemm")
    torch.cuda.synchronize()
    err = rel_l2(out.float(), ref)
    print(f"gemm M={M} N={N} K={K} f16={out_f16} rel_l2={err:.3e}")
    assert torch.isfinite(out.float()).all()
    assert err < (1e-3 if out_f16 else 2e-6), err


def test_gemm_rejects_misaligned_epilogue_pointers():
    """the epilogue reads bias and residual as float2 pairs: a pointer that is not 8-byte aligned is a bad argument
    (status -1), caught before any launch"""
    f = _ffi()
    A = torch.zeros(128, 64, device="cuda", dtype=torch.float16)
    W = torch.zeros(128, 64, device="cuda", dtype=torch.float16)
    out = torch.zeros(128, 128, device="cuda")
    buf = torch.zeros(128 * 128 + 2, device="cuda")
    odd = buf.data_ptr() + 4
    for bias, resid in ((odd, None), (None, odd)):
        st = f.lib().bg_op_gemm_f16(A.data_ptr(), 64, W.data_ptr(), 64, 128, 128, 64, out.data_ptr(), 128, 0, 0, bias,
                                    resid, 128, None, 1, 128, f.current_stream())
        assert st == -1 and b"8-byte aligned" in f.lib().bg_last_error()


def _attn_ref(qkv, B, L, mask):
    q, k, v = qkv.float().view(B, L, 3, 12, 64).permute(2, 0, 3, 1, 4)   # (B,12,L,64)
    s = q @ k.transpose(-1, -2) / 8.0
    if mask is not None:
        s = s.masked_fill(mask.view(B, 1, 1, L), float("-inf"))
    o = torch.softmax(s, -1) @ v
    return o.transpose(1, 2).reshape(B * L, 768)


ATTN_CASES = [
    # B, L, mask kind, block list
    (2, 30, None, 0), (2, 100, "tail", 0), (1, 128, None, 0), (3, 100, "rand", 1),
    (1, 300, None, 0), (2, 257, "rand", 0), (2, 1000, "blocks", 1), (2, 1000, "blocks", 0),
    (1, 4000, None, 0), (2, 1800, "tail", 1),
    # more work items than SMs and a different number of listed key blocks per sample (persistent kernel: items of
    # unequal length, barrier phases running across items)
    (8, 1000, "ragged", 1), (5, 700, None, 0), (16, 300, "ragged", 1),
]


@pytest.mark.parametrize("B,L,mkind,blist", ATTN_CASES)
def test_attention(B, L, mkind, blist):
    f = _ffi()
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + L)
    qkv = (torch.randn(B * L, 2304, generator=g, device="cuda") * 1.5).half()
    mask = None
    if mkind == "tail":
        mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
        mask[0, L // 2:] = True
    elif mkind == "rand":
        mask = torch.rand(B, L, generator=g, device="cuda") < 0.3
        mask[:, 0] = False
    elif mkind == "ragged":
        nvalid = torch.randint(1, L + 1, (B,), generator=g, device="cuda")
        nvalid[0] = L
        mask = torch.arange(L, device="cuda")[None, :] >= nvalid[:, None]
        mask |= torch.rand(B, L, generator=g, device="cuda") < 0.1
        mask[:, 0] = False
    elif mkind == "blocks":
        mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
        mask[0, 128:512] = True      # three fully padded key blocks
        mask[1, 700:] = True
        mask[1, 5] = True
    ref = _attn_ref(qkv, B, L, mask)
    out = torch.full((B * L, 768), float("nan"), device="cuda", dtype=torch.float16)
    nkb = (L + 127) // 128
    scratch = torch.zeros(B * (5 * nkb + 1), dtype=torch.int32, device="cuda")
    f.check(f.lib().bg_op_attention(qkv.data_ptr(), out.data_ptr(), B, L, f.ptr(mask), blist, scratch.data_ptr(),
                                   f.current_stream()), "attention")
    torch.cuda.synchronize()
    err = rel_l2(out.float(), ref)
    print(f"attention B={B} L={L} mask={mkind} blist={blist} rel_l2={err:.3e}")
    assert torch.isfinite(out.float()).all()
    assert err < 2e-3, err


@pytest.mark.parametrize("rows,act", [(1, 0), (77, 0), (5000, 1)])
def test_layernorm(rows, act):
    f = _ffi()
    g = torch.Generator(device="cuda").manual_seed(rows)
    x = torch.randn(rows, 768, generator=g, device="cuda") * 3 + 0.5
    gamma = 1 + 0.1 * torch.randn(768, generator=g, device="cuda")
    beta = 0.1 * torch.randn(768, generator=g, device="cuda")
    ref = torch.nn.functional.layer_norm(x, (768,), gamma, beta, 1e-5)
    if act:
        ref = torch.nn.functional.silu(ref)
    y = torch.empty(rows, 768, device="cuda", dtype=torch.float16)
    f.check(f.lib().bg_op_layernorm_f16(x.data_ptr(), 768, gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), 768, rows, act,
                                       f.current_stream()), "layernorm")
    torch.cuda.synchronize()
    assert rel_l2(y.float(), ref) < 1e-3


def test_fused_ddpm_and_pndm_steps():
    f = _ffi()
    g = torch.Generator(device="cuda").manual_seed(3)
    n = 100003
    eps, eps_u, x, noise = (torch.randn(n, generator=g, device="cuda") for _ in range(4))
    out = torch.empty(n, device="cuda")
    w, sb, sa, clip, c0, cx, sig = 0.6, 0.8, 0.6, 3.0, 0.3, 0.69, 0.05
    f.check(f.lib().bg_ddpm_step(eps.data_ptr(), eps_u.data_ptr(), w, x.data_ptr(), out.data_ptr(), noise.data_ptr(), 0, 0,
                                None, 0, 0, n, sb, sa, clip, c0, cx, sig, f.current_stream()))
    e = eps * (1 + w) - eps_u * w
    ref = c0 * ((x - sb * e) / sa).clamp(-clip, clip) + cx * x + sig * noise
    assert (out - ref).abs().max() < 1e-5
    # in-kernel Philox noise: zero-mean unit-variance, reproducible for a (seed, offset)
    zeros = torch.zeros(n, device="cuda")
    o1, o2 = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    for o in (o1, o2):
        f.check(f.lib().bg_ddpm_step(zeros.data_ptr(), None, 0.0, zeros.data_ptr(), o.data_ptr(), None, 1234, 77, None, 0,
                                    0, n, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, f.current_stream()))
    assert torch.equal(o1, o2)
    assert abs(float(o1.mean())) < 0.02 and abs(float(o1.std()) - 1) < 0.02
    es = [torch.randn(n, generator=g, device="cuda") for _ in range(4)]
    f.check(f.lib().bg_pndm_step(x.data_ptr(), out.data_ptr(), n, 1.01, 0.2, es[0].data_ptr(), 55 / 24, es[1].data_ptr(),
                                -59 / 24, es[2].data_ptr(), 37 / 24, es[3].data_ptr(), -9 / 24, f.current_stream()))
    ref = 1.01 * x - 0.2 * (55 * es[0] - 59 * es[1] + 37 * es[2] - 9 * es[3]) / 24
    assert (out - ref).abs().max() < 1e-5
