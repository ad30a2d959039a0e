"""GPU parity of the wgmma GEMM modes the product path runs but bg_op_gemm_f16 cannot reach, through the test entry points
bg_op_gemm_f16_ex, bg_op_conv_f16 and bg_op_layernorm_f16_ex:

  a_kwrap            A re-read cyclically along K: split-weight GEMMs [W_hi | W_lo] and the compensated fc_out
                     [x_hi | x_lo | x_hi] x [W_hi | W_hi | W_lo]
  n_short / k_short  the q|k column tiles of the fused QKV GEMM stop after the hi half of K
  m_dev              device-side row count (token compaction)
  row_map            rowvec row of the compacted token-embedding GEMM
  ConvGeom           implicit convolution: TMA box per tap, zero "same" padding, [hi | lo] plane per product term
  lo_offset/rows_dev the LayerNorm's hi / lo split that feeds the compensated fc_out

Reference = fp64 torch on exactly the fp16 operands the kernel sees.  A dropped or misread lo term moves a compensated
product by about one fp16 rounding (1.4e-4 - 2e-4 relative here), which a 1e-3 end-to-end bar cannot see; so every split
or compensated case also asserts its gain: against fp64 on the unsplit operands it must be several times closer than the
plain fp16 product.

The tensor cores' fp32 accumulation loses precision linearly in K, not as sqrt(K): measured on an H100 (SXM, 400 W),
the relative L2 error of these products against fp64 of their own operands is 1.0e-9 K - 1.8e-9 K (1.6e-6 at K = 1536,
1.5e-5 at K = 13824, the 3-term 3x3 convolution over 512 channels).  So the fp32-output bar is the 2e-6 of the other
GEMM tests up to K ~ 800 and K u / 24 (u = 2^-24) beyond, and the gain the compensation can show shrinks as 1 / K: the
required gain is 50 up to K = 2000 (every denoiser GEMM but the fc_out tail) and 1e5 / K beyond (measured: 63 - 83x at
K <= 2304, 13 - 18x at K = 9216 - 13824).

An fp16 output carries its own rounding of 2^-11, so no gain can show in its relative error; fp16 outputs must instead be
correctly rounded (within half an fp16 ulp of the fp64 value, plus 4e-5 of the RMS for the accumulation) against their
own operands and against the unsplit ones, and the plain fp16 product, rounded to fp16, must miss that bound by at least
10x the allowance.

The buffers are built so that a wrong read shows: A columns past a_kwrap are NaN (a tensor map over K columns would read
them; a loop that ignores the wrap reads zero fill instead, which the gain assertion catches), the unused lo half of the
q|k weight rows holds large values, the unused lo plane of a 2-term convolution is NaN, and outputs start as NaN.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

NAN = float("nan")
F16_SLACK = 4e-5
F16_GAIN = 10.0


def f32_bar(K):
    """relative-L2 bar of an fp32 output against fp64 of the kernel's own operands (see the module docstring)"""
    return max(2e-6, K * 2.0 ** -24 / 24)


def gain_needed(K):
    return min(50.0, 1e5 / K)


def _ffi():
    from brepgen_b200 import _ffi
    return _ffi


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def f16_excess(out16, ref):
    """largest distance of an fp16 result from the fp64 value `ref` beyond correct rounding (half an fp16 ulp of ref),
    relative to the RMS of ref; <= 0 when every element is correctly rounded"""
    ref = ref.double()
    half_ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 11)
    return float(((out16.double() - ref).abs() - half_ulp).max() / ref.pow(2).mean().sqrt())


def split(x):
    """fp16 hi / lo pair of an fp32 tensor, as the packers and the LayerNorm store it"""
    hi = x.half()
    return hi, (x - hi.float()).half()


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.cuda.synchronize()


def rows_around_switch(N):
    """row counts for an N-column GEMM: `below` gives fewer 128 x 256 tiles than SMs (so 128 x 128 tiles run), `at` just
    enough for 128 x 256 tiles, `many` four times as many tiles as SMs (persistent CTAs wrap); all end in a partial tile"""
    per = N // 256
    t = -(-torch.cuda.get_device_properties(0).multi_processor_count // per)
    return {"below": 128 * (t - 1) - 5, "at": 128 * t - 5, "many": 128 * 4 * t + 37}


def gemm_ex(A, lda, W, ldw, M, N, K, out, ldo, *, bias=None, resid=None, ldr=0, rowvec=None, rpv=1, ldv=0, relu=0,
            a_kwrap=0, n_short=0, k_short=0, m_dev=None, row_map=None):
    f = _ffi()
    f.check(f.lib().bg_op_gemm_f16_ex(A.data_ptr(), lda, W.data_ptr(), ldw, M, N, K, out.data_ptr(), ldo,
                                      int(out.dtype == torch.float16), relu, f.ptr(bias), f.ptr(resid), ldr, f.ptr(rowvec),
                                      rpv, ldv, a_kwrap, n_short, k_short, f.ptr(m_dev), f.ptr(row_map),
                                      f.current_stream()), "gemm_ex")


def check_compensated(name, K, out, exact, target, plain):
    """out: the kernel's result over K; exact: fp64 of the kernel's own fp16 operands; target: fp64 on the unsplit
    operands; plain: fp64 of the plain fp16 product (all after the same epilogue)"""
    assert torch.isfinite(out.float()).all(), name
    if out.dtype == torch.float16:
        e_exact, e_target = f16_excess(out, exact), f16_excess(out, target)
        e_plain = f16_excess(plain.half(), target)
        print(f"{name}: fp16 rounding excess vs own operands {e_exact:.2e}, vs unsplit {e_target:.2e} "
              f"(plain fp16 product {e_plain:.2e}, {e_plain / F16_SLACK:.0f}x the allowance)")
        assert e_exact <= F16_SLACK and e_target <= F16_SLACK, (e_exact, e_target)
        assert e_plain >= F16_GAIN * F16_SLACK, e_plain
    else:
        e_exact, e_target, e_plain = rel_l2(out, exact), rel_l2(out, target), rel_l2(plain, target)
        print(f"{name}: rel_l2 vs own operands {e_exact:.2e} (bar {f32_bar(K):.1e}), vs unsplit {e_target:.2e}, plain fp16 "
              f"product {e_plain:.2e} (gain {e_plain / e_target:.0f}x, needed {gain_needed(K):.0f}x)")
        assert e_exact < f32_bar(K), e_exact
        assert e_target * gain_needed(K) <= e_plain, (e_target, e_plain)


def epilogue(v, bias, resid, relu):
    if bias is not None:
        v = v + bias.double()
    if resid is not None:
        v = v + resid.double()
    return v.relu() if relu else v


# ------------------------------------------------------------------------------------------------ a_kwrap
def kwrap_operands(layout, M, N, D, g):
    """A buffer (NaN in columns [a_kwrap, lda)), packed weights and the fp64 products (exact, target, plain)"""
    W32 = torch.randn(N, D, generator=g, device="cuda") / math.sqrt(D)
    W_hi, W_lo = split(W32)
    if layout == "w_split":             # [A] x [W_hi | W_lo]: a_kwrap = D, K = 2D
        A_hi = torch.randn(M, D, generator=g, device="cuda").half()
        Abuf = torch.full((M, 2 * D), NAN, device="cuda", dtype=torch.float16)
        Abuf[:, :D] = A_hi
        Wbuf = torch.cat([W_hi, W_lo], 1).contiguous()
        a = A_hi.double()
        exact = a @ (W_hi.double() + W_lo.double()).t()
        target = a @ W32.double().t()
        plain = a @ W_hi.double().t()
        return Abuf, 2 * D, Wbuf, D, 2 * D, exact, target, plain
    # fc_out: [x_hi | x_lo | NaN] (pitch 3D) x [W_hi | W_hi | W_lo]: a_kwrap = 2D, K = 3D
    x32 = torch.randn(M, D, generator=g, device="cuda")
    x_hi, x_lo = split(x32)
    Abuf = torch.full((M, 3 * D), NAN, device="cuda", dtype=torch.float16)
    Abuf[:, :D] = x_hi
    Abuf[:, D:2 * D] = x_lo
    Wbuf = torch.cat([W_hi, W_hi, W_lo], 1).contiguous()
    xh, xl, wh, wl = x_hi.double(), x_lo.double(), W_hi.double().t(), W_lo.double().t()
    exact = xh @ wh + xl @ wh + xh @ wl
    target = x32.double() @ W32.double().t()
    plain = xh @ wh
    return Abuf, 3 * D, Wbuf, 2 * D, 3 * D, exact, target, plain


KWRAP_CASES = [
    # name, layout, D (A columns), N, bias, in-place residual, fp16 out, ReLU
    ("out_proj", "w_split", 768, 768, True, True, 0, 0),
    ("linear2", "w_split", 1024, 768, True, True, 0, 0),
    ("linear1", "w_split", 768, 1024, True, False, 1, 1),
    ("v_rows", "w_split", 768, 768, True, False, 1, 0),
    ("no_bias", "w_split", 1024, 1024, False, False, 0, 0),
    ("fc_out", "fc_out", 768, 768, True, False, 0, 0),
    ("fc_out_relu", "fc_out", 768, 768, False, False, 0, 1),
]


@pytest.mark.parametrize("m_kind", ["below", "at", "many"])
@pytest.mark.parametrize("name,layout,D,N,use_bias,use_resid,out_f16,relu", KWRAP_CASES)
def test_kwrap_gemm(name, layout, D, N, use_bias, use_resid, out_f16, relu, m_kind):
    M = rows_around_switch(N)[m_kind]
    g = torch.Generator(device="cuda").manual_seed(M + N + D)
    Abuf, lda, Wbuf, a_kwrap, K, exact, target, plain = kwrap_operands(layout, M, N, D, g)
    bias = torch.randn(N, generator=g, device="cuda") * 0.5 if use_bias else None
    resid = torch.randn(M, N, generator=g, device="cuda") if use_resid else None
    if use_resid:
        out = resid.clone()             # in place, as the encoder runs out_proj / linear2
    else:
        out = torch.full((M, N), NAN, device="cuda", dtype=torch.float16 if out_f16 else torch.float32)
    gemm_ex(Abuf, lda, Wbuf, K, M, N, K, out, N, bias=bias, resid=out if use_resid else None, ldr=N, relu=relu,
            a_kwrap=a_kwrap)
    torch.cuda.synchronize()
    ep = lambda v: epilogue(v, bias, resid, relu)
    check_compensated(f"kwrap {name} M={M} K={K} a_kwrap={a_kwrap}", K, out, ep(exact), ep(target), ep(plain))


# ------------------------------------------------------------------------------------------------ n_short / k_short
def qkv_operands(M, g):
    """the precision-1 QKV call: A = Xn [M][768] (NaN past column 768 of a 1536 pitch); W [2304][1536] with q|k rows
    [W_hi | large values the GEMM must not read] and v rows [W_hi | W_lo]"""
    D, N = 768, 2304
    A_hi = torch.randn(M, D, generator=g, device="cuda").half()
    Abuf = torch.full((M, 2 * D), NAN, device="cuda", dtype=torch.float16)
    Abuf[:, :D] = A_hi
    W32 = torch.randn(N, D, generator=g, device="cuda") / math.sqrt(D)
    W_hi, W_lo = split(W32)
    Wbuf = torch.cat([W_hi, W_lo], 1)
    Wbuf[:2 * D, D:] = (torch.randn(2 * D, D, generator=g, device="cuda") * 300).half()
    return A_hi, Abuf, W32, W_hi, W_lo, Wbuf.contiguous()


@pytest.mark.parametrize("m_kind", ["below", "many"])
@pytest.mark.parametrize("out_f16", [1, 0])
def test_qkv_short_columns(out_f16, m_kind):
    D, N = 768, 2304
    M = rows_around_switch(N)[m_kind]
    g = torch.Generator(device="cuda").manual_seed(M + out_f16)
    A_hi, Abuf, W32, W_hi, W_lo, Wbuf = qkv_operands(M, g)
    bias = torch.randn(N, generator=g, device="cuda") * 0.5
    out = torch.full((M, N), NAN, device="cuda", dtype=torch.float16 if out_f16 else torch.float32)
    gemm_ex(Abuf, 2 * D, Wbuf, 2 * D, M, N, 2 * D, out, N, bias=bias, a_kwrap=D, n_short=2 * D, k_short=D)
    torch.cuda.synchronize()
    a, b = A_hi.double(), bias.double()
    qk_ref = a @ W_hi[:2 * D].double().t() + b[:2 * D]          # q|k tiles: hi half of K only
    qk = out[:, :2 * D]
    assert torch.isfinite(qk.float()).all()
    if out_f16:
        e = f16_excess(qk, qk_ref)
        print(f"qkv M={M} f16 q|k columns: fp16 rounding excess vs hi-only product {e:.2e}")
        assert e <= F16_SLACK, e
    else:
        e = rel_l2(qk, qk_ref)
        print(f"qkv M={M} f32 q|k columns: rel_l2 vs hi-only product {e:.2e}")
        assert e < f32_bar(D), e
    v = slice(2 * D, N)
    check_compensated(f"qkv M={M} v columns", 2 * D, out[:, v], a @ (W_hi[v].double() + W_lo[v].double()).t() + b[v],
                      a @ W32[v].double().t() + b[v], a @ W_hi[v].double().t() + b[v])


# ------------------------------------------------------------------------------------------------ m_dev
def m_dev_values(M):
    return [0, 1, 63, 64, 65, 127, 128, 129, M - 1, M, M + 5]


@pytest.mark.parametrize("m_kind", ["below", "many"])
@pytest.mark.parametrize("kind", ["out_proj", "qkv"])
def test_device_row_count(kind, m_kind):
    """only rows below min(M, *m_dev) are written, bit-identical to the run without m_dev; rows from there on keep their
    bytes (the residual of the in-place fp32 out_proj, the NaN sentinel of the fp16 QKV output)"""
    D = 768
    if kind == "out_proj":
        N = D
        M = rows_around_switch(N)[m_kind]
        g = torch.Generator(device="cuda").manual_seed(M)
        Abuf, lda, Wbuf, a_kwrap, K, *_ = kwrap_operands("w_split", M, N, D, g)
        bias = torch.randn(N, generator=g, device="cuda")
        resid = torch.randn(M, N, generator=g, device="cuda")
        fresh = lambda: resid.clone()
        run = lambda out, m_dev: gemm_ex(Abuf, lda, Wbuf, K, M, N, K, out, N, bias=bias, resid=out, ldr=N,
                                         a_kwrap=a_kwrap, m_dev=m_dev)
    else:
        N = 3 * D
        M = rows_around_switch(N)[m_kind]
        g = torch.Generator(device="cuda").manual_seed(M)
        _, Abuf, _, _, _, Wbuf = qkv_operands(M, g)
        bias = torch.randn(N, generator=g, device="cuda")
        fresh = lambda: torch.full((M, N), NAN, device="cuda", dtype=torch.float16)
        run = lambda out, m_dev: gemm_ex(Abuf, 2 * D, Wbuf, 2 * D, M, N, 2 * D, out, N, bias=bias, a_kwrap=D,
                                         n_short=2 * D, k_short=D, m_dev=m_dev)
    full = fresh()
    run(full, None)
    torch.cuda.synchronize()
    assert torch.isfinite(full.float()).all()
    for m in m_dev_values(M):
        out, before = fresh(), fresh()
        run(out, torch.tensor([m], dtype=torch.int32, device="cuda"))
        torch.cuda.synchronize()
        k = min(m, M)
        assert torch.equal(bits(out[:k]), bits(full[:k])), f"{kind} M={M} m_dev={m}: computed rows differ"
        assert torch.equal(bits(out[k:]), bits(before[k:])), f"{kind} M={M} m_dev={m}: rows past the count were written"
    print(f"m_dev {kind} M={M}: {len(m_dev_values(M))} row counts exact")


# ------------------------------------------------------------------------------------------------ row_map
@pytest.mark.parametrize("B,L,rpv", [(6, 300, 1), (6, 300, 7), (6, 300, 40), (3, 4000, 4000)])
def test_row_map_rowvec(B, L, rpv):
    """the compacted token-embedding GEMM: row r of the compact layout adds rowvec[row_map[r] / rows_per_vec], with the
    sorted valid-token map b * L + t the compaction kernel builds (sample 0 all valid, sample 1 all padded)"""
    M, N, K = B * L, 768, 1536
    g = torch.Generator(device="cuda").manual_seed(B * L + rpv)
    valid = torch.rand(B, L, generator=g, device="cuda") > 0.35
    valid[0] = True
    valid[1] = False
    idx = torch.nonzero(valid.flatten()).flatten().int()
    m = idx.numel()
    row_map = torch.zeros(M, dtype=torch.int32, device="cuda")
    row_map[:m] = idx
    m_dev = torch.tensor([m], dtype=torch.int32, device="cuda")
    A = torch.randn(M, K, generator=g, device="cuda").half()
    W = (torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K)).half()
    bias = torch.randn(N, generator=g, device="cuda")
    rowvec = torch.randn((M + rpv - 1) // rpv, N, generator=g, device="cuda")
    out = torch.full((M, N), NAN, device="cuda")
    gemm_ex(A, K, W, K, M, N, K, out, N, bias=bias, rowvec=rowvec, rpv=rpv, ldv=N, m_dev=m_dev, row_map=row_map)
    torch.cuda.synchronize()
    ref = A[:m].double() @ W.double().t() + bias.double() + rowvec.double()[idx.long() // rpv]
    err = rel_l2(out[:m], ref)
    print(f"row_map B={B} L={L} rows_per_vec={rpv} valid={m}/{M} rel_l2={err:.2e}")
    assert torch.isfinite(out[:m]).all()
    assert err < f32_bar(K), err
    assert torch.isnan(out[m:]).all(), "rows past the valid count were written"


# ------------------------------------------------------------------------------------------------ implicit convolution
def conv_f16(x, ldc, w, Cout, N, H, W, C, taps, kw, terms, out, bias, resid):
    f = _ffi()
    f.check(f.lib().bg_op_conv_f16(x.data_ptr(), ldc, w.data_ptr(), Cout, N, H, W, C, taps, kw, 1, terms, out.data_ptr(),
                                   Cout, bias.data_ptr(), f.ptr(resid), Cout, f.current_stream()), "conv")


def run_conv(H, W, C, taps, kw, N, Cout, terms, seed):
    """one implicit convolution of an (N, H, W) image with C channels (1-D: H = 1, kw = taps) against fp64 F.conv2d /
    F.conv1d with padding k // 2.  3 terms: [x_hi | x_lo] image, in-place residual; 2 terms: lo plane NaN (never read),
    out-of-place into NaN.  The image pitch has 64 NaN channels past the planes."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    kh = taps // kw
    two_d = H > 1 or kh > 1
    x32 = torch.randn(N, H, W, C, generator=g, device="cuda")        # every pixel non-zero, borders included
    x_hi, x_lo = split(x32)
    ldc = 2 * C + 64
    xbuf = torch.full((N, H, W, ldc), NAN, device="cuda", dtype=torch.float16)
    xbuf[..., :C] = x_hi
    if terms == 3:
        xbuf[..., C:2 * C] = x_lo
    w32 = torch.randn(Cout, C, kh, kw, generator=g, device="cuda") / math.sqrt(C * taps)
    w_hi, w_lo = split(w32)
    pk = lambda t: t.permute(0, 2, 3, 1).reshape(Cout, taps * C)   # k = tap * C + c, tap = ky * kw + kx
    wbuf = torch.cat([pk(w_hi), pk(w_hi), pk(w_lo)] if terms == 3 else [pk(w_hi), pk(w_lo)], 1).contiguous()
    bias = torch.randn(Cout, generator=g, device="cuda") * 0.5
    rows = N * H * W
    resid = torch.randn(rows, Cout, generator=g, device="cuda") if terms == 3 else None
    out = resid.clone() if terms == 3 else torch.full((rows, Cout), NAN, device="cuda")
    conv_f16(xbuf, ldc, wbuf, Cout, N, H, W, C, taps, kw, terms, out, bias, out if terms == 3 else None)
    torch.cuda.synchronize()

    def conv(a, b):       # channels-last image (N, H, W, C), weights (Cout, C, kh, kw) -> (rows, Cout), fp64
        a, b = a.double(), b.double()
        if two_d:
            y = F.conv2d(a.permute(0, 3, 1, 2), b, padding=(kh // 2, kw // 2)).permute(0, 2, 3, 1)
        else:
            y = F.conv1d(a[:, 0].permute(0, 2, 1), b[:, :, 0], padding=kw // 2).permute(0, 2, 1)
        return y.reshape(rows, Cout)

    ep = lambda v: epilogue(v, bias, resid, 0)
    if terms == 3:
        exact = conv(x_hi, w_hi) + conv(x_lo, w_hi) + conv(x_hi, w_lo)
        target = conv(x32, w32)
    else:
        exact = conv(x_hi, w_hi) + conv(x_hi, w_lo)
        target = conv(x_hi, w32)         # 2 terms split the weights only: the image operand is x_hi
    check_compensated(f"conv {'2d' if two_d else '1d'} {H}x{W} C={C} taps={taps} N={N} Cout={Cout} terms={terms}",
                      terms * taps * C, out,
                      ep(exact), ep(target), ep(conv(x_hi, w_hi)))


# (extent, C) of every implicit convolution the four VAEs run (surface decoder at latents 1..4, surface encoder at inputs
# 8..32, edge decoder / encoder), plus C = 64 at every extent
CONV2D = [(1, 512), (2, 256), (2, 512), (4, 128), (4, 256), (4, 512), (8, 128), (8, 256), (8, 512), (16, 128),
          (16, 256), (16, 512), (32, 128), (32, 256)] + [(e, 64) for e in (1, 2, 4, 8, 16, 32)]
CONV1D = [(4, 256, 5), (4, 512, 5), (8, 128, 5), (8, 256, 5), (8, 512, 5), (16, 128, 5), (16, 256, 5), (4, 512, 3),
          (32, 128, 3)] + [(e, 64, k) for e in (4, 8, 16, 32) for k in (5, 3)]


def _images(hw):
    """N with N * hw not a multiple of 128 where that is possible (hw < 128): a partial last tile"""
    return 2 * (128 // hw) + 1 if hw < 128 else 3


@pytest.mark.parametrize("terms", [3, 2])
@pytest.mark.parametrize("hw,C", CONV2D)
def test_implicit_conv2d(hw, C, terms):
    run_conv(hw, hw, C, 9, 3, _images(hw * hw), 128 if C == 64 else 256, terms, seed=hw * 1000 + C + terms)


@pytest.mark.parametrize("terms", [3, 2])
@pytest.mark.parametrize("L,C,taps", CONV1D)
def test_implicit_conv1d(L, C, taps, terms):
    run_conv(1, L, C, taps, taps, _images(L), 128 if C == 64 else 256, terms, seed=L * 1000 + C + taps + terms)


@pytest.mark.parametrize("terms", [3, 2])
def test_implicit_conv_many_tiles(terms):
    """more 128 x 256 tiles than SMs (persistent CTAs wrap) with a ragged image count"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    run_conv(4, 4, 512, 9, 3, 16 * sms + 3, 512, terms, seed=7 + terms)
    run_conv(1, 8, 256, 5, 5, 32 * sms + 5, 256, terms, seed=9 + terms)


# ------------------------------------------------------------------------------------------------ LayerNorm hi / lo
@pytest.mark.parametrize("rows,rows_dev", [(1, None), (77, None), (5000, None), (5000, 4097), (300, 0), (300, 299)])
def test_layernorm_split(rows, rows_dev):
    """y = [hi | lo | untouched] with pitch 2304 and lo_offset 768, as the compensated fc_out reads it: hi + lo is the
    fp64 LayerNorm to 1e-6, hi alone one fp16 rounding; rows at or past *rows_dev and columns past 1536 keep their NaN"""
    f = _ffi()
    D, ldy = 768, 3 * 768
    g = torch.Generator(device="cuda").manual_seed(rows * 3 + (rows_dev or 0))
    x = torch.randn(rows, D, generator=g, device="cuda") * 3 + 0.5
    gamma = 1 + 0.1 * torch.randn(D, generator=g, device="cuda")
    beta = 0.1 * torch.randn(D, generator=g, device="cuda")
    y = torch.full((rows, ldy), NAN, device="cuda", dtype=torch.float16)
    rd = None if rows_dev is None else torch.tensor([rows_dev], dtype=torch.int32, device="cuda")
    f.check(f.lib().bg_op_layernorm_f16_ex(x.data_ptr(), D, gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), ldy, rows,
                                          0, D, f.ptr(rd), f.current_stream()), "layernorm_ex")
    torch.cuda.synchronize()
    k = rows if rows_dev is None else min(rows, rows_dev)
    assert torch.isnan(y[k:]).all(), "rows past the device row count were written"
    assert torch.isnan(y[:, 2 * D:]).all(), "columns past the lo half were written"
    if k == 0:
        return
    ref = F.layer_norm(x[:k].double(), (D,), gamma.double(), beta.double(), 1e-5)
    hi, lo = y[:k, :D], y[:k, D:2 * D]
    e_split, e_hi = rel_l2(hi.double() + lo.double(), ref), rel_l2(hi, ref)
    print(f"layernorm split rows={rows} rows_dev={rows_dev}: hi+lo rel_l2={e_split:.2e}, hi alone {e_hi:.2e} "
          f"(gain {e_hi / e_split:.0f}x)")
    assert e_split <= 1e-6, e_split
    assert 2.0 ** -14 < e_hi < 2.0 ** -11, e_hi
    assert e_split * 50 <= e_hi
