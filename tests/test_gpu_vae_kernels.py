"""Op-level parity of the VAEs' CUDA-core kernels (vae.cu) through their unit-level entry points, each of which runs the
networks' own launch code: GroupNorm (the `groupnorm()` dispatcher: register-resident kernels for P in {4, 8, 16, 32, 64},
the generic kernel otherwise), the mid blocks' small attention, the edge VAEs' cubic resampling, the [hi | lo] fp16
producers (cast_split, upsample2x_split, postquant) and the explicit im2col gather.

Every kernel is compared with a float64 reference on exactly the operands it sees.  Where the oracle states the operation,
the reference is the oracle's own function run in float64 (oracle.vae._gn, cubic_upsample1d, cubic_downsample1d; the
attention statement of _attn2d / _attn1d).  The CPU tests at the end check each reference helper against its fp32 oracle
counterpart.

Bars:
  - data movement (im2col, the upsample / cast hi and lo halves, the encoders' identity post_quant_conv): bit-exact;
  - fp32 arithmetic: |y - y64| <= tau * max(1, |y64|) per element, tau at most 4x the worst error measured below;
  - [hi | lo] outputs: hi is the fp16 rounding of the kernel's fp32 value (hi + lo), |lo| <= half an fp16 ulp of hi, hi + lo
    meets the fp32 bar, and hi alone misses it by at least 10x (so a dropped lo half cannot pass).

The inputs are built so that a wrong kernel fails: every (sample, group) of a GroupNorm input has its own scale
(10^-1.5 .. 10^1.5) and offset, one group has variance eps (a wrong eps moves its outputs by up to 2.3x), one group is
constant and one all zero (no NaN from 0 * rsqrt; without an activation the zero group's output must be the exact fp16
split of beta), the attention's logits reach +-100 (beyond __expf's range without the max shift, below it
with a max started at 0) and one head's V is 1e3 times larger; every output buffer starts as NaN.  A group with mean 1e3 and
std 1e-2 is not used: fp32 rounding of its mean alone is ~1e-2 of its std, so no fp32 GroupNorm could meet the bar there.

Worst elementwise errors measured on an H100 80GB HBM3 (700 W limit); the tests print them:
  GroupNorm         1.08e-6 (G 32, eps 1e-6, P 1024: the generic kernel's longest sums); 6.5e-7 (G 1, eps 1e-5)  bar 4e-6
  small attention   4.8e-7 (unit logits)                                                                        bar 1.8e-6
                    5.1e-6 (peaked: logits near +-100 carry an fp32 rounding of 2^-24 * 100 = 6e-6)             bar 1.8e-5
  cubic resampling  1.7e-7 (the two outputs at each end), 1.9e-7 (interior)                                     bar 7e-7
  postquant         4.6e-7                                                                                      bar 1.5e-6
hi alone misses every [hi | lo] bar by at least 26x (attention over one position excepted: its exact result is V).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from brepgen_b200.spec import CUBIC_DOWN_KERNEL, CUBIC_UP_KERNEL
from oracle import vae as OV

gpu = pytest.mark.gpu

NAN = float("nan")
TAU_GN = 4e-6
TAU_CUBIC = 7e-7
TAU_ATTN = {False: 1.8e-6, True: 1.8e-5}     # unit-scale / peaked logits
TAU_POSTQUANT = 1.5e-6


def _ffi():
    from brepgen_b200 import _ffi
    return _ffi


def call(name, *args):
    f = _ffi()
    f.check(getattr(f.lib(), name)(*args, f.current_stream()), name)
    torch.cuda.synchronize()


def p(t):
    return _ffi().ptr(t)


# ------------------------------------------------------------------------------------------------ float64 references
def gn_ref(x, gamma, beta, G, eps, act, resid=None):
    """x (N, P, C) channels-last -> oracle.vae._gn in float64, then the activation and the residual, in the order the VAE
    blocks apply them (act 0 none, 1 SiLU, 2 GELU)"""
    sd = {"n.weight": gamma.double(), "n.bias": beta.double()}
    y = OV._gn(x.double().permute(0, 2, 1), sd, "n", G, eps).permute(0, 2, 1)
    y = F.silu(y) if act == 1 else F.gelu(y) if act == 2 else y
    return y if resid is None else y + resid.double()


def attn_ref(qkv, Hh, scale):
    """qkv (N, T, [q | k | v]) -> (N, T, C): the attention statement of oracle.vae._attn2d / _attn1d, softmax(q k^T * scale) v
    per head, in float64"""
    N, T, C3 = qkv.shape
    C = C3 // 3
    dh = C // Hh
    q, k, v = (qkv[..., i * C:(i + 1) * C].double().reshape(N, T, Hh, dh).transpose(1, 2) for i in range(3))
    a = torch.softmax(q @ k.transpose(-1, -2) * scale, dim=-1) @ v
    return a.transpose(1, 2).reshape(N, T, C)


def cubic_ref(x, kernel, up):
    """x (N, L, C) channels-last -> oracle.vae.cubic_upsample1d / cubic_downsample1d in float64"""
    fn = OV.cubic_upsample1d if up else OV.cubic_downsample1d
    return fn(x.double().permute(0, 2, 1), kernel.double()).permute(0, 2, 1)


def im2col_ref(img, kh, kw, stride, Kpad):
    """img (N, H, W, C) -> (N * Ho * Wo, Kpad) with k = (ky * kw + kx) * C + c, by slicing a zero-padded copy: stride 1
    pads kh // 2 rows / kw // 2 columns on each side ("same"), stride 2 pads the bottom / right only (Downsample2D with
    padding=0); columns past kh * kw * C are zero"""
    N, H, W, C = img.shape
    Ho, Wo = H // stride, W // stride
    t, l = (kh // 2, kw // 2) if stride == 1 else (0, 0)
    xp = F.pad(img.permute(0, 3, 1, 2), (l, kw - 1 - l, t, kh - 1 - t))
    taps = [xp[:, :, ky:ky + stride * Ho:stride, kx:kx + stride * Wo:stride] for ky in range(kh) for kx in range(kw)]
    A = torch.cat(taps, 1).reshape(N, kh * kw, C, Ho, Wo).permute(0, 3, 4, 1, 2).reshape(N * Ho * Wo, kh * kw * C)
    return F.pad(A, (0, Kpad - kh * kw * C))


# ------------------------------------------------------------------------------------------------ checks
def elem_err(y, ref):
    """max over elements of |y - ref| / max(1, |ref|)"""
    ref = ref.double()
    return float(((y.double() - ref).abs() / ref.abs().clamp_min(1.0)).max())


def check_f32(name, y, ref, tau):
    assert torch.isfinite(y).all(), f"{name}: non-finite output"
    e = elem_err(y, ref)
    print(f"{name}: max elementwise error {e:.2e} (bar {tau:.1e})")
    assert e <= tau, (name, e)
    return e


def check_hl(name, out16, ref, tau, lo_needed=True):
    """out16 (..., [C hi | C lo]) fp16 against the float64 ref (..., C); lo_needed=False where the exact result is itself an
    fp16 value (attention over one position returns V)"""
    C = ref.shape[-1]
    hi, lo = out16[..., :C], out16[..., C:]
    assert torch.isfinite(hi).all() and torch.isfinite(lo).all(), f"{name}: non-finite output"
    v = hi.double() + lo.double()          # the kernel's fp32 value, to the rounding of lo (2^-11 of lo)
    # hi is the fp16 rounding of v: the nearest fp16 (ties either way, v then lies exactly between two)
    r = v.float().half()
    tie = (r.double() - v).abs() == (hi.double() - v).abs()
    assert ((r == hi) | tie).all(), f"{name}: hi is not the fp16 rounding of hi + lo"
    half_ulp = torch.exp2(torch.floor(torch.log2(hi.double().abs().clamp_min(2.0 ** -14))) - 11)
    assert (lo.double().abs() <= half_ulp).all(), f"{name}: |lo| exceeds half an ulp of hi"
    e, e_hi = elem_err(v, ref), elem_err(hi, ref)
    print(f"{name}: max elementwise error hi + lo {e:.2e} (bar {tau:.1e}), hi alone {e_hi:.2e}")
    assert e <= tau, (name, e)
    assert e_hi >= 10 * tau or not lo_needed, (name, e_hi)
    return e


def split_exact(name, out16, x):
    """out16 (..., [C hi | C lo]) must be the bit-exact fp16 split of the fp32 values x (..., C)"""
    C = x.shape[-1]
    hi = x.half()
    lo = (x - hi.float()).half()
    assert torch.equal(out16[..., :C].view(torch.int16), hi.view(torch.int16)), f"{name}: hi differs"
    assert torch.equal(out16[..., C:].view(torch.int16), lo.view(torch.int16)), f"{name}: lo differs"


# ------------------------------------------------------------------------------------------------ GroupNorm
def gn_input(N, P, C, G, eps, g):
    """x (N, P, C): each (sample, group) at its own scale 10^U(-1.5, 1.5) and an offset within one std; group G // 2 of
    sample 0 with variance ~eps; group G - 1 constant in the last two samples: a dyadic value in sample N - 2 (its sums are
    exact) and zero in sample N - 1 (mean, variance and x - mean all exactly 0, so the output must be exactly beta before
    the activation)"""
    cpg = C // G
    std = 10 ** (3 * torch.rand(N, 1, G, 1, generator=g, dtype=torch.float64) - 1.5)
    off = std * (2 * torch.rand(N, 1, G, 1, generator=g, dtype=torch.float64) - 1)
    x = torch.randn(N, P, G, cpg, generator=g, dtype=torch.float64) * std + off
    x[0, :, G // 2] = (torch.randn(P, cpg, generator=g, dtype=torch.float64) + 0.5) * math.sqrt(eps)
    x[N - 2, :, G - 1] = 3 * 2.0 ** -11
    x[N - 1, :, G - 1] = 0.0
    return x.reshape(N, P, C).float().cuda()


def check_zero_group(name, y, gamma, beta, G, act, resid=None):
    """the all-zero group (sample N - 1, group G - 1) of a GroupNorm output y (fp32 (N, P, C), or the [hi | lo] fp16
    (N, P, 2C)): exactly the fp16 split of beta without an activation; act(beta) (+ resid) to TAU_GN otherwise, and the same
    bits at every position"""
    N, P = y.shape[:2]
    C = beta.numel()
    c0 = C - C // G
    b = beta[c0:].expand(P, C - c0)
    if y.dtype == torch.float16:
        got = torch.cat([y[N - 1, :, c0:C], y[N - 1, :, C + c0:]], -1)
        if act == 0:
            return split_exact(name + " zero group", got, b)
        got = got[:, :C - c0].double() + got[:, C - c0:].double()
    else:
        got = y[N - 1, :, c0:]
    assert torch.isfinite(got).all(), f"{name}: zero group not finite"
    assert (got == got[:1]).all() or resid is not None, f"{name}: zero group differs between positions"
    ref = F.silu(b.double()) if act == 1 else F.gelu(b.double()) if act == 2 else b.double()
    if resid is not None:
        ref = ref + resid[N - 1, :, c0:].double()
    e = elem_err(got, ref)
    assert e <= TAU_GN, (name + " zero group", e)


def run_gn(N, P, C, G, eps, act, mode, seed):
    g = torch.Generator().manual_seed(seed)
    x = gn_input(N, P, C, G, eps, g)
    gamma = (1 + 0.5 * torch.randn(C, generator=g)).cuda()
    beta = (0.5 * torch.randn(C, generator=g)).cuda()
    name = f"groupnorm N={N} P={P} C={C} G={G} eps={eps:g} act={act} {mode}"
    if mode == "out16":
        out16 = torch.full((N, P, 2 * C), NAN, device="cuda", dtype=torch.float16)
        call("bg_op_groupnorm", p(x), N, P, C, G, eps, p(gamma), p(beta), act, None, None, p(out16))
        check_zero_group(name, out16, gamma, beta, G, act)
        return check_hl(name, out16, gn_ref(x, gamma, beta, G, eps, act), TAU_GN)
    # out32 with the residual read from and written to the same buffer, as resconv1d runs it
    resid = torch.randn(N, P, C, generator=g).cuda()
    out = resid.clone()
    call("bg_op_groupnorm", p(x), N, P, C, G, eps, p(gamma), p(beta), act, p(out), p(out), None)
    check_zero_group(name, out, gamma, beta, G, act, resid)
    return check_f32(name, out, gn_ref(x, gamma, beta, G, eps, act, resid), TAU_GN)


# P: the register-resident cases and every other extent the VAEs run (decode_hw 1..3, the 24 x 24 encoder)
GN_P = [1, 4, 8, 9, 16, 32, 36, 64, 144, 256, 576, 1024]
# 2-D blocks and both heads: G 32, eps 1e-6, SiLU into [hi | lo]; the mid-block attention's norm: C 512, no activation
GN_2D = [(P, C, 1) for P in GN_P for C in (128, 256, 512)] + [(P, 512, 0) for P in GN_P]


@gpu
@pytest.mark.parametrize("P,C,act", GN_2D)
def test_groupnorm_2d(P, C, act):
    run_gn(3, P, C, 32, 1e-6, act, "out16", seed=P * 1000 + C + act)


# 1-D ResConvBlocks and the 1-D attention's norm: G 1, eps 1e-5; GELU into [hi | lo] (group_norm_1) or onto the aliased
# residual (group_norm_2), and no activation into [hi | lo] (attention)
@gpu
@pytest.mark.parametrize("mode,act", [("out16", 2), ("out32_resid", 2), ("out16", 0)])
@pytest.mark.parametrize("C", [128, 256, 512])
@pytest.mark.parametrize("P", [1, 4, 8, 9, 16, 32, 64])
def test_groupnorm_1d(P, C, mode, act):
    run_gn(4, P, C, 1, 1e-5, act, mode, seed=P * 1000 + C + act + len(mode))


# ------------------------------------------------------------------------------------------------ small attention
def attn_input(N, T, Hh, peaked, g):
    """qkv (N, T, 3 * 512) fp16.  unit: q, k ~ N(0, 1), so the logits q k / sqrt(dh) are ~N(0, 1).  peaked: the keys of a
    head share a +-1 direction b and the query rows carry +100 / scale and -100 / scale along it in turn, so whole rows of
    logits sit near +100 or -100, spread by 2.2 (one head) or 8.8 (16 heads) within a row.  q and k are multiples of 1/8
    (|q| < 32, |k| < 4), so every product and partial sum of a logit is exact in fp32 and the logits carry only the
    rounding of the final * scale.  Head Hh // 2 (with one head: every second sample) has V in [1e3, 2e3)."""
    C = 512
    dh = C // Hh
    scale = 1 / math.sqrt(dh)
    q = torch.randn(N, T, Hh, dh, generator=g)
    k = torch.randn(N, T, Hh, dh, generator=g)
    v = torch.randn(N, T, Hh, dh, generator=g)
    if peaked:
        b = torch.where(torch.rand(N, 1, Hh, dh, generator=g) < 0.5, -1.0, 1.0)
        c = round(100 / (scale * dh) * 8) / 8
        sign = 1 - 2 * (torch.arange(N * T * Hh) % 2).reshape(N, T, Hh, 1)
        q = sign * c * b + 0.5 * q
        k = b + 0.5 * k
    q = (torch.round(q * 8) / 8).clamp(-31, 31)
    k = (torch.round(k * 8) / 8).clamp(-3.875, 3.875)
    big = 1e3 * (1 + torch.rand(v.shape, generator=g))      # positive: a weighted mean of them cannot cancel to ~0
    if Hh > 1:
        v[:, :, Hh // 2] = big[:, :, Hh // 2]
    else:
        v[1::2] = big[1::2]
    qkv = torch.cat([t.reshape(N, T, C) for t in (q, k, v)], -1).half().cuda()
    return qkv, scale


@gpu
@pytest.mark.parametrize("peaked", [False, True])
@pytest.mark.parametrize("T,Hh", [(1, 1), (4, 1), (9, 1), (16, 1), (4, 16)])
def test_vae_attention(T, Hh, peaked):
    N, C = 5, 512
    g = torch.Generator().manual_seed(T * 100 + Hh + peaked)
    qkv, scale = attn_input(N, T, Hh, peaked, g)
    q, k = qkv[..., :C].double().reshape(N, T, Hh, -1), qkv[..., C:2 * C].double().reshape(N, T, Hh, -1)
    logits = torch.einsum("nihd,njhd->nhij", q, k) * scale
    if peaked:   # some logit beyond __expf's range (88.7), and some whole row below -88 (exp underflows without the shift)
        assert float(logits.max()) > 90 and float(logits.amax(-1).min()) < -90
    out = torch.full((N * T, 2 * C), NAN, device="cuda", dtype=torch.float16)
    call("bg_op_vae_attention", p(qkv), p(out), N, T, Hh, scale)
    ref = attn_ref(qkv, Hh, scale).reshape(N * T, C)
    check_hl(f"vae attention T={T} Hh={Hh} {'peaked' if peaked else 'unit'} logits (|logit| <= "
             f"{float(logits.abs().max()):.0f})", out, ref, TAU_ATTN[peaked], lo_needed=T > 1)


# ------------------------------------------------------------------------------------------------ cubic resampling
# (L, C) of the edge decoder's three Upsample1d and the edge encoder's three Downsample1d
CUBIC = [(True, 4, 512), (True, 8, 256), (True, 16, 128), (False, 32, 128), (False, 16, 128), (False, 8, 256)]


@gpu
@pytest.mark.parametrize("up,L,C", CUBIC)
def test_cubic1d(up, L, C):
    """the two outputs at each end (where the reflect padding is read) are checked apart from the interior"""
    N = 3
    g = torch.Generator().manual_seed(L * 10 + C + up)
    x = (torch.randn(N, L, C, generator=g) + torch.linspace(-2, 3, L)[None, :, None]).cuda()
    kern = torch.tensor(CUBIC_UP_KERNEL if up else CUBIC_DOWN_KERNEL, device="cuda")
    Lo = 2 * L if up else L // 2
    y = torch.full((N, Lo, C), NAN, device="cuda")
    call("bg_op_cubic1d", p(x), p(y), N, L, C, p(kern), int(up))
    ref = cubic_ref(x, kern, up)
    ends = [0, 1, Lo - 2, Lo - 1]
    name = f"cubic {'up' if up else 'down'} L={L} C={C}"
    check_f32(name + " ends", y[:, ends], ref[:, ends], TAU_CUBIC)
    if Lo > 4:
        check_f32(name + " interior", y[:, 2:Lo - 2], ref[:, 2:Lo - 2], TAU_CUBIC)


# ------------------------------------------------------------------------------------------------ hi / lo producers
def wide_values(shape, g):
    """fp32 values over 10^-6 .. 10^4 in magnitude, both signs: lo halves from fp16 subnormals to large"""
    mag = 10 ** (10 * torch.rand(*shape, generator=g) - 6)
    return (torch.where(torch.rand(*shape, generator=g) < 0.5, -mag, mag)).cuda()


@gpu
@pytest.mark.parametrize("rows,C", [(1, 128), (1000, 128), (257, 256), (64, 512), (4 * 32 * 32, 128)])
def test_cast_split(rows, C):
    g = torch.Generator().manual_seed(rows + C)
    x = wide_values((rows, C), g)
    out = torch.full((rows, 2 * C), NAN, device="cuda", dtype=torch.float16)
    call("bg_op_cast_split", p(x), p(out), rows, C)
    split_exact(f"cast_split rows={rows} C={C}", out, x)


# (H, C) of the surface decoder's upsamplers at latents 1..4
@gpu
@pytest.mark.parametrize("H,W,C", [(1, 1, 512), (2, 2, 512), (3, 3, 512), (4, 4, 512), (6, 6, 512), (8, 8, 512),
                                   (12, 12, 256), (16, 16, 256), (3, 5, 64)])
def test_upsample2x_split(H, W, C):
    """nearest 2x, bit-exact; each input pixel differs from its transpose, so swapped axes show"""
    N = 2
    g = torch.Generator().manual_seed(H * 100 + W + C)
    x = (torch.randn(N, H, W, C, generator=g) + 10 * torch.arange(H)[None, :, None, None]
         + 1000 * torch.arange(W)[None, None, :, None]).cuda()
    out = torch.full((N, 2 * H, 2 * W, 2 * C), NAN, device="cuda", dtype=torch.float16)
    call("bg_op_upsample2x_split", p(x), p(out), N, H, W, C)
    up = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    split_exact(f"upsample2x_split {H}x{W} C={C}", out, up)


@gpu
@pytest.mark.parametrize("P", [1, 4, 9, 16, 32, 64, 1024])
def test_postquant(P):
    """the decoders' post_quant_conv (3 x 3 weights) to tau, and the encoders' identity bit-exact"""
    N = 3
    g = torch.Generator().manual_seed(P)
    z = (3 * torch.randn(N, 3, P, generator=g)).cuda()
    w = torch.randn(3, 3, generator=g).cuda()
    b = torch.randn(3, generator=g).cuda()
    out = torch.full((N, P, 6), NAN, device="cuda", dtype=torch.float16)
    call("bg_op_postquant", p(z), p(w), p(b), p(out), N, P)
    ref = torch.einsum("oc,ncp->npo", w.double(), z.double()) + b.double()
    check_hl(f"postquant P={P}", out, ref, TAU_POSTQUANT)
    eye, zero = torch.eye(3, device="cuda"), torch.zeros(3, device="cuda")
    out.fill_(NAN)
    call("bg_op_postquant", p(z), p(eye), p(zero), p(out), N, P)
    split_exact(f"postquant identity P={P}", out, z.permute(0, 2, 1))


# ------------------------------------------------------------------------------------------------ im2col
def run_im2col(N, H, W, C, kh, kw, stride, seed):
    """both planes of a [hi | lo] image (pitch 2C per pixel) into the two halves of an [A_hi | A_lo] matrix (pitch 2 Kpad),
    as conv() gathers them, bit-exact; A starts as NaN, so every zero (padding, K tail) must be written"""
    g = torch.Generator().manual_seed(seed)
    Kpad = (kh * kw * C + 63) // 64 * 64
    img = torch.randn(N, H, W, 2 * C, generator=g).half().cuda()
    rows = N * (H // stride) * (W // stride)
    A = torch.full((rows, 2 * Kpad), NAN, device="cuda", dtype=torch.float16)
    for part in range(2):
        call("bg_op_im2col", img.data_ptr() + 2 * part * C, 2 * C, A.data_ptr() + 2 * part * Kpad, 2 * Kpad, N, H, W, C,
             kh, kw, stride, Kpad)
    for part in range(2):
        ref = im2col_ref(img[..., part * C:(part + 1) * C], kh, kw, stride, Kpad)
        got = A[:, part * Kpad:(part + 1) * Kpad]
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), \
            f"im2col {H}x{W} C={C} {kh}x{kw} stride {stride} plane {part}: {int((got != ref).sum())} elements differ"


# stride 2: the surface encoder's Downsample2D convolutions at 32 / 16 / 8 and along the 24 -> 12 -> 6 chain
@gpu
# (C = 8: a VEC = 8 gather with a zero K tail, 72 of 128 columns; the product's 3 x 3 stride-2 K = 9C has none)
@pytest.mark.parametrize("H,C", [(32, 128), (16, 256), (8, 512), (24, 128), (12, 256), (6, 512), (8, 8)])
def test_im2col_stride2(H, C):
    run_im2col(3, H, H, C, 3, 3, 2, seed=H * 1000 + C)


# the 3-channel stems (VEC = 1, K 27 / 9 of 64): surface decoder at latents 1..4, surface encoder at 8..32, edge decoder /
# encoder; the stride-1 extents the implicit convolution does not take (3 x 3, 24 x 24); and VEC = 8 with a zero K tail
# (C = 8: K 72 of 128, 40 of 64)
@gpu
@pytest.mark.parametrize("H,W,C,kh,kw", [(1, 1, 3, 3, 3), (3, 3, 3, 3, 3), (4, 4, 3, 3, 3), (8, 8, 3, 3, 3),
                                         (24, 24, 3, 3, 3), (32, 32, 3, 3, 3), (1, 4, 3, 1, 3), (1, 32, 3, 1, 3),
                                         (3, 3, 512, 3, 3), (24, 24, 128, 3, 3), (8, 8, 8, 3, 3), (1, 16, 8, 1, 5)])
def test_im2col_stride1(H, W, C, kh, kw):
    run_im2col(2, H, W, C, kh, kw, 1, seed=H * 1000 + W * 10 + C)


# ------------------------------------------------------------------------------------------------ references vs oracle (CPU)
def _close(a, b, tol):
    e = float((a.double() - b.double()).norm() / b.double().norm())
    assert e < tol, e


def test_gn_ref_matches_oracle():
    g = torch.Generator().manual_seed(0)
    for G, eps, act, resid in ((32, 1e-6, 1, False), (1, 1e-5, 2, True), (32, 1e-6, 0, False)):
        x = torch.randn(2, 16, 256, generator=g) * 3 + 1
        gamma, beta = torch.randn(256, generator=g), torch.randn(256, generator=g)
        r = torch.randn(2, 16, 256, generator=g) if resid else None
        y = OV._gn(x.permute(0, 2, 1), {"n.weight": gamma, "n.bias": beta}, "n", G, eps)
        y = (F.silu(y) if act == 1 else F.gelu(y) if act == 2 else y).permute(0, 2, 1)
        _close(gn_ref(x, gamma, beta, G, eps, act, r), y if r is None else y + r, 1e-6)


@pytest.mark.parametrize("two_d", [True, False])
def test_attn_ref_matches_oracle(two_d):
    """the mid-block attention of the oracle = x + proj(attn_ref(qkv(GroupNorm(x))))"""
    g = torch.Generator().manual_seed(1)
    C, N, T = 512, 2, 9 if two_d else 4
    names = ("to_q", "to_k", "to_v", "to_out.0") if two_d else ("query", "key", "value", "proj_attn")
    sd = {"a.group_norm.weight": 1 + 0.1 * torch.randn(C, generator=g), "a.group_norm.bias": 0.1 * torch.randn(C, generator=g)}
    for n in names:
        sd[f"a.{n}.weight"] = torch.randn(C, C, generator=g) / math.sqrt(C)
        sd[f"a.{n}.bias"] = 0.1 * torch.randn(C, generator=g)
    x = torch.randn(N, C, T, generator=g)
    if two_d:
        want = OV._attn2d(sd, "a", x.reshape(N, C, 3, 3)).reshape(N, C, T)
        G, eps, Hh = 32, 1e-6, 1
    else:
        want = OV._attn1d(sd, "a", x)
        G, eps, Hh = 1, 1e-5, 16
    h = gn_ref(x.permute(0, 2, 1), sd["a.group_norm.weight"], sd["a.group_norm.bias"], G, eps, 0)
    qkv = torch.cat([h @ sd[f"a.{n}.weight"].double().t() + sd[f"a.{n}.bias"].double() for n in names[:3]], -1)
    a = attn_ref(qkv, Hh, 1 / math.sqrt(C // Hh))
    got = x.double() + (a @ sd[f"a.{names[3]}.weight"].double().t() + sd[f"a.{names[3]}.bias"].double()).permute(0, 2, 1)
    _close(got, want, 1e-5)


@pytest.mark.parametrize("up", [True, False])
def test_cubic_ref_matches_oracle(up):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 16, 64, generator=g)
    kern = torch.tensor(CUBIC_UP_KERNEL if up else CUBIC_DOWN_KERNEL)
    fn = OV.cubic_upsample1d if up else OV.cubic_downsample1d
    _close(cubic_ref(x, kern, up), fn(x.permute(0, 2, 1), kern).permute(0, 2, 1), 1e-6)


@pytest.mark.parametrize("H,stride,kh,kw", [(8, 2, 3, 3), (6, 2, 3, 3), (5, 1, 3, 3), (1, 1, 1, 3)])
def test_im2col_ref_is_the_convolution_operand(H, stride, kh, kw):
    """im2col_ref x W^T = the oracle's convolution: _downsample2d(padding=0) for stride 2, F.conv2d with "same" padding else"""
    g = torch.Generator().manual_seed(3)
    N, C, Co, W = 2, 8, 5, 7 if H > 1 else 9
    W = H if stride == 2 else W
    x = torch.randn(N, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Co, C, kh, kw, generator=g, dtype=torch.float64)
    b = torch.randn(Co, generator=g, dtype=torch.float64)
    if stride == 2:
        want = OV._downsample2d({"d.conv.weight": w, "d.conv.bias": b}, "d", x, padding=0)
    else:
        want = F.conv2d(x, w, b, padding=(kh // 2, kw // 2))
    A = im2col_ref(x.permute(0, 2, 3, 1), kh, kw, stride, kh * kw * C + 5)
    got = A[:, :kh * kw * C] @ w.permute(0, 2, 3, 1).reshape(Co, -1).t() + b
    assert (A[:, kh * kw * C:] == 0).all()
    _close(got, want.permute(0, 2, 3, 1).reshape(-1, Co), 1e-12)
