"""Float64 parity of the flash-attention kernel (csrc/attn.cu) through bg_op_attention (with and without the block list,
its scratch read back) and bg_op_attention_varlen, at element level.

Two float64 references, on exactly the kernel's fp16 operands, per (sample, head):
  - plain:    softmax(q k^T / 8 + mask) v;
  - emulated: the operation attn.cu documents, block by block over the 128-key blocks the kernel visits.  r_j is the running
              max over the valid keys of blocks 0..j (0 while there is none), p_k = 2^(c (s_k - r_j)) with the kernel's
              c = fp32(log2 e) / 8, P16_k = fp16_rne(p_k) (fp16 subnormals included),
              O = sum_j 2^(c (r_j - r_last)) sum_{k in j} P16_k v_k,  l = sum_k 2^(c (s_k - r_last)) from the UNROUNDED p,
              mu = O / l (0 when l = 0).  A = sum_k p_k |v_k| / l (per output element) scales the arithmetic allowance.

Checks, for every output element (padded query rows of dense launches included):
  - tight:    |y - mu| <= 1/2 ulp16 + amb + tau A.  amb covers the keys whose p lies so close to an fp16 rounding midpoint that
              the kernel's fp32 p (nm = fp32(r c), one fma, ex2.approx: relative error <= ln2 2^-24 (|c r| + |c (s - r)|)
              + 2^-21) may round the other way: sum over those keys of |fp16(p (1 + rho)) - fp16(p (1 - rho))| |v| / l;
  - provable: |y - plain| <= 1/2 ulp16 + (2^-11 sum p_k |v_k| + 2^-25 sum |v_k|) / l + tau A, which any kernel that rounds P
              to fp16 meets, whatever exponential it uses.
tau is one number per input family, at most 4x the worst value measured on an H100 (see TAU); the tests print the worst
tau each check needed next to its bar.  test_checker_power shows that the tight bar tests the modelled rounding: fp16 of the
plain softmax (P not rounded), of the emulation with P rounded toward zero, and of the emulation with l summed from P16 all
fail it on the unit-logit family.

Inputs are built so that a wrong kernel fails.  q and k are multiples of 1/8 (|x| <= 255), so every logit sum is exact in
fp32.  Families: unit logits (std 2.25); every logit of a row in about [-1000, -150] (a max started at 0 underflows every
P16); the row max rising by ~30 per key block (alpha ~ 1e-13 at every step: prologue, steady state and drain); the row max in
the first block with later blocks' P in fp16's subnormal and zero range; q = 0 (the output is the mean of the valid v);
one head with V of 1e3 and three heads of one-hot rows (logit gap 110); single valid keys, single invalid keys and masks
with holes.  The per-key offsets of these families ride on the last four head dimensions (q = 8, k = offset / 4).  Padded
and out-of-sample key rows hold +-6e4 in k and v (finite: 0 * NaN would be NaN in P V), so a key let through the mask moves
the output far.  Every output buffer starts as NaN and has spare NaN rows after the last sample; varlen samples are placed
with gaps, one at an odd row, the last ending at the buffer's end (its tail tile is zero-filled by TMA), and rows outside
every sample must keep their NaN.

Across paths the results must be bit-identical: dense + key_mask without the list (ballot words), with it (blk_words table),
varlen (words computed from len) and dense unmasked at L = len, and a relaunch; skipping blocks without a valid key changes
nothing, as the kernel's header states.

Worst tau needed by the tight check, measured on an H100 80GB HBM3 (700 W limit); the provable check held without any tau
everywhere.  The unit-logit error grows with the number of keys (fp32 sums over L keys: 5.9e-6 at L = 4000):
  unit logits (all its tests)   1.16e-5 (L = 8192)   tau 4e-5
  logits in [-1000, -150]       1.74e-5 (L = 129)    tau 6e-5      (fp32 rounding of r c ~ 1e3 shifts whole blocks)
  max rising per block          1.45e-5 (L = 4000)   tau 5.5e-5
  max in the first block        1.21e-5 (L = 8192)   tau 4e-5
  q = 0                         3.7e-9  (L = 8192)   tau 1.4e-8
  V of 1e3, one-hot heads       3.9e-7  (L = 4000)   tau 1.5e-6
"""
import math

import pytest
import torch

gpu = pytest.mark.gpu

NAN = float("nan")
INF = float("inf")
PAD = 6.0e4                                                         # k and v of padded / out-of-sample key rows
SPARE = 128                                                         # NaN rows after the last sample of every output
SENTINEL = 0x5A5A5A5A                                               # scratch entries the block list must not write
C_KERNEL = float(torch.tensor(math.log2(math.e), dtype=torch.float32)) / 8   # the kernel's scale_log2
C_EXACT = math.log2(math.e) / 8
FAMILIES = ["unit", "negative", "rising", "first_block", "zero_q", "mixed"]
# one tau per family (tight and provable checks alike), at most 4x the worst measured
TAU = {"unit": 4e-5, "negative": 6e-5, "rising": 5.5e-5, "first_block": 4e-5, "zero_q": 1.4e-8, "mixed": 1.5e-6}


def _ffi():
    from brepgen_b200 import _ffi
    return _ffi


def ptr(t):
    return None if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------------ float64 references
def fp16_round(x, toward_zero=False):
    """x (float64) rounded to the nearest fp16 value, ties to even (or toward zero), subnormals included; |x| < 65520"""
    _, e = torch.frexp(x)
    ulp = torch.exp2((e.to(x.dtype) - 11).clamp_min(-24))
    y = x / ulp
    return (torch.trunc(y) if toward_zero else torch.round(y)) * ulp


def half_ulp16(x):
    _, e = torch.frexp(x)
    e = torch.where(x == 0, -100, e)
    return torch.exp2((e.to(x.dtype) - 12).clamp_min(-25))


def emulate(q, k, v, valid, blocks=None, c=C_KERNEL, p_round=fp16_round, l_from_p16=False):
    """the kernel's operation in float64 for query rows q (nq, 64) over keys k, v (nk, 64), valid (nk,) bool, visiting the
    128-key `blocks` in order (default: all).  Returns mu, A, amb, sv (nq, 64): the output, the row magnitude sum p |v| / l,
    the allowance for P16 roundings the kernel's fp32 p may take the other way, and sum |v| over the valid keys / l."""
    nq, nk = q.shape[0], k.shape[0]
    if blocks is None:
        blocks = range((nk + 127) // 128)
    blocks = torch.as_tensor(list(blocks), dtype=torch.long, device=q.device)
    nb = blocks.numel()
    if nb == 0:
        z = torch.zeros_like(q)
        return z, z, z, z
    idx = (blocks[:, None] * 128 + torch.arange(128, device=q.device)).reshape(-1)
    ok = idx < nk
    idx = idx.clamp_max(nk - 1)
    ok &= valid[idx]
    vv = torch.where(ok[:, None], v[idx], 0.0)
    s = (q @ k[idx].T).masked_fill(~ok, -INF).view(nq, nb, 128)
    m = s.amax(-1).cummax(1).values
    none = m == -INF
    r = torch.where(none, 0.0, m)
    x = c * (s - r[..., None])
    p = torch.exp2(x)
    scale = torch.where(none, 0.0, torch.exp2(c * (r - r[:, -1:])))[..., None]
    P16 = p_round(p)
    rho = math.log(2) * 2.0 ** -24 * ((c * r).abs()[..., None] + x.clamp_min(-1e4).abs()) + 2.0 ** -21
    amb_w = ((fp16_round(p * (1 + rho)) - fp16_round(p * (1 - rho))) * scale).view(nq, -1)
    pw = (p * scale).view(nq, -1)
    w = (P16 * scale).view(nq, -1)
    l = (w if l_from_p16 else pw).sum(-1, keepdim=True)
    l = torch.where(l > 0, l, 1.0)
    va = vv.abs()
    return (w @ vv) / l, (pw @ va) / l, (amb_w @ va) / l, va.sum(0, keepdim=True) / l


def plain(q, k, v, valid):
    """softmax(q k^T / 8 + mask) v in float64 (over the valid keys only); 0 for rows without a valid key"""
    k, v = k[valid], v[valid]
    return torch.softmax(q @ k.T / 8, -1) @ v


def needed_tau(y, q, k, v, valid, blocks=None):
    """per element, the tau the tight and the provable check need for output y (nq, 64) (0 where they hold without it)"""
    mu, A, amb, sv = emulate(q, k, v, valid, blocks)
    pl = plain(q, k, v, valid)
    yd = y.double()
    ex_t = (yd - mu).abs() - half_ulp16(torch.maximum(yd.abs(), mu.abs())) - amb
    ex_p = (yd - pl).abs() - half_ulp16(torch.maximum(yd.abs(), pl.abs())) - 2.0 ** -11 * A - 2.0 ** -25 * sv
    return (torch.where(ex_t > 0, ex_t / A, 0.0), torch.where(ex_p > 0, ex_p / A, 0.0))


class Worst:
    """worst tau needed over the checks of one test"""

    def __init__(self, tag, tau):
        self.tag, self.tau, self.tight, self.prov = tag, tau, 0.0, 0.0

    def check(self, what, y, qkv_rows, h, valid, q_rows=None, chunk=512):
        """y (nq, 64): the head-h output of query rows q_rows (default all) of one sample whose rows are qkv_rows"""
        assert torch.isfinite(y).all(), f"{self.tag} {what}: non-finite output"
        x = qkv_rows.double()
        q = x[:, h * 64:(h + 1) * 64] if q_rows is None else x[q_rows, h * 64:(h + 1) * 64]
        k, v = x[:, 768 + h * 64:768 + (h + 1) * 64], x[:, 1536 + h * 64:1536 + (h + 1) * 64]
        blocks = [kb for kb in range((k.shape[0] + 127) // 128) if valid[kb * 128:(kb + 1) * 128].any()]
        for i in range(0, q.shape[0], chunk):
            t, pv = needed_tau(y[i:i + chunk], q[i:i + chunk], k, v, valid, blocks)
            wt, wp = float(t.max()), float(pv.max())
            self.tight, self.prov = max(self.tight, wt), max(self.prov, wp)
            assert wt <= self.tau, f"{self.tag} {what} head {h}: tight check needs tau {wt:.2e} > {self.tau:.1e}"
            assert wp <= self.tau, f"{self.tag} {what} head {h}: provable check needs tau {wp:.2e} > {self.tau:.1e}"

    def report(self):
        print(f"{self.tag}: worst tau needed tight {self.tight:.2e}, provable {self.prov:.2e} (bar {self.tau:.1e})")


# ------------------------------------------------------------------------------------------------ inputs
def eighths(g, shape, std, device):
    return (torch.randn(shape, generator=g, device=device) * (8 * std)).round().clamp(-2040, 2040) / 8


def sample_rows(n, family, seed, valid, device="cuda"):
    """the fp16 qkv rows (n, 2304) of one sample of `family`; key rows outside `valid` hold +-6e4 in k and v"""
    g = torch.Generator(device=device).manual_seed(seed)
    shape = (n, 12, 64)
    std = 1.5 if family == "unit" else 1.0
    q, k = eighths(g, shape, std, device), eighths(g, shape, std, device)
    v = torch.randn(shape, generator=g, device=device)
    kb = (torch.arange(n, device=device) // 128)[:, None].float()
    u = torch.rand((n, 12), generator=g, device=device)
    off = None
    if family == "negative":
        off = -150 - 850 * u
    elif family == "rising":
        off = 30 * kb - 15 * ((n + 127) // 128) + 0 * u
    elif family == "first_block":
        off = torch.where(kb == 0, 0.0, -6 - 16 * u)
    elif family == "zero_q":
        q.zero_()
    elif family == "mixed":
        v[:, 3] *= 1e3
        off = torch.zeros_like(u)
        keys = valid.nonzero().flatten()
        for h, key in ((5, keys[0]), (6, keys[keys.numel() // 2]), (7, keys[-1])):
            off[:, h] = -110
            off[key, h] = 0
    if off is not None:
        q[..., 60:] = 8
        k[..., 60:] = ((off * 2).round() / 8)[..., None]
    sign = torch.where(torch.rand((n, 2, 12, 64), generator=g, device=device) < 0.5, -PAD, PAD)
    inval = ~valid.to(device)[:, None, None]
    k = torch.where(inval, sign[:, 0], k)
    v = torch.where(inval, sign[:, 1], v)
    return torch.cat([q, k, v], 1).reshape(n, 2304).half()


def gap_rows(n, seed):
    """rows that belong to no sample: q random, k and v +-6e4"""
    return sample_rows(n, "unit", seed, torch.zeros(n, dtype=torch.bool, device="cuda"))


# ------------------------------------------------------------------------------------------------ kernel launches
def run_dense(qkv, B, L, mask=None, use_list=False):
    """bg_op_attention -> out (B L, 768) and the scratch (or None); rows past the last sample must stay NaN"""
    f = _ffi()
    nkb = (L + 127) // 128
    out = torch.full((B * L + SPARE, 768), NAN, dtype=torch.float16, device="cuda")
    scratch = torch.full((B * (5 * nkb + 1),), SENTINEL, dtype=torch.int32, device="cuda") if use_list else None
    f.check(f.lib().bg_op_attention(qkv.data_ptr(), out.data_ptr(), B, L, ptr(mask), int(use_list), ptr(scratch),
                                    f.current_stream()), "attention")
    torch.cuda.synchronize()
    assert out[B * L:].isnan().all(), "rows past the last sample were written"
    return out[:B * L], scratch


def run_varlen(qkv, B, L, row0, lens):
    """bg_op_attention_varlen over qkv (B L rows) -> out (B L, 768); rows outside every sample must stay NaN"""
    f = _ffi()
    r0 = torch.tensor(row0, dtype=torch.int32, device="cuda")
    ln = torch.tensor(lens, dtype=torch.int32, device="cuda")
    out = torch.full((B * L + SPARE, 768), NAN, dtype=torch.float16, device="cuda")
    f.check(f.lib().bg_op_attention_varlen(qkv.data_ptr(), out.data_ptr(), B, L, r0.data_ptr(), ln.data_ptr(),
                                           f.current_stream()), "attention varlen")
    torch.cuda.synchronize()
    outside = torch.ones(B * L + SPARE, dtype=torch.bool, device="cuda")
    for r, n in zip(row0, lens):
        outside[r:r + n] = False
    assert out[outside].isnan().all(), "varlen wrote rows outside every sample"
    return out[:B * L]


def same(a, b, what):
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{what}: results differ"


def tail_lengths(L):
    return [L, max(1, 2 * L // 3 + 1), max(1, L // 5)]


# ------------------------------------------------------------------------------------------------ GPU tests
LS = [1, 2, 63, 64, 65, 100, 127, 128, 129, 255, 256, 257, 2000, 4000, 8192]


@gpu
@pytest.mark.parametrize("L", LS)
@pytest.mark.parametrize("family", FAMILIES)
def test_family_paths(family, L):
    """three tail-padded samples (lengths L, ~2L/3, ~L/5) through all four paths: dense + key_mask (checked against both
    references, padded query rows included), the same with the block list, varlen with gaps, and dense unmasked at L = len;
    all bit-identical on the valid rows, and a relaunch bit-identical to the first launch"""
    B, lens = 3, tail_lengths(L)
    seed = 1000 * FAMILIES.index(family) + L
    ar = torch.arange(L, device="cuda")
    valid = [ar < n for n in lens]
    rows = [sample_rows(L, family, seed + b, valid[b]) for b in range(B)]
    qkv = torch.cat(rows)
    mask = torch.stack([~vb for vb in valid])

    out, _ = run_dense(qkv, B, L, mask)
    again, _ = run_dense(qkv, B, L, mask)
    same(out, again, "relaunch")
    listed, _ = run_dense(qkv, B, L, mask, use_list=True)
    same(out, listed, "with and without the block list")

    # varlen: a gap of 3 rows (odd row0), a gap of 5, the last sample ending at the buffer's end; B * Lv rows
    Lv = min(L + 8, 8192)
    row0 = [3, 8 + lens[0], B * Lv - lens[2]]
    qv = gap_rows(B * Lv, seed + 7)
    for b in range(B):
        qv[row0[b]:row0[b] + lens[b]] = rows[b][:lens[b]]
    vout = run_varlen(qv, B, Lv, row0, lens)
    for b in range(B):
        same(vout[row0[b]:row0[b] + lens[b]], out[b * L:b * L + lens[b]], f"varlen sample {b}")
        one, _ = run_dense(rows[b][:lens[b]].contiguous(), 1, lens[b])
        same(one, out[b * L:b * L + lens[b]], f"dense unmasked at L = len, sample {b}")

    w = Worst(f"{family} L={L}", TAU[family])
    for b in range(B):
        for h in range(12):
            w.check(f"sample {b}", out[b * L:(b + 1) * L, h * 64:(h + 1) * 64], rows[b], h, valid[b])
    w.report()


def mask_kind(kind, B, L, g):
    """(B, L) bool, True = padded key"""
    ar = torch.arange(L, device="cuda")
    if kind == "one_valid":
        # the single valid key at positions 0, 31, 32, 127 of a block past the first, and at the last key
        kb = max(1, (L // 128) // 2)
        keys = [kb * 128 + i for i in (0, 31, 32, 127)] + [L - 1]
        return torch.stack([ar != key for key in keys])
    if kind == "one_invalid":
        keys = [0, 127, 128, L - 1, L // 2 + 3]
        return torch.stack([ar == key for key in keys])
    # holes: random keys, a fully padded block in the middle, a fully padded first block, a sparse sample
    mask = torch.rand(B, L, generator=g, device="cuda") < 0.3
    nkb = (L + 127) // 128
    mask[0, (nkb // 2) * 128:(nkb // 2 + 1) * 128] = True
    mask[1, :128] = True
    mask[2] = torch.rand(L, generator=g, device="cuda") < 0.97
    mask[2, L - 1] = False
    mask[3, ::2] = True
    mask[4, 1::2] = True
    return mask


@gpu
@pytest.mark.parametrize("L", [257, 1000, 4000])
@pytest.mark.parametrize("kind", ["one_valid", "one_invalid", "holes"])
def test_masks(kind, L):
    """unit logits under masks with exactly one valid key (positions 0, 31, 32, 127 of a block, and the last key), one
    invalid key, or holes; dense with and without the block list, bit-identical"""
    B = 5
    g = torch.Generator(device="cuda").manual_seed(L + len(kind))
    mask = mask_kind(kind, B, L, g)
    rows = [sample_rows(L, "unit", 77 * L + b, ~mask[b]) for b in range(B)]
    qkv = torch.cat(rows)
    out, _ = run_dense(qkv, B, L, mask)
    listed, _ = run_dense(qkv, B, L, mask, use_list=True)
    same(out, listed, "with and without the block list")
    w = Worst(f"masks {kind} L={L}", TAU["unit"])
    for b in range(B):
        for h in range(12):
            w.check(f"sample {b}", out[b * L:(b + 1) * L, h * 64:(h + 1) * 64], rows[b], h, ~mask[b])
    w.report()


@gpu
@pytest.mark.parametrize("stage,L", [("surface", 30), ("surface", 50), ("surface", 100), ("edge", 2000), ("edge", 4000)])
def test_production_shapes(stage, L):
    """B = 64 tail-padded samples of unit logits as the denoisers run them: dense + key_mask with and without the block
    list, and the compacted varlen form (samples packed back to back); bit-identical.  Every sample is checked against
    the references at the surface stage, every fourth at the edge stage."""
    B = 64
    g = torch.Generator().manual_seed(L)
    lens = torch.randint(max(1, L // 4), L + 1, (B,), generator=g).tolist()
    lens[0], lens[1] = L, 1
    ar = torch.arange(L, device="cuda")
    valid = [ar < n for n in lens]
    rows = [sample_rows(L, "unit", 5 * L + b, valid[b]) for b in range(B)]
    qkv = torch.cat(rows)
    mask = torch.stack([~vb for vb in valid])
    out, _ = run_dense(qkv, B, L, mask)
    listed, _ = run_dense(qkv, B, L, mask, use_list=True)
    same(out, listed, "with and without the block list")
    row0 = [0] + torch.tensor(lens).cumsum(0)[:-1].tolist()
    qv = gap_rows(B * L, L + 1)
    for b in range(B):
        qv[row0[b]:row0[b] + lens[b]] = rows[b][:lens[b]]
    vout = run_varlen(qv, B, L, row0, lens)
    for b in range(B):
        same(vout[row0[b]:row0[b] + lens[b]], out[b * L:b * L + lens[b]], f"compacted varlen sample {b}")
    w = Worst(f"{stage} B=64 L={L}", TAU["unit"])
    for b in range(0, B, 1 if stage == "surface" else 4):
        for h in range(12):
            w.check(f"sample {b}", out[b * L:(b + 1) * L, h * 64:(h + 1) * 64], rows[b], h, valid[b])
    w.report()


def expected_scratch(mask, L):
    """the block list, counts and invalid-key words bg_op_attention must leave in its scratch, unwritten entries kept"""
    B = mask.shape[0]
    nkb = (L + 127) // 128
    bad = torch.ones(B, nkb * 128, dtype=torch.bool)
    bad[:, :L] = mask.cpu()
    bits = bad.view(B, nkb, 4, 32).long() << torch.arange(32)
    words = bits.sum(-1)                                              # (B, nkb, 4) as int64 in [0, 2^32)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).int()
    exp = torch.full((B * (5 * nkb + 1),), SENTINEL, dtype=torch.int32)
    blk_list, cnt, wds = exp[:B * nkb].view(B, nkb), exp[B * nkb:B * (nkb + 1)], exp[B * (nkb + 1):].view(B, nkb, 4)
    for b in range(B):
        listed = [kb for kb in range(nkb) if not bool(bad[b, kb * 128:(kb + 1) * 128].all())]
        cnt[b] = len(listed)
        for i, kb in enumerate(listed):
            blk_list[b, i] = kb
            wds[b, i] = words[b, kb]
    return exp


@gpu
@pytest.mark.parametrize("L", [1000, 4000, 8192])
@pytest.mark.parametrize("kind", ["random", "ragged", "all_padded"])
def test_block_list_contents(kind, L):
    """blk_list (list order), blk_count and blk_words (the listed blocks' invalid-key words in list order, keys >= L set),
    read back from the scratch, equal a Python construction exactly; the entries past each count stay unwritten"""
    B = 3
    g = torch.Generator(device="cuda").manual_seed(L)
    nkb = (L + 127) // 128
    if kind == "random":
        # every key block padded with its own probability: all, 99.5 %, half or none of its keys
        dens = torch.tensor([1.0, 0.995, 0.5, 0.0], device="cuda")[torch.randint(0, 4, (B, nkb), generator=g,
                                                                                 device="cuda")]
        mask = torch.rand(B, nkb * 128, generator=g, device="cuda") < dens.repeat_interleave(128, 1)
        mask = mask[:, :L].contiguous()
    elif kind == "ragged":
        ar = torch.arange(L, device="cuda")
        mask = torch.stack([ar >= n for n in (L, L // 2 + 7, 129)])
    else:
        mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
        mask[1] = True
        mask[2, :L - 1] = True
    qkv = torch.zeros(B * L, 2304, dtype=torch.float16, device="cuda")
    _, scratch = run_dense(qkv, B, L, mask, use_list=True)
    exp = expected_scratch(mask, L)
    got = scratch.cpu()
    assert torch.equal(got[:B * nkb], exp[:B * nkb]), "blk_list"
    assert torch.equal(got[B * nkb:B * (nkb + 1)], exp[B * nkb:B * (nkb + 1)]), "blk_count"
    assert torch.equal(got, exp), "blk_words"


@gpu
@pytest.mark.parametrize("use_list", [False, True])
def test_all_padded_sample_gives_zeros(use_list):
    """a sample with every key padded gives exact zeros, with and without the block list; its neighbours are unaffected"""
    B, L = 3, 300
    mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    mask[1] = True
    mask[2, 200:] = True
    rows = [sample_rows(L, "unit", 90 + b, ~mask[b]) for b in range(B)]
    out, _ = run_dense(torch.cat(rows), B, L, mask, use_list=use_list)
    assert torch.equal(out[L:2 * L], torch.zeros_like(out[L:2 * L])), "a sample without a valid key must give zeros"
    w = Worst(f"all padded, list {use_list}", TAU["unit"])
    for b in (0, 2):
        for h in range(12):
            w.check(f"sample {b}", out[b * L:(b + 1) * L, h * 64:(h + 1) * 64], rows[b], h, ~mask[b])
    w.report()


@gpu
@pytest.mark.parametrize("mode", ["dense", "block_list", "varlen"])
def test_rejects_sequence_over_8192(mode):
    """L = 8193 returns status -1 with a message and launches nothing (the block list included)"""
    f = _ffi()
    B, L = 1, 8193
    nkb = (L + 127) // 128
    qkv = torch.zeros(B * L, 2304, dtype=torch.float16, device="cuda")
    out = torch.full((B * L, 768), NAN, dtype=torch.float16, device="cuda")
    mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    scratch = torch.full((B * (5 * nkb + 1),), SENTINEL, dtype=torch.int32, device="cuda")
    ints = torch.tensor([0, L], dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    n0 = f.lib().bg_launch_count()
    if mode == "varlen":
        st = f.lib().bg_op_attention_varlen(qkv.data_ptr(), out.data_ptr(), B, L, ints[:1].data_ptr(),
                                            ints[1:].data_ptr(), f.current_stream())
    else:
        st = f.lib().bg_op_attention(qkv.data_ptr(), out.data_ptr(), B, L, mask.data_ptr(), int(mode == "block_list"),
                                     scratch.data_ptr(), f.current_stream())
    torch.cuda.synchronize()
    assert st == -1, st
    assert b"8192" in f.lib().bg_last_error()
    assert f.lib().bg_launch_count() == n0, "a rejected call launched a kernel"
    assert (scratch == SENTINEL).all() and out.isnan().all()


@gpu
def test_sequence_of_8192_with_block_list():
    """L = 8192, the longest accepted, with the block list skipping padded blocks in the middle; against both references"""
    B, L = 1, 8192
    mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    mask[0, 1024:3000] = True
    rows = sample_rows(L, "unit", 8192, ~mask[0])
    out, scratch = run_dense(rows, B, L, mask, use_list=True)
    nkb = L // 128
    assert int(scratch[nkb]) == nkb - 15
    ref, _ = run_dense(rows, B, L, mask)
    same(out, ref, "with and without the block list")
    w = Worst("L=8192 listed", TAU["unit"])
    for h in (0, 11):
        w.check("sample 0", out[:, h * 64:(h + 1) * 64], rows, h, ~mask[0])
    w.report()


# ------------------------------------------------------------------------------------------------ CPU tests
def _cpu_rows(n, family, seed, nvalid):
    valid = torch.arange(n) < nvalid
    return sample_rows(n, family, seed, valid, device="cpu").double(), valid


def _qkv(x, h):
    return (x[:, i * 768 + h * 64:i * 768 + (h + 1) * 64] for i in range(3))


def _no_rounding(p):
    return p


@pytest.mark.parametrize("case", ["one_block", "32_blocks_max_rises_and_falls", "padded_blocks_skipped"])
def test_emulation_without_rounding_is_softmax(case):
    """with fp16 rounding of P switched off (and the exact log2 e), the block-by-block emulation is the plain softmax"""
    if case == "one_block":
        x, valid = _cpu_rows(100, "unit", 1, 90)
        blocks = None
    else:
        n = 32 * 128
        x, valid = _cpu_rows(n, "unit", 2, n)
        if case == "32_blocks_max_rises_and_falls":
            # per-block offsets that rise and fall by up to 40, carried by the last four head dimensions
            kb = torch.arange(n) // 128
            off = (40 * torch.sin(kb.double() * 1.3)).round()
            x[:, 60:64] = 8
            x[:, 768 + 60:768 + 64] = (off / 4)[:, None]
            blocks = None
        else:
            for kb in (0, 5, 6, 7, 20, 31):
                valid[kb * 128:(kb + 1) * 128] = False
            blocks = [kb for kb in range(32) if valid[kb * 128:(kb + 1) * 128].any()]
    q, k, v = _qkv(x, 0)
    mu, A, _, _ = emulate(q, k, v, valid, blocks, c=C_EXACT, p_round=_no_rounding)
    ref = plain(q, k, v, valid)
    err = float(((mu - ref).abs() / A.clamp_min(1e-300)).max())
    print(f"{case}: emulation without rounding vs softmax {err:.1e}")
    assert err <= 1e-12, err


def test_zero_q_gives_the_exact_mean():
    """q = 0: every logit is 0, so every P16 is 1 and the emulation is the fp64 mean of the valid v"""
    x, valid = _cpu_rows(700, "zero_q", 3, 533)
    for h in (0, 7):
        q, k, v = _qkv(x, h)
        mu, _, amb, _ = emulate(q, k, v, valid)
        mean = v[valid].mean(0, keepdim=True).expand_as(mu)
        assert float((mu - mean).abs().max()) <= 1e-15 * float(mean.abs().max())
        assert float(amb.max()) == 0.0


def test_fp16_round():
    """fp16_round is torch's fp32 -> fp16 conversion (round to nearest even, subnormals included) on fp32 values"""
    g = torch.Generator().manual_seed(4)
    x = torch.cat([torch.exp2(torch.rand(100000, generator=g) * 40 - 30),
                   torch.arange(0, 4096).float() * 2.0 ** -25]).float()
    assert torch.equal(fp16_round(x.double()), x.half().double())


# fake "kernel outputs" on the unit-logit family and how many of their elements violate the tight check (of 3 x 257 x
# 12 x 64 = 592128); each must fail it
# measured: 48458, 172624 and 533
FAKE_MIN_VIOLATIONS = {"P not rounded": 24000, "P rounded toward zero": 86000, "l summed from P16": 250}


def test_checker_power():
    """fp16 of the plain softmax (P not rounded), of the emulation with P rounded toward zero, and of the emulation with l
    summed from P16 each fail the tight check on unit logits; fp16 of the emulation itself passes it"""
    counts = dict.fromkeys(FAKE_MIN_VIOLATIONS, 0)
    n_exact = 0
    tau = TAU["unit"]
    L = 257
    for b, n in enumerate(tail_lengths(L)):
        x, valid = _cpu_rows(L, "unit", 50 + b, n)
        for h in range(12):
            q, k, v = _qkv(x, h)
            fakes = {
                "P not rounded": plain(q, k, v, valid),
                "P rounded toward zero": emulate(q, k, v, valid, p_round=lambda p: fp16_round(p, toward_zero=True))[0],
                "l summed from P16": emulate(q, k, v, valid, l_from_p16=True)[0],
            }
            mu = emulate(q, k, v, valid)[0]
            t, _ = needed_tau(mu.half(), q, k, v, valid)
            n_exact += int((t > tau).sum())
            for name, y in fakes.items():
                t, _ = needed_tau(y.half(), q, k, v, valid)
                counts[name] += int((t > tau).sum())
    print(f"tight-check violations at tau {tau:.1e}: {counts}; fp16 of the emulation: {n_exact}")
    assert n_exact == 0
    for name, c in counts.items():
        assert c >= FAKE_MIN_VIOLATIONS[name], (name, c)
