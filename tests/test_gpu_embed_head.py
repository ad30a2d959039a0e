"""Op-level parity of the denoisers' CUDA-core ends (elementwise.cu) through their unit-level entry points: the first
kernel of every forward (embed_in: Linear -> LayerNorm -> SiLU -> fp16, gathering source rows through token compaction's
row_map), the last one (ln_silu_head: LayerNorm -> SiLU -> Linear in fp32, scattering rows back through row_map) and the
compaction itself (seq_len, seq_row0, m_valid, row_map of a key-padding mask).

The references are the oracle's own statements run in float64: embed_in is the front of oracle.denoisers.embed_mlp up to
its second Linear, ln_silu_head the back of it from the LayerNorm on (the two GEMMs in between run on the tensor cores and
are pinned elsewhere).  The CPU tests at the end check that both helpers recompose oracle.denoisers.embed_mlp in fp32.

Bars: ln_silu_head |y - y64| <= 2e-6 max(1, |y64|) per element; embed_in writes fp16, so each output must be the fp16
rounding of the reference up to 2e-6 max(1, |y64|) (its distance from y64 beyond half an fp16 ulp); compaction exact.  Rows at
or past *rows_dev are never written (they keep their NaN), and the scattered head rows land exactly at row_map[r].

Worst errors measured on an H100 80GB HBM3 (700 W limit); the tests print them, and the bars are at most 4x above:
  embed_in      6.3e-7 beyond fp16 rounding
  ln_silu_head  5.5e-7
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import denoisers as O

gpu = pytest.mark.gpu

NAN = float("nan")
D = 768
TAU = 2e-6


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
def _sd64(sd):
    return {k: v.double() for k, v in sd.items()}


def embed_ref(sd, name, x):
    """SiLU(LayerNorm(Linear .0 (x))): oracle.denoisers.embed_mlp before its Linear .3, in float64"""
    sd = _sd64(sd)
    return F.silu(O._ln(O._lin(x.double(), sd, name + ".0"), sd, name + ".1"))


def head_ref(sd, name, h):
    """Linear .3 (SiLU(LayerNorm .1 (h))): oracle.denoisers.embed_mlp after its Linear .0, in float64"""
    sd = _sd64(sd)
    return O._lin(F.silu(O._ln(h.double(), sd, name + ".1")), sd, name + ".3")


def compact_ref(mask):
    """mask (B, L) bool, True = padded -> seq_len, seq_row0 (exclusive prefix sum), m_valid, row_map (valid b * L + t in
    order), all int32 numpy"""
    valid = ~mask
    seq_len = valid.sum(1).astype(np.int32)
    seq_row0 = (np.cumsum(seq_len) - seq_len).astype(np.int32)
    return seq_len, seq_row0, int(seq_len.sum()), np.flatnonzero(valid.reshape(-1)).astype(np.int32)


def mlp_sd(d_in, d_out, g):
    """weights of one embed MLP / fc_out (Linear d_in -> 768, LayerNorm, SiLU, Linear 768 -> d_out)"""
    r = lambda *s: torch.randn(*s, generator=g)
    return {"m.0.weight": r(D, d_in) / d_in ** 0.5, "m.0.bias": 0.5 * r(D), "m.1.weight": 1 + 0.2 * r(D),
            "m.1.bias": 0.2 * r(D), "m.3.weight": r(d_out, D) / D ** 0.5, "m.3.bias": 0.5 * r(d_out)}


# ------------------------------------------------------------------------------------------------ row maps
M_ROWS = 9001          # more rows than one pass of either kernel's grid covers (8 rows per 256-thread block)


def row_mode(mode, M, g):
    """(rows_dev, row_map, k): None / None / M, or the device row count `mode` with a shuffled permutation as the map"""
    if mode == "plain":
        return None, None, M
    k = {"0": 0, "1": 1, "M-1": M - 1, "M": M}[mode]
    row_map = torch.randperm(M, generator=g).int()
    return torch.tensor([k], dtype=torch.int32).cuda(), row_map.cuda(), k


MODES = ["plain", "0", "1", "M-1", "M"]


# ------------------------------------------------------------------------------------------------ embed_in
# (d_in, source pitch, source column, output pitch, output column): SurfPosNet / SurfZNet p_embed and EdgePosNet's embeds
# (pitch 6), SurfZNet / the edge nets' z embeds (48), EdgeZNet's edgez_embed / vertp_fc from x (pitch 18, columns 0 / 12)
EMBED = [(6, 6, 0, D, 0), (48, 48, 0, 2 * D, 0), (6, 6, 0, 2 * D, D), (12, 18, 0, 3 * D, D), (6, 18, 12, 3 * D, 2 * D)]


@gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("d_in,ldx,col,ldy,ycol", EMBED)
def test_embed_in(d_in, ldx, col, ldy, ycol, mode):
    M = M_ROWS
    g = torch.Generator().manual_seed(d_in * 100 + ldx + col + MODES.index(mode))
    sd = mlp_sd(d_in, 8, g)
    src = (2 * torch.randn(M, ldx, generator=g)).cuda()
    rows_dev, row_map, k = row_mode(mode, M, g)
    W0t = sd["m.0.weight"].t().contiguous().cuda()
    b0, gam, bet = (sd[n].cuda() for n in ("m.0.bias", "m.1.weight", "m.1.bias"))
    y = torch.full((M, ldy), NAN, device="cuda", dtype=torch.float16)
    call("bg_op_embed_in", src.data_ptr() + 4 * col, ldx, d_in, p(W0t), p(b0), p(gam), p(bet), y.data_ptr() + 2 * ycol, ldy,
         M, p(rows_dev), p(row_map))
    out = y[:, ycol:ycol + D]
    rest = torch.cat([y[:, :ycol], y[:, ycol + D:]], 1)
    assert torch.isnan(rest).all(), "columns outside the output block were written"
    assert torch.isnan(out[k:]).all(), "rows at or past the device row count were written"
    if k == 0:
        return
    srows = row_map[:k].long() if row_map is not None else torch.arange(k, device="cuda")
    ref = embed_ref(sd, "m", src[srows, col:col + d_in].cpu()).cuda()
    got = out[:k]
    assert torch.isfinite(got).all()
    half_ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 11)
    excess = float((((got.double() - ref).abs() - half_ulp) / ref.abs().clamp_min(1.0)).max())
    print(f"embed_in d_in={d_in} pitch={ldx} col={col} {mode}: rows {k}/{M}, worst excess over fp16 rounding {excess:.2e}")
    assert excess <= TAU, excess


# ------------------------------------------------------------------------------------------------ ln_silu_head
@gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("d_out", [6, 18, 32, 48, 64])
def test_ln_silu_head(d_out, mode):
    """d_out 6 / 48 / 6 / 18 of the four nets, plus 32 and 64: whole and partial 32-column groups of the store loop"""
    M = M_ROWS
    g = torch.Generator().manual_seed(d_out * 10 + MODES.index(mode))
    sd = mlp_sd(8, d_out, g)
    x = (3 * torch.randn(M, D, generator=g) + torch.randn(M, 1, generator=g)).cuda()
    rows_dev, row_map, k = row_mode(mode, M, g)
    gam, bet, W, bias = (sd[n].cuda() for n in ("m.1.weight", "m.1.bias", "m.3.weight", "m.3.bias"))
    out = torch.full((M, d_out), NAN, device="cuda")
    call("bg_op_ln_silu_head", p(x), D, p(gam), p(bet), p(W), p(bias), p(out), d_out, M, p(rows_dev), p(row_map))
    drows = row_map[:k].long() if row_map is not None else torch.arange(k, device="cuda")
    written = torch.zeros(M, dtype=torch.bool, device="cuda")
    written[drows] = True
    assert torch.isnan(out[~written]).all(), "rows that no valid row maps to were written"
    if k == 0:
        return
    ref = head_ref(sd, "m", x[:k].cpu()).cuda()
    got = out[drows]
    assert torch.isfinite(got).all(), "a valid row's output is missing or non-finite"
    e = float(((got.double() - ref).abs() / ref.abs().clamp_min(1.0)).max())
    print(f"ln_silu_head d_out={d_out} {mode}: rows {k}/{M}, max elementwise error {e:.2e} (bar {TAU:.1e})")
    assert e <= TAU, e


# ------------------------------------------------------------------------------------------------ compaction
def make_mask(kind, B, L, g):
    if kind == "all_valid":
        return np.zeros((B, L), bool)
    if kind == "one_padded":        # random, with one sample all padded and one all valid
        m = g.random((B, L)) < 0.4
        m[B // 2] = True
        m[0] = False
        return m
    if kind == "single":            # one valid token in the whole batch, in the last sample's last position
        m = np.ones((B, L), bool)
        m[B - 1, L - 1] = False
        return m
    return g.random((B, L)) < g.random((B, 1))     # random, a different padding rate per sample


def run_compact(B, L, kind):
    g = np.random.default_rng(L * 10 + len(kind) + (0 if B == 64 else B * 100000))
    mask = make_mask(kind, B, L, g)
    seq_len = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    seq_row0, m_valid = seq_len.clone(), torch.full((1,), -7, dtype=torch.int32, device="cuda")
    row_map = torch.full((B * L,), -7, dtype=torch.int32, device="cuda")
    mdev = torch.from_numpy(mask.astype(np.uint8)).cuda()
    call("bg_op_compact", p(mdev), B, L, p(seq_len), p(seq_row0), p(m_valid), p(row_map))
    r_len, r_row0, r_m, r_map = compact_ref(mask)
    assert np.array_equal(seq_len.cpu().numpy(), r_len)
    assert np.array_equal(seq_row0.cpu().numpy(), r_row0)
    assert int(m_valid.item()) == r_m
    got = row_map.cpu().numpy()
    assert np.array_equal(got[:r_m], r_map), f"row_map differs at {np.flatnonzero(got[:r_m] != r_map)[:8]}"
    assert (got[r_m:] == -7).all(), "row_map entries past m_valid were written"


@gpu
@pytest.mark.parametrize("kind", ["all_valid", "one_padded", "single", "random"])
@pytest.mark.parametrize("L", [1, 31, 32, 33, 4000])
def test_compact(L, kind):
    run_compact(64, L, kind)


@gpu
@pytest.mark.parametrize("kind", ["all_valid", "single", "random"])
@pytest.mark.parametrize("L", [1, 33, 4000])
@pytest.mark.parametrize("B", [1, 3])
def test_compact_small_batch(B, L, kind):
    """one sample (seq_row0 is a single 0) and a batch smaller than a warp"""
    run_compact(B, L, kind)


# ------------------------------------------------------------------------------------------------ references vs oracle (CPU)
def test_embed_and_head_refs_recompose_the_oracle_mlp():
    g = torch.Generator().manual_seed(0)
    for d_in, d_out in ((6, 6), (48, 48), (12, 18)):
        sd = mlp_sd(d_in, d_out, g)
        x = torch.randn(50, d_in, generator=g)
        want = O.embed_mlp(sd, "m", x).double()
        via_embed = O._lin(embed_ref(sd, "m", x), _sd64(sd), "m.3")
        via_head = head_ref(sd, "m", O._lin(x.double(), _sd64(sd), "m.0"))
        for got in (via_embed, via_head):
            assert float((got - want).norm() / want.norm()) < 1e-5


def test_compact_ref():
    mask = np.array([[0, 1, 0, 0], [1, 1, 1, 1], [1, 0, 1, 0]], bool)
    seq_len, seq_row0, m, row_map = compact_ref(mask)
    assert seq_len.tolist() == [3, 0, 2] and seq_row0.tolist() == [0, 3, 3] and m == 5
    assert row_map.tolist() == [0, 2, 3, 9, 11]
