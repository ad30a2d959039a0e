"""The attention kernel's 192-row query tiles (csrc/attn.cu: three consumer warpgroups of 64 rows), through the C ABI.

A tile's last rows may lie beyond its sample, so a tile has 1, 2 or 3 consumer warpgroups with rows to compute; the
others skip the key loop, and the K / V ring's empty barriers must count only the warpgroups that take part.  The cases
put sample ends on either side of the 64-row warpgroup edges and the 192-row tile edges.  Every case is checked against
fp32 torch at the 2e-3 relative-L2 bar of test_gpu_ops.py; a second launch must reproduce the first bit for bit, and
rows that belong to no sample must be left as they were.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

BQ = 192   # query rows per CTA


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


def _attn_one(qkv_rows, keep=None):
    """softmax(q k^T / 8) v of one sample's rows [n, 2304], keys restricted to `keep` (bool [n]) if given -> [n, 768]"""
    n = qkv_rows.shape[0]
    q, k, v = qkv_rows.float().view(n, 3, 12, 64).permute(1, 2, 0, 3)   # (12, n, 64)
    s = q @ k.transpose(-1, -2) / 8.0
    if keep is not None:
        s = s.masked_fill(~keep.view(1, 1, n), float("-inf"))
    return (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(n, 768)


def _bits(t):
    return t.view(torch.int16)


def _last_tile_warpgroups(n):
    """consumer warpgroups with at least one row in the last query tile of a sample of n tokens"""
    return (n - (n - 1) // BQ * BQ + 63) // 64


def _launch_twice(launch, rows):
    """two launches into NaN-filled [rows, 768] buffers; they must agree bit for bit"""
    outs = []
    for _ in range(2):
        out = torch.full((rows, 768), float("nan"), device="cuda", dtype=torch.float16)
        launch(out)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "two launches on the same input differ"
    return outs[0]


def _assert_unwritten(out, rows):
    untouched = torch.isnan(out[rows].float()).all().item()
    assert untouched, "rows outside every sample were written"


def test_varlen_tile_edges():
    """one variable-length batch with sample ends at the 64-row warpgroup and 192-row tile edges: last tiles with 1, 2
    and 3 consumer warpgroups; 4000 ends in a 160-row tile.  Rows past the packed samples are not written."""
    f = _ffi()
    lens = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 383, 384, 385, 4000]
    assert {_last_tile_warpgroups(n) for n in lens} == {1, 2, 3}
    B, L = len(lens), 4000
    g = torch.Generator(device="cuda").manual_seed(31)
    lens_t = torch.tensor(lens, dtype=torch.int32, device="cuda")
    row0 = torch.zeros_like(lens_t)
    row0[1:] = torch.cumsum(lens_t, 0)[:-1]
    qkv = (torch.randn(B * L, 2304, generator=g, device="cuda") * 1.5).half()
    out = _launch_twice(lambda o: f.check(f.lib().bg_op_attention_varlen(
        qkv.data_ptr(), o.data_ptr(), B, L, row0.data_ptr(), lens_t.data_ptr(), f.current_stream()), "attention varlen"),
        B * L)
    _assert_unwritten(out, slice(sum(lens), B * L))
    for b, n in enumerate(lens):
        r = int(row0[b])
        got = out[r:r + n]
        assert torch.isfinite(got.float()).all(), f"sample {b} (len {n}) has non-finite rows"
        err = rel_l2(got.float(), _attn_one(qkv[r:r + n]))
        print(f"varlen len {n} ({_last_tile_warpgroups(n)} warpgroups in the last tile) rel_l2={err:.3e}")
        assert err < 2e-3, (n, err)


def _run_masked(qkv, B, L, mask, guard):
    """bg_op_attention with the block list into a buffer of B * L + guard rows; returns (out, listed block counts)"""
    f = _ffi()
    nkb = (L + 127) // 128
    scratch = torch.zeros(B * (5 * nkb + 1), dtype=torch.int32, device="cuda")
    out = _launch_twice(lambda o: f.check(f.lib().bg_op_attention(
        qkv.data_ptr(), o.data_ptr(), B, L, f.ptr(mask), 1, scratch.data_ptr(), f.current_stream()), "attention"),
        B * L + guard)
    _assert_unwritten(out, slice(B * L, B * L + guard))
    return out[:B * L].view(B, L, 768), scratch[B * nkb:B * nkb + B].tolist()


def test_block_list_three_tiles():
    """block-list mode at L = 576 (three whole 192-row tiles, five key blocks) with 0, 1, 2 and 3 listed blocks.  Sample
    0 has every key padded, so its rows must come out as exact zeros."""
    B, L = 4, 576
    g = torch.Generator(device="cuda").manual_seed(32)
    qkv = (torch.randn(B * L, 2304, generator=g, device="cuda") * 1.5).half()
    mask = torch.ones(B, L, dtype=torch.bool, device="cuda")        # True = padded key
    mask[1, 520:576] = False                                         # one block (the short fifth), partly valid
    mask[2, 0:100] = False                                           # two blocks: 0 and 3
    mask[2, 400:512] = False
    mask[3, 128:384] = False                                         # three blocks: 1, 2 and 4, with holes
    mask[3, 512:576] = False
    mask[3] |= torch.rand(L, generator=g, device="cuda") < 0.2
    mask[3, 130] = False
    out, counts = _run_masked(qkv, B, L, mask, guard=BQ)
    assert counts == [0, 1, 2, 3], counts
    assert torch.equal(out[0], torch.zeros_like(out[0])), "a sample without any valid key must give zero rows"
    for b in range(1, B):
        ref = _attn_one(qkv.view(B, L, 2304)[b], keep=~mask[b])
        err = rel_l2(out[b].float(), ref)
        print(f"block list L=576: sample {b} ({counts[b]} blocks) rel_l2={err:.3e}")
        assert torch.isfinite(out[b].float()).all()
        assert err < 2e-3, err


@pytest.mark.parametrize("masked", [False, True])
def test_surface_stage_shape(masked):
    """L = 100, the surface stages' sequence: one tile per sample with two active consumer warpgroups, dense or with a
    key-padding mask; the tile of the last sample runs past the end of the buffer, whose guard rows stay unwritten"""
    B, L = 3, 100
    g = torch.Generator(device="cuda").manual_seed(33)
    qkv = (torch.randn(B * L, 2304, generator=g, device="cuda") * 1.5).half()
    mask = None
    if masked:
        mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
        mask[0, 60:] = True
        mask[2, 1::3] = True
    out, _ = _run_masked(qkv, B, L, mask, guard=BQ)
    for b in range(B):
        keep = None if mask is None else ~mask[b]
        err = rel_l2(out[b].float(), _attn_one(qkv.view(B, L, 2304)[b], keep=keep))
        print(f"L=100 masked={masked}: sample {b} rel_l2={err:.3e}")
        assert torch.isfinite(out[b].float()).all()
        assert err < 2e-3, err
