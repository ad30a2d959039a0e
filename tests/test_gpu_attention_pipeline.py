"""Edge cases of the software-pipelined attention kernel (csrc/attn.cu), through the C ABI.

The kernel issues the next key block's Q K^T together with the previous block's P V and waits for them separately, so
the prologue / drain for 0, 1 and 2 key blocks, query tiles that lie partly or wholly beyond a sample's length, and many
tiles of unequal length are where it can go wrong.  Every case is
checked against fp32 torch at the 2e-3 relative-L2 bar of test_gpu_ops.py, and a second launch must reproduce the first
bit for bit.
"""
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


def _run_varlen(lens, L, seed):
    f = _ffi()
    g = torch.Generator(device="cuda").manual_seed(seed)
    lens_t = torch.tensor(lens, dtype=torch.int32, device="cuda")
    row0 = torch.zeros_like(lens_t)
    row0[1:] = torch.cumsum(lens_t, 0)[:-1]
    # the buffers have B * L rows, as in a compacted forward; the samples are packed at the front
    qkv = (torch.randn(len(lens) * L, 2304, generator=g, device="cuda") * 1.5).half()
    outs = []
    for _ in range(2):
        out = torch.full((len(lens) * L, 768), float("nan"), device="cuda", dtype=torch.float16)
        f.check(f.lib().bg_op_attention_varlen(qkv.data_ptr(), out.data_ptr(), len(lens), L, row0.data_ptr(),
                                              lens_t.data_ptr(), f.current_stream()), "attention varlen")
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "two launches on the same input differ"
    worst = 0.0
    for b, n in enumerate(lens):
        if n == 0:
            continue
        r = int(row0[b])
        got = outs[0][r:r + n]
        assert torch.isfinite(got.float()).all(), f"sample {b} (len {n}) has non-finite rows"
        worst = max(worst, rel_l2(got.float(), _attn_one(qkv[r:r + n])))
    return worst


def test_varlen_edge_lengths():
    """one batch with lengths 0 (no tile at all), 1, 127 / 128 / 129 (tile and key-block edges), 255 and 4000 (32 key
    blocks); tiles of short samples read the next sample's rows, which must be masked"""
    err = _run_varlen([0, 1, 127, 128, 129, 255, 4000], 4000, seed=11)
    print(f"varlen edge lengths rel_l2={err:.3e}")
    assert err < 2e-3, err


def test_varlen_many_unequal_tiles():
    """far more CTAs than SMs, samples of very different length (1 .. 3 key blocks and up to 16)"""
    g = torch.Generator().manual_seed(5)
    lens = torch.randint(1, 2049, (48,), generator=g).tolist()
    lens[0], lens[1], lens[2] = 2048, 64, 200
    err = _run_varlen(lens, 2048, seed=12)
    print(f"varlen 48 unequal samples rel_l2={err:.3e}")
    assert err < 2e-3, err


def test_block_list_0_to_3_blocks():
    """block-list mode with 0, 1, 2 and 3 listed key blocks (L = 512: four blocks).  Sample 0 has every key padded, so
    no block is listed and its rows must come out as exact zeros."""
    f = _ffi()
    B, L = 4, 512
    g = torch.Generator(device="cuda").manual_seed(21)
    qkv = (torch.randn(B * L, 2304, generator=g, device="cuda") * 1.5).half()
    mask = torch.ones(B, L, dtype=torch.bool, device="cuda")        # True = padded key
    mask[1, 256:300] = False                                         # one block, partly valid
    mask[2, 0:128] = False                                           # two blocks: 0 and 3
    mask[2, 400:512] = False
    mask[3, 0:256] = False                                           # three blocks: 0, 1 and 3, with holes
    mask[3, 384:512] = False
    mask[3] |= torch.rand(L, generator=g, device="cuda") < 0.2
    mask[3, 0] = False
    nkb = (L + 127) // 128
    outs = []
    for _ in range(2):
        scratch = torch.zeros(B * (5 * nkb + 1), dtype=torch.int32, device="cuda")
        out = torch.full((B * L, 768), float("nan"), device="cuda", dtype=torch.float16)
        f.check(f.lib().bg_op_attention(qkv.data_ptr(), out.data_ptr(), B, L, mask.data_ptr(), 1, scratch.data_ptr(),
                                       f.current_stream()), "attention")
        outs.append(out)
    torch.cuda.synchronize()
    counts = scratch[B * nkb:B * nkb + B].tolist()
    assert counts == [0, 1, 2, 3], counts
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "two launches on the same input differ"
    out = outs[0].view(B, L, 768)
    assert torch.equal(out[0], torch.zeros_like(out[0])), "a sample without any valid key must give zero rows"
    for b in range(1, B):
        ref = _attn_one(qkv.view(B, L, 2304)[b], keep=~mask[b])
        err = rel_l2(out[b].float(), ref)
        print(f"block list: sample {b} ({counts[b]} blocks) rel_l2={err:.3e}")
        assert torch.isfinite(out[b].float()).all()
        assert err < 2e-3, err
