"""GPU parity AT THE BENCHMARK'S OWN SHAPES (BASELINE.json configs[2]: S = 100 faces x E = 40 edges = L = 4000 tokens).

Goldens = outputs of the reference's OWN EdgePosNet / EdgeZNet classes (network.py:1257-1286, 1357-1393)
at that shape, written by tests/golden/make_golden_l4000.py: B = 2 and 3, dense and ragged masks (whole 128-key blocks
padded, 30 % random edge masks), scalar and per-sample timesteps, classifier-free labels on / off, plus a 4-step DDPM chain
with injected noise.  This is the kernel instantiation the headline number is measured on (flash attention over 32 key blocks
with a block list, one 128-row query tile per CTA, persistent GEMMs at M = B * 4000, the multi-GB workspace carve).  Compared on valid tokens
(padded tokens are discarded by the cascade, sample.py:245,284); bar 1e-3 relative L2 (BASELINE.json).
"""
import os

import numpy as np
import pytest
import torch

from brepgen_b200.spec import denoiser_spec
from brepgen_b200.synth import synth_state_dict
from make_golden_l4000 import CASES, CHAIN, case_inputs_l4000, chain_noise

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "denoisers_l4000_golden.npz"))
TOL = 1e-3


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _model(kind, use_cf):
    from brepgen_b200.models import NETS
    m = NETS[kind](use_cf)
    m.load_state_dict(synth_state_dict(denoiser_spec(kind, use_cf), seed=7))
    return m.cuda().eval()


def _cuda(v):
    return v.cuda() if torch.is_tensor(v) else v


@pytest.mark.parametrize("name", list(CASES))
def test_golden_l4000(name):
    spec = CASES[name]
    inp, valid = case_inputs_l4000(spec)
    m = _model(spec[0], spec[1])
    with torch.no_grad():
        y = m(*[_cuda(v) for v in inp.values()]).cpu()
    ref = torch.from_numpy(GOLD[name])
    assert y.shape == ref.shape
    assert torch.isfinite(y).all()
    err = rel_l2(y[valid], ref[valid])
    # per-sample errors too: a wrong batch pitch would hide in the aggregate of a large batch
    per = [rel_l2(y[b][valid[b]], ref[b][valid[b]]) for b in range(y.shape[0])]
    print(f"l4000 golden {name}: rel_l2={err:.3e} per-sample={['%.2e' % e for e in per]}")
    assert err < TOL and max(per) < TOL, (err, per)


def test_chain4_l4000():
    """4 DDPM steps t = 999..996 of EdgePosNet at L = 4000 with injected noise (the loop body of sample.py:145-153)"""
    from brepgen_b200.schedulers import DDPMScheduler
    inp, valid = case_inputs_l4000(CHAIN)
    m = _model(CHAIN[0], CHAIN[1])
    sched = DDPMScheduler(num_train_timesteps=1000, beta_schedule="linear", prediction_type="epsilon", beta_start=0.0001,
                          beta_end=0.02, clip_sample=True, clip_sample_range=3)
    sched.set_timesteps(1000)
    x = inp["edgePos"].cuda()
    sP, sZ, mask = inp["surfPos"].cuda(), inp["surfZ"].cuda(), inp["mask"].cuda()
    with torch.no_grad():
        for k, t in enumerate(CHAIN[5]):
            pred = m(x, torch.tensor([t]).cuda(), sP, sZ, mask, None)
            x = sched.step(pred, t, x, noise=chain_noise(k, x.shape).cuda()).prev_sample
    ref = torch.from_numpy(GOLD["edgepos_chain4_b2"])
    err = rel_l2(x.cpu()[valid], ref[valid])
    print(f"l4000 4-step chain rel_l2={err:.3e}")
    assert err < TOL, err


def test_attention_op_b8_l4000_masked():
    """bg_op_attention at B = 8, L = 4000 with ragged + random masks and the block list, against fp32 torch on the GPU"""
    from brepgen_b200 import _ffi as f
    B, L = 8, 4000
    g = torch.Generator(device="cuda").manual_seed(4000)
    qkv = (torch.randn(B * L, 2304, generator=g, device="cuda") * 1.5).half()
    nvalid = torch.tensor([4000, 3999, 1480, 129, 128, 2560, 1, 3000], device="cuda")
    mask = torch.arange(L, device="cuda")[None, :] >= nvalid[:, None]
    mask |= torch.rand(B, L, generator=g, device="cuda") < 0.3
    mask[:, 0] = False
    out = torch.full((B * L, 768), float("nan"), device="cuda", dtype=torch.float16)
    nkb = (L + 127) // 128
    scratch = torch.zeros(B * (5 * nkb + 1), dtype=torch.int32, device="cuda")
    f.check(f.lib().bg_op_attention(qkv.data_ptr(), out.data_ptr(), B, L, mask.data_ptr(), 1, scratch.data_ptr(),
                                   f.current_stream()), "attention")
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    out = out.float().view(B, L, 768)
    worst = 0.0
    for b in range(B):                                  # one sample at a time: the fp32 score tensor is 768 MB
        q, k, v = qkv.view(B, L, 3, 12, 64)[b].float().permute(1, 2, 0, 3)
        s = (q @ k.transpose(-1, -2)) / 8.0
        s = s.masked_fill(mask[b].view(1, 1, L), float("-inf"))
        ref = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(L, 768)
        worst = max(worst, rel_l2(out[b], ref))
    print(f"attention op B=8 L=4000 masked: worst per-sample rel_l2={worst:.3e}")
    assert worst < 2e-3, worst
