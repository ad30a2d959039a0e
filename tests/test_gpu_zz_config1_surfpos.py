"""GPU: BASELINE.json configs[1] as a parity case -- SurfPosNet with the 1000-step DDPM scheduler, 30 face tokens,
batch 64 (SURVEY.md section 8(d) input 2): single forwards at t in {999, 500, 249, 10, 0} and two 10-step chains
(t = 999..990 and t = 9..0) with the step noise shared with the CPU fp32 oracle; bar 1e-3 relative (L2).

Strict: no expected failures.
"""
import pytest
import torch

from brepgen_b200.spec import denoiser_spec
from brepgen_b200.synth import synth_state_dict
from oracle import denoisers as O
from oracle.schedulers import DDPMOracle

pytestmark = pytest.mark.gpu
B, S = 64, 30


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_config1_surfposnet_ddpm1000_b64_s30():
    from brepgen_b200.models import SurfPosNet
    from brepgen_b200.schedulers import DDPMScheduler
    sd = synth_state_dict(denoiser_spec("surfpos", False), seed=7)
    m = SurfPosNet(False)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(0)
    x0 = torch.randn(B, S, 6, generator=g)
    sched, orc = DDPMScheduler(clip_sample=True, clip_sample_range=3), DDPMOracle(clip_sample=True, clip_sample_range=3.0)
    sched.set_timesteps(1000), orc.set_timesteps(1000)
    with torch.no_grad():
        for t in (999, 500, 249, 10, 0):
            tt = torch.tensor([t])
            err = rel_l2(m(x0.cuda(), tt.cuda(), None).cpu(), O.surfpos_forward(sd, x0, tt, None))
            print(f"config1 forward t={t} rel_l2={err:.3e}")
            assert err < 1e-3, (t, err)
        for start in (999, 9):
            xo, xg = x0.clone(), x0.clone().cuda()
            for t in range(start, start - 10, -1):
                tt = torch.tensor([t])
                nz = torch.randn(B, S, 6, generator=g)
                xo = orc.step(O.surfpos_forward(sd, xo, tt, None), t, xo, nz if t > 0 else None)
                xg = sched.step(m(xg, tt.cuda(), None), tt[0], xg, noise=nz if t > 0 else None).prev_sample
            err = rel_l2(xg.cpu(), xo)
            print(f"config1 10-step chain from t={start} rel_l2={err:.3e}")
            assert err < 1e-3, (start, err)
