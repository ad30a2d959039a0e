"""GPU: the CUDA-graph form of a DDPM loop (sampler.Cascade._loop_graph: step counter / timestep advance -> forward -> fused
table-driven scheduler step, captured once and replayed) against the eager loop with the same Philox stream, and the whole
cascade with graphs on vs off.  Loop body mirrored: sample.py:145-153; SURVEY.md 7.2 step 4."""
import pytest
import torch

from brepgen_b200.spec import denoiser_spec
from brepgen_b200.synth import synth_state_dict

pytestmark = pytest.mark.gpu


def _models(use_cf, kinds=("surfpos", "surfz", "edgepos", "edgez")):
    from brepgen_b200.models import NETS
    out = {}
    for k in kinds:
        m = NETS[k](use_cf)
        m.load_state_dict(synth_state_dict(denoiser_spec(k, use_cf), seed=3))
        out[k] = m.cuda().eval()
    return out


def test_graph_loop_equals_eager_loop_config1_shape():
    """SurfPosNet, B = 64, S = 30 (BASELINE configs[1] shape), the last 25 steps of the 1000-step DDPM schedule"""
    from brepgen_b200.sampler import Cascade, CascadeConfig
    casc = Cascade(_models(False, ("surfpos",)), device="cuda")
    x = torch.randn(64, 30, 6, generator=torch.Generator().manual_seed(0)).cuda()
    fwd = lambda xi, t: casc.m["surfpos"](xi, t, None)
    casc.ddpm.set_timesteps(1000)
    ts = casc.ddpm.timesteps[-25:]
    outs = {}
    for mode in ("off", "on"):
        cfg = CascadeConfig(batch_size=64, schedule="ddpm", graph=mode)
        casc.ddpm.set_noise_seed(77, 0, 0)
        with torch.no_grad():
            outs[mode] = casc._loop(cfg, casc.ddpm, ts, x.clone(), fwd, None, None)
    torch.cuda.synchronize()
    assert casc.last_graph_steps == 25
    assert torch.isfinite(outs["on"]).all()
    err = float((outs["on"] - outs["off"]).abs().max() / outs["off"].abs().max())
    print(f"graph vs eager, 25 DDPM steps: max rel diff {err:.2e}")
    assert err < 1e-5, err


@pytest.mark.parametrize("use_cf", [False, True])
def test_cascade_with_graphs_equals_eager(use_cf):
    """whole cascade (DDPM-12 per stage, late face increase, both dedups), graph = on vs off: identical masks, equal tensors"""
    from brepgen_b200.sampler import Cascade, CascadeConfig
    casc = Cascade(_models(use_cf), device="cuda")
    res = {}
    for mode in ("off", "on"):
        cfg = CascadeConfig(batch_size=2, num_surfaces=6, num_edges=4, use_cf=use_cf, class_label=6, schedule="ddpm",
                            ddpm_steps=12, seed=5, decode=False, graph=mode)
        res[mode] = casc.run(cfg)
    torch.cuda.synchronize()
    for k in res["off"]:
        a, b = res["off"][k], res["on"][k]
        assert a.shape == b.shape, k
        if a.dtype == torch.bool:
            assert torch.equal(a, b), k
        else:
            assert torch.isfinite(b).all(), k
            assert float((a - b).abs().max()) <= 1e-4 * max(1.0, float(a.abs().max())), k
