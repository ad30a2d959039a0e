"""Time DDIM inversion and interpolation on one GPU.

  1. bg_slerp at the edgeZV size of the benchmark (B = 64 samples of 100 faces x 40 edges x 18 values: 4.6 M elements,
     a quarter of the faces masked), against the torch expression it replaces (per-sample dot product and norms, then
     the weighted sum, in fp32).  Rounds alternate; median per-launch times.
  2. Cascade.run at the benchmark workload (B = 64, S0 = 50, E = 40, schedule "ddim", ddim_steps = 50, random-init
     weights, per-sample noise, de-duplication on, both decoders), alternating four runs: plain; a variation of the plain
     run's output at strength 0.5 (start "noise"); the same variation inverted (start "invert"); and an interpolation at
     strength 0.5, alpha 0.5, between that output and a second plain run's.  Seconds per cascade, launches, denoiser
     evaluations (an interpolation inverts its two designs as one batch of 2B) and valid faces per sample.

    python tools/inversion_time.py            # env: DDIM_STEPS (50), CASCADES (3 of each)
Prints the card, its power limit and the median SM clock sampled while the cascades ran.
"""
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from brepgen_b200 import _ffi as f  # noqa: E402
from ddim_time import SmClock, smi  # noqa: E402

DDIM_STEPS = int(os.environ.get("DDIM_STEPS", 50))
CASCADES = int(os.environ.get("CASCADES", 3))


def kernel_times(B=64, S=100, E=40, iters=200, rounds=15):
    from brepgen_b200.sampler import slerp
    g = torch.Generator(device="cuda").manual_seed(0)
    a, b = (torch.randn(B, S * E, 18, generator=g, device="cuda") for _ in range(2))
    mask = (torch.rand(B, S, generator=g, device="cuda") < 0.25)[..., None].expand(B, S, E).reshape(B, S * E)
    alpha = torch.rand(B, generator=g, device="cuda") * 0.8 + 0.1
    out = torch.empty_like(a)

    def kernel():
        slerp(a, b, alpha, mask, out=out)

    def torch_slerp():
        keep = (~mask)[..., None].float()
        ka, kb = a * keep, b * keep
        c = (ka * kb).sum((1, 2)) / (ka.norm(dim=(1, 2)) * kb.norm(dim=(1, 2)))
        th = torch.acos(c.clamp(-1, 1))
        ca, cb = torch.sin((1 - alpha) * th) / torch.sin(th), torch.sin(alpha * th) / torch.sin(th)
        o = ca[:, None, None] * a + cb[:, None, None] * b
        out.copy_(torch.where(mask[..., None], a, o))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / iters
    fns = {"bg_slerp": kernel, "torch slerp (fp32)": torch_slerp}
    for fn in fns.values():
        timed(fn)
    ts = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ts[k].append(timed(fn))
    for k, v in ts.items():
        print(f"slerp of edgeZV, {a.numel()} elements: {k} {statistics.median(v):.1f} us "
              f"(spread {min(v):.1f}-{max(v):.1f})", flush=True)


def cascade_times(B=64, S0=50, E=40):
    from brepgen_b200.models import NETS
    from brepgen_b200.sampler import Cascade, CascadeConfig, Interpolation, Variation, stage_timesteps
    from brepgen_b200.schedulers import strength_timesteps
    from brepgen_b200.spec import denoiser_spec
    from brepgen_b200.synth import synth_state_dict
    from brepgen_b200.vae import build_synthetic_decoders
    dev = torch.device("cuda")
    models = {}
    for kind in NETS:
        m = NETS[kind](False)
        m.load_state_dict(synth_state_dict(denoiser_spec(kind, False), seed=1))
        models[kind] = m.to(dev).eval()
    sv, ev = build_synthetic_decoders(dev)
    casc = Cascade(models, sv, ev, device=dev)
    cfg = CascadeConfig(batch_size=B, num_surfaces=S0, num_edges=E, schedule="ddim", ddim_steps=DDIM_STEPS,
                        noise="per_sample", seed=1000)
    plain = casc.run(cfg)
    other = casc.run(CascadeConfig(**{**cfg.__dict__, "seed": 2000}))
    torch.cuda.synchronize()
    s = 0.5
    kw = {"plain": {}, "variation s = 0.5 (noise)": dict(source=Variation.from_outputs(plain, s)),
          "variation s = 0.5 (invert)": dict(source=Variation.from_outputs(plain, s, start="invert")),
          "interpolation s = 0.5, alpha = 0.5": dict(source=Interpolation(
              Variation.from_outputs(plain, s), Variation.from_outputs(other, s), [0.5] * B))}
    ts = stage_timesteps(cfg)
    k = 4 * len(strength_timesteps(ts, s))       # steps of the four tails; an inversion evaluates the denoiser as often
    calls = {"plain": 4 * len(ts), "variation s = 0.5 (noise)": k, "variation s = 0.5 (invert)": 2 * k,
             "interpolation s = 0.5, alpha = 0.5": 2 * k}
    for name in kw:                              # warm-up: packs weights, allocates workspaces
        out = casc.run(cfg, **kw[name])
        torch.cuda.synchronize()
        nv = (~out["surfMask"]).sum(1)
        print(f"{name}: valid faces per sample {int(nv.min())}-{int(nv.max())}", flush=True)
    clk = SmClock()
    clk.start()
    res = {name: [] for name in kw}
    launches = {}
    for _ in range(CASCADES):
        for name in kw:
            l0 = f.lib().bg_launch_count() + f.replayed_launches
            t0 = time.perf_counter()
            casc.run(cfg, **kw[name])
            torch.cuda.synchronize()
            res[name].append(time.perf_counter() - t0)
            launches[name] = f.lib().bg_launch_count() + f.replayed_launches - l0
    mhz = clk.stop()
    for name, v in res.items():
        t = statistics.median(v)
        print(f"cascade {name} DDIM-{DDIM_STEPS} B={B} S0={S0} E={E} per-sample noise: {t:.3f} s per cascade (spread "
              f"{min(v):.3f}-{max(v):.3f}), {launches[name]} launches, {calls[name]} denoiser evaluations", flush=True)
    print(f"median SM clock {mhz} MHz", flush=True)


if __name__ == "__main__":
    print("GPU:", smi("name,power.limit,clocks.max.sm"), flush=True)
    kernel_times()
    cascade_times()
