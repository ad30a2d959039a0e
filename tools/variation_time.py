"""Time B-rep variations on one GPU.

  1. The start of a varied stage at the edgeZV size of the benchmark (B = 64 samples of 100 faces x 40 edges x 18 values:
     4.6 M elements), per-sample keys: bg_fill_index (the pad_repeat map of every face's source edges) and
     bg_add_noise_gather (gather, scale, add_noise with the keyed start noise drawn in the kernel), against the torch
     gather + add_noise they replace (z from bg_randn_keyed, the same map).  Rounds alternate; median per-launch times.
  2. Cascade.run at the benchmark workload (B = 64, S0 = 50, E = 40, schedule "ddim", ddim_steps = 50, random-init
     weights, per-sample noise, de-duplication on, both decoders), alternating three runs: plain; a variation of the
     plain run's output at strength 0.5; and at (0, 0, 0.5, 0.5) (faces and their latents kept, edges varied).  Seconds
     per cascade, launches, denoiser forwards and valid faces per sample.

    python tools/variation_time.py            # env: DDIM_STEPS (50), CASCADES (3 of each)
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
    import numpy as np
    from brepgen_b200.schedulers import DDPMScheduler, sample_keys
    lib, st = f.lib(), f.current_stream()
    g = torch.Generator(device="cuda").manual_seed(0)
    src = torch.randn(B * S * E, 18, generator=g, device="cuda")
    # sources shaped like a design: 8..40 valid edges per face, a quarter of the faces without a source
    nv = torch.randint(8, E + 1, (B * S, 1), generator=g, device="cuda")
    emask = (torch.arange(E, device="cuda")[None, :] >= nv).to(torch.uint8).contiguous()
    rows = torch.randperm(B * S, generator=g, device="cuda").to(torch.int32)
    rows[torch.rand(B * S, generator=g, device="cuda") < 0.25] = -1
    idx = torch.empty(B * S, E, dtype=torch.int32, device="cuda")
    out = torch.empty(B * S * E, 18, device="cuda")
    z = torch.empty_like(out)
    keys = torch.from_numpy(sample_keys(list(range(B)), 3).view(np.int64)).cuda()
    sa, sb = DDPMScheduler().replace_coefficients(500, initial=True)
    n_tok = B * S * E

    def fill():
        return lib.bg_fill_index(emask.data_ptr(), rows.data_ptr(), B * S, B * S, E, E, idx.data_ptr(), st)

    def gather():
        return lib.bg_add_noise_gather(src.data_ptr(), n_tok, idx.data_ptr(), n_tok, 18, 1.0, sa, sb, None,
                                       keys.data_ptr(), S * E, 1, 0, out.data_ptr(), st)

    def start():
        fill()
        return gather()

    def torch_start():
        assert lib.bg_randn_keyed(keys.data_ptr(), B, S * E * 18, 1, 0, z.data_ptr(), st) == 0
        i = idx.view(-1).long()
        out.copy_(torch.where((i == -1)[:, None], z, sa * (1.0 * src[i.clamp(min=0)]) + sb * z))
        return 0

    assert fill() == 0 and gather() == 0
    torch.cuda.synchronize()
    i = idx.view(-1).long()
    assert lib.bg_randn_keyed(keys.data_ptr(), B, S * E * 18, 1, 0, z.data_ptr(), st) == 0
    ref = torch.where((i == -1)[:, None], z, sa * (1.0 * src[i.clamp(min=0)]) + sb * z)
    assert torch.equal(ref, out), "bg_add_noise_gather differs from the torch expression"

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / iters
    fns = {"bg_fill_index": fill, "bg_add_noise_gather (keyed)": gather, "fill + gather": start,
           "torch: bg_randn_keyed + gather + add_noise": torch_start}
    for fn in fns.values():
        assert fn() == 0
        timed(fn)
    ts = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ts[k].append(timed(fn))
    for k, v in ts.items():
        print(f"start of edgeZV, {n_tok * 18} elements: {k} {statistics.median(v):.1f} us "
              f"(spread {min(v):.1f}-{max(v):.1f})", flush=True)


def cascade_times(B=64, S0=50, E=40):
    from brepgen_b200.models import NETS
    from brepgen_b200.sampler import Cascade, CascadeConfig, Variation, stage_timesteps
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
    torch.cuda.synchronize()
    arms = {"plain": None, "variation s = 0.5": 0.5, "variation s = (0, 0, 0.5, 0.5)": (0, 0, 0.5, 0.5)}
    ts = stage_timesteps(cfg)
    forwards = {name: 4 * len(ts) if s is None else
                sum(len(strength_timesteps(ts, v)) for v in ([s] * 4 if isinstance(s, float) else s))
                for name, s in arms.items()}
    kw = {name: {} if s is None else dict(source=Variation.from_outputs(plain, s)) for name, s in arms.items()}
    for name in arms:                            # warm-up: packs weights, allocates workspaces
        out = casc.run(cfg, **kw[name])
        torch.cuda.synchronize()
        nv = (~out["surfMask"]).sum(1)
        print(f"{name}: valid faces per sample {int(nv.min())}-{int(nv.max())}", flush=True)
    clk = SmClock()
    clk.start()
    res = {name: [] for name in arms}
    launches = {}
    for _ in range(CASCADES):
        for name in arms:
            l0 = f.lib().bg_launch_count() + f.replayed_launches
            t0 = time.perf_counter()
            casc.run(cfg, **kw[name])
            torch.cuda.synchronize()
            res[name].append(time.perf_counter() - t0)
            launches[name] = f.lib().bg_launch_count() + f.replayed_launches - l0
    mhz = clk.stop()
    for name, v in res.items():
        s = statistics.median(v)
        print(f"cascade {name} DDIM-{DDIM_STEPS} B={B} S0={S0} E={E} per-sample noise: {s:.3f} s per cascade (spread "
              f"{min(v):.3f}-{max(v):.3f}), {B / s:.3f} B-reps/s, {launches[name]} launches, {forwards[name]} forwards",
              flush=True)
    print(f"median SM clock {mhz} MHz", flush=True)


if __name__ == "__main__":
    print("GPU:", smi("name,power.limit,clocks.max.sm"), flush=True)
    kernel_times()
    cascade_times()
