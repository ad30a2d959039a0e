"""Time B-rep completion on one GPU.

  1. bg_replace_known_tab against bg_ddim_step_tab at the edgeZV size of the benchmark (B = 64 samples of 100 x 40 x 18
     elements: 4.6 M), per-sample keys, with 10 of 100 faces known (all their edges) and with every token known.  Rounds
     alternate between the kernels; prints the median per-launch time of each.
  2. Cascade.run at the benchmark workload (B = 64, S0 = 50, E = 40, schedule "ddim", ddim_steps = 50, random-init weights,
     per-sample noise, de-duplication on, both decoders), alternating three runs: plain; a completion with nothing known
     (n_faces = 0: the replacement launches alone, same token counts as the plain run); a completion of 10 known faces per
     sample with their edges.  Random-init denoisers place every generated face on the same box, so the de-duplication
     keeps one generated face per sample: the third run carries 11 valid faces per sample into the later stages where
     the others carry 1, and its time includes that larger workload.  Seconds per cascade, B-reps/s and launches.

    python tools/completion_time.py            # env: DDIM_STEPS (50), CASCADES (3 of each)
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
    from brepgen_b200.schedulers import DDIMScheduler, sample_keys
    per = S * E * 18
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(0)
    eps, x, known = (torch.randn(n, generator=g, device="cuda") for _ in range(3))
    lib, st = f.lib(), f.current_stream()
    s = DDIMScheduler(clip_sample=True, clip_sample_range=3)
    s.set_timesteps(50)
    coef = s.coefficient_table(s.timesteps).cuda()
    rtab = s.replace_table(s.timesteps).cuda()
    step = torch.full((1,), 10, dtype=torch.int32, device="cuda")
    t_cur = torch.full((1,), int(s.timesteps[10]), dtype=torch.int64, device="cuda")
    keys = torch.from_numpy(sample_keys(list(range(B)), 3).view(np.int64)).cuda()
    some = (torch.arange(S, device="cuda")[None, :, None] < 10).expand(B, S, E).to(torch.uint8).contiguous()
    every = torch.ones(B, S, E, dtype=torch.uint8, device="cuda")

    def ddim():
        return lib.bg_ddim_step_tab(eps.data_ptr(), None, 0.0, x.data_ptr(), x.data_ptr(), 0, 0, 0, keys.data_ptr(), per,
                                    t_cur.data_ptr(), n, coef.data_ptr(), step.data_ptr(), 3.0, 0, st)

    def replace(m):
        return lambda: lib.bg_replace_known_tab(x.data_ptr(), known.data_ptr(), m.data_ptr(), n, 18, 0, keys.data_ptr(),
                                                per, t_cur.data_ptr(), rtab.data_ptr(), step.data_ptr(), st)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / iters
    fns = {"bg_ddim_step_tab": ddim, "bg_replace_known_tab 10% known": replace(some),
           "bg_replace_known_tab all known": replace(every)}
    for fn in fns.values():
        assert fn() == 0
        timed(fn)
    ts = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ts[k].append(timed(fn))
    for k, v in ts.items():
        print(f"kernel n = {n}: {k} {statistics.median(v):.1f} us (spread {min(v):.1f}-{max(v):.1f})", flush=True)


def cascade_times(B=64, S0=50, E=40):
    from brepgen_b200.models import NETS
    from brepgen_b200.sampler import Cascade, CascadeConfig, Completion
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
    K = 10
    g = torch.Generator().manual_seed(5)
    corner = torch.rand(B, 1, 3, generator=g) * 0.2
    lo = corner + torch.arange(K)[None, :, None] * 0.1     # distinct boxes: 0.3 apart in model units (> bbox_threshold)
    edge_mask = (torch.arange(E)[None, None, :] >= 8).expand(B, K, E).contiguous()
    known = Completion(n_faces=[K] * B, surfPos=torch.cat([lo, lo + 0.05], -1), surfZ=torch.randn(B, K, 48, generator=g),
                       edgePos=torch.rand(B, K, E, 6, generator=g) * 0.2, edge_z=torch.randn(B, K, E, 12, generator=g),
                       edgeV=torch.randn(B, K, E, 6, generator=g), edge_mask=edge_mask)
    nothing = Completion(**dict(vars(known), n_faces=[0] * B))
    arms = {"plain": {}, "completion, nothing known": dict(known=nothing), f"completion, {K} known faces": dict(known=known)}
    for kw in arms.values():                     # warm-up: packs weights, allocates workspaces
        out = casc.run(cfg, **kw)
        torch.cuda.synchronize()
        print(f"valid faces per sample: {int((~out['surfMask']).sum(1).min())}-{int((~out['surfMask']).sum(1).max())}",
              flush=True)
    clk = SmClock()
    clk.start()
    res = {name: [] for name in arms}
    launches = {}
    for _ in range(CASCADES):
        for name, kw in arms.items():
            l0 = f.lib().bg_launch_count() + f.replayed_launches
            t0 = time.perf_counter()
            casc.run(cfg, **kw)
            torch.cuda.synchronize()
            res[name].append(time.perf_counter() - t0)
            launches[name] = f.lib().bg_launch_count() + f.replayed_launches - l0
    mhz = clk.stop()
    for name, v in res.items():
        s = statistics.median(v)
        print(f"cascade {name} DDIM-{DDIM_STEPS} B={B} S0={S0} E={E} per-sample noise: {s:.3f} s per cascade (spread "
              f"{min(v):.3f}-{max(v):.3f}), {B / s:.3f} B-reps/s, {launches[name]} launches", flush=True)
    print(f"median SM clock {mhz} MHz", flush=True)


if __name__ == "__main__":
    print("GPU:", smi("name,power.limit,clocks.max.sm"), flush=True)
    kernel_times()
    cascade_times()
