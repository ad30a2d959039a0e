"""Time RePaint resampling on one GPU.

  1. bg_repaint_step_tab against bg_ddim_step_tab + bg_replace_known_tab (the unfused completion step it replaces) at the
     edgeZV size of the benchmark (B = 64 samples of 100 x 40 x 18 elements: 4.6 M), per-sample keys, 10 of 100 faces
     known with all their edges; and bg_repaint_undo_tab at n = 20 transitions (N = 50).  Rounds alternate between the
     arms; prints the median per-launch time of each and the bytes each moves per element.
  2. Cascade.run completions at the benchmark workload (B = 64, S0 = 50, E = 40, random-init weights, per-sample noise,
     de-duplication on, both decoders, 10 known faces per sample with their edges): schedule "repaint" at
     (N, jump_length, jump_n_sample) = (50, 5, 5) and (50, 5, 1) (DDIM-50's list through the RePaint path) against
     schedule "ddim" with 50 steps, alternated.  Seconds per cascade, B-reps/s, launches, network evaluations (step
     entries x 4 stages) and the valid faces per sample each arm carries into the edge stages: random-init denoisers
     decide how many generated faces survive the de-duplication, and the edge stages' cost grows with them.

    python tools/repaint_time.py            # env: CASCADES (1 of each after a warm-up of each)
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

CASCADES = int(os.environ.get("CASCADES", 1))


def kernel_times(B=64, S=100, E=40, iters=200, rounds=15):
    import numpy as np
    from brepgen_b200.schedulers import DDIMScheduler, RePaintScheduler, repaint_entries, sample_keys
    per = S * E * 18
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(0)
    eps, x, known = (torch.randn(n, generator=g, device="cuda") for _ in range(3))
    lib, st = f.lib(), f.current_stream()
    d = DDIMScheduler(clip_sample=True, clip_sample_range=3)
    d.set_timesteps(50)
    coef_d = d.coefficient_table(d.timesteps).cuda()
    rtab = d.replace_table(d.timesteps).cuda()
    r = RePaintScheduler(clip_sample=True, clip_sample_range=3)
    r.set_timesteps(50, 5, 5)
    ents = repaint_entries(r.timesteps)
    k_step = next(k for k, (s, t) in enumerate(ents) if s and t == int(d.timesteps[10]))
    k_undo = next(k for k, (s, _) in enumerate(ents) if not s)
    coef_r, utab = r.coefficient_table().cuda(), r.undo_table().cuda()
    nt = r.undo_transitions
    step_d = torch.full((1,), 10, dtype=torch.int32, device="cuda")
    step_r = torch.full((1,), k_step, dtype=torch.int32, device="cuda")
    step_u = torch.full((1,), k_undo, dtype=torch.int32, device="cuda")
    t_cur = torch.full((1,), int(d.timesteps[10]), dtype=torch.int64, device="cuda")
    keys = torch.from_numpy(sample_keys(list(range(B)), 3).view(np.int64)).cuda()
    some = (torch.arange(S, device="cuda")[None, :, None] < 10).expand(B, S, E).to(torch.uint8).contiguous()

    def unfused():
        a = lib.bg_ddim_step_tab(eps.data_ptr(), None, 0.0, x.data_ptr(), x.data_ptr(), 0, 0, 0, keys.data_ptr(), per,
                                 t_cur.data_ptr(), n, coef_d.data_ptr(), step_d.data_ptr(), 3.0, 0, st)
        return a or lib.bg_replace_known_tab(x.data_ptr(), known.data_ptr(), some.data_ptr(), n, 18, 0, keys.data_ptr(),
                                             per, t_cur.data_ptr(), rtab.data_ptr(), step_d.data_ptr(), st)

    def fused():
        return lib.bg_repaint_step_tab(eps.data_ptr(), None, 0.0, x.data_ptr(), x.data_ptr(), known.data_ptr(),
                                       some.data_ptr(), 18, 0, keys.data_ptr(), per, n, coef_r.data_ptr(),
                                       step_r.data_ptr(), 3.0, st)

    def undo():
        return lib.bg_repaint_undo_tab(x.data_ptr(), n, nt, 0, keys.data_ptr(), per, utab.data_ptr(), step_u.data_ptr(),
                                       st)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / iters
    # algorithmic bytes per element: DDIM 12 (eps, x, out) + replace 0.8 (the 10% known: known read, x written);
    # RePaint step 12 (the unknown 90%: eps, x, out; the known 10%: known, out); undo 8 (x read and written once)
    fns = {"bg_ddim_step_tab + bg_replace_known_tab, 10% known": (unfused, 12.0 + 0.1 * 8.0),
           "bg_repaint_step_tab, 10% known": (fused, 0.9 * 12.0 + 0.1 * 8.0),
           f"bg_repaint_undo_tab, n = {nt}": (undo, 8.0)}
    for fn, _ in fns.values():
        assert fn() == 0
        timed(fn)
    ts = {k: [] for k in fns}
    for _ in range(rounds):
        for k, (fn, _) in fns.items():
            ts[k].append(timed(fn))
    for k, v in ts.items():
        med = statistics.median(v)
        print(f"kernel n = {n}: {k} {med:.1f} us (spread {min(v):.1f}-{max(v):.1f}), "
              f"{fns[k][1] * n / med / 1e6:.2f} TB/s algorithmic", flush=True)


def cascade_times(B=64, S0=50, E=40):
    from brepgen_b200.models import NETS
    from brepgen_b200.sampler import Cascade, CascadeConfig, Completion
    from brepgen_b200.schedulers import repaint_entries, repaint_timesteps
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
    base = dict(batch_size=B, num_surfaces=S0, num_edges=E, noise="per_sample", seed=1000)
    K = 10
    g = torch.Generator().manual_seed(5)
    corner = torch.rand(B, 1, 3, generator=g) * 0.2
    lo = corner + torch.arange(K)[None, :, None] * 0.1     # distinct boxes: 0.3 apart in model units (> bbox_threshold)
    edge_mask = (torch.arange(E)[None, None, :] >= 8).expand(B, K, E).contiguous()
    known = Completion(n_faces=[K] * B, surfPos=torch.cat([lo, lo + 0.05], -1), surfZ=torch.randn(B, K, 48, generator=g),
                       edgePos=torch.rand(B, K, E, 6, generator=g) * 0.2, edge_z=torch.randn(B, K, E, 12, generator=g),
                       edgeV=torch.randn(B, K, E, 6, generator=g), edge_mask=edge_mask)
    steps = sum(s for s, _ in repaint_entries(repaint_timesteps(50, 5, 5)))
    rp = lambda jn: CascadeConfig(schedule="repaint", repaint_steps=50, repaint_jump_length=5, repaint_jump_n_sample=jn,
                                  **base)
    arms = {"DDIM-50 completion": (CascadeConfig(schedule="ddim", ddim_steps=50, **base), 4 * 50),
            "RePaint (50, 5, 1) completion (DDIM-50's list)": (rp(1), 4 * 50),
            "RePaint (50, 5, 5) completion": (rp(5), 4 * steps)}
    for name, (cfg, _) in arms.items():          # warm-up: packs weights, allocates workspaces
        out = casc.run(cfg, known=known)
        torch.cuda.synchronize()
        nv = (~out["surfMask"]).sum(1)
        print(f"{name}: valid faces per sample {int(nv.min())}-{int(nv.max())} (mean {float(nv.float().mean()):.1f})",
              flush=True)
    clk = SmClock()
    clk.start()
    res = {name: [] for name in arms}
    launches = {}
    for _ in range(CASCADES):
        for name, (cfg, _) in arms.items():
            l0 = f.lib().bg_launch_count() + f.replayed_launches
            t0 = time.perf_counter()
            casc.run(cfg, known=known)
            torch.cuda.synchronize()
            res[name].append(time.perf_counter() - t0)
            launches[name] = f.lib().bg_launch_count() + f.replayed_launches - l0
    mhz = clk.stop()
    for name, v in res.items():
        s = statistics.median(v)
        print(f"cascade {name} B={B} S0={S0} E={E} per-sample noise: {s:.3f} s per cascade (spread {min(v):.3f}-"
              f"{max(v):.3f}), {B / s:.3f} B-reps/s, {launches[name]} launches, {arms[name][1]} network evaluations",
              flush=True)
    print(f"median SM clock {mhz} MHz", flush=True)


if __name__ == "__main__":
    print("GPU:", smi("name,power.limit,clocks.max.sm"), flush=True)
    kernel_times()
    if os.environ.get("KERNELS_ONLY") != "1":
        cascade_times()
