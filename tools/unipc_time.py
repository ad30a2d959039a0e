"""Time the UniPC step and UniPC cascades against DPM-Solver++ and DDIM on one GPU.

  1. bg_unipc_step against bg_dpm_step (second order, ODE) at the edgeZV size of the benchmark (B = 64 samples of
     100 x 40 x 18 = 72 000 elements: 4.6 M): UniPC order 2 with its corrector and order 3 with its corrector, CFG off
     and on.  Rounds alternate between the two kernels; prints the median per-launch time of each.
  2. Cascade.run at the benchmark workload (B = 64, S0 = 50, E = 40, dense masks, random-init weights, both decoders) for
     UniPC-10, DPM-20 and DDIM-50, alternated in one process: seconds per cascade, B-reps/s, kernel launches (host
     launches + kernels in graph replays) and network evaluations.  The whole schedule runs; nothing is scaled.

    python tools/unipc_time.py          # env: CASCADES (3)
Prints the card, its power limit and the median SM clock sampled while the cascades ran.  Needs a GPU.
"""
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from brepgen_b200 import _ffi as f  # noqa: E402
from ddim_time import SmClock, smi  # noqa: E402

CASCADES = int(os.environ.get("CASCADES", 3))


def step_times(B=64, per=100 * 40 * 18, iters=200, rounds=15):
    from brepgen_b200.schedulers import DPMSolverMultistepScheduler, UniPCMultistepScheduler
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(0)
    eps_c, eps_u, x = (torch.randn(n, generator=g, device="cuda") for _ in range(3))
    out, hist_d, last = torch.empty_like(x), torch.zeros_like(x), torch.zeros_like(x)
    hist_u = torch.zeros(3, n, device="cuda")
    lib, st = f.lib(), f.current_stream()
    d = DPMSolverMultistepScheduler(clip_sample=True, clip_sample_range=3)
    d.set_timesteps(20)
    cd, td = d.step_coefficients(10, 2), int(d.timesteps[10])

    def dpm_fn(u):
        return lambda: lib.bg_dpm_step(eps_c.data_ptr(), f.ptr(u), 0.6, x.data_ptr(), out.data_ptr(), hist_d.data_ptr(),
                                       None, 7, 0, None, 0, td, n, *cd, 3.0, st)

    def unipc_fn(u, order):
        s = UniPCMultistepScheduler(solver_order=order, final_sigmas_type="zero", clip_sample=True, clip_sample_range=3)
        s.set_timesteps(20)
        row = s.coefficient_table()[10]
        assert int(row[2]) == order and int(row[3]) == order       # a middle step: corrector and predictor of that order
        return lambda: lib.bg_unipc_step(eps_c.data_ptr(), f.ptr(u), 0.6, x.data_ptr(), out.data_ptr(), last.data_ptr(),
                                         hist_u.data_ptr(), order, per, n, row.data_ptr(), 3.0, st)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / iters
    for order in (2, 3):
        for cfg, u in (("no CFG", None), ("CFG", eps_u)):
            fa, fb = dpm_fn(u), unipc_fn(u, order)
            assert fa() == 0 and fb() == 0
            for _ in range(3):
                timed(fa), timed(fb)
            ta, tb = [], []
            for _ in range(rounds):
                ta.append(timed(fa))
                tb.append(timed(fb))
            ma, mb = statistics.median(ta), statistics.median(tb)
            base = n * 4 * (4 if u is not None else 3)  # eps [+ uncond], x, out
            nb_a = base + n * 4 * 2                     # + hist read and write
            nb_b = base + n * 4 * (2 + order + 1)       # + last read and write, order slots read, one written
            print(f"step UniPC order {order} with corrector (vs DPM++ 2M) {cfg}: n = {n}  bg_dpm_step {ma:.1f} us "
                  f"({nb_a / ma / 1e3:.0f} GB/s)  bg_unipc_step {mb:.1f} us ({nb_b / mb / 1e3:.0f} GB/s)  unipc / dpm = "
                  f"{mb / ma:.3f}  (spread {min(ta):.1f}-{max(ta):.1f} / {min(tb):.1f}-{max(tb):.1f} us)", flush=True)


def cascade_times(B=64, S0=50, E=40):
    from brepgen_b200.models import NETS
    from brepgen_b200.sampler import Cascade, CascadeConfig
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
    base = dict(batch_size=B, num_surfaces=S0, num_edges=E, dense_masks=True, seed=1000)
    arms = {"UniPC-10": (CascadeConfig(schedule="unipc", unipc_steps=10, **base), 10),
            "DPM-20": (CascadeConfig(schedule="dpm", dpm_steps=20, **base), 20),
            "DDIM-50": (CascadeConfig(schedule="ddim", ddim_steps=50, **base), 50)}
    g = torch.Generator().manual_seed(1000)
    S = 2 * S0
    init = {k: torch.randn(s, generator=g).to(dev) for k, s in
            {"surfPos": (B, S0, 6), "surfZ": (B, S, 48), "edgePos": (B, S, E, 6), "edgeZV": (B, S, E, 18)}.items()}
    for cfg, _ in arms.values():                        # warm-up: packs weights, allocates workspaces
        out = casc.run(cfg, init_noise=init)
        torch.cuda.synchronize()
        assert all(torch.isfinite(v.float()).all() for v in out.values())
    clk = SmClock()
    clk.start()
    times, launches = {k: [] for k in arms}, {}
    for _ in range(CASCADES):
        for name, (cfg, _) in arms.items():
            l0 = f.lib().bg_launch_count() + f.replayed_launches
            t0 = time.perf_counter()
            casc.run(cfg, init_noise=init)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            launches[name] = f.lib().bg_launch_count() + f.replayed_launches - l0
    mhz = clk.stop()
    for name, (_, steps) in arms.items():
        s = statistics.median(times[name])
        print(f"cascade {name} B={B} S0={S0} E={E} dense: {s:.3f} s per cascade (spread {min(times[name]):.3f}-"
              f"{max(times[name]):.3f}), {B / s:.3f} B-reps/s, {launches[name]} launches, {4 * steps} network "
              f"evaluations", flush=True)
    print(f"median SM clock over the cascades: {mhz} MHz", flush=True)


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("tools/unipc_time.py measures on the GPU and needs one")
    print("GPU:", smi("name,power.limit,clocks.max.sm"), flush=True)
    step_times()
    cascade_times()
