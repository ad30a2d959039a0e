"""Time the DDIM step and a DDIM cascade on one GPU.

  1. bg_ddim_step against bg_ddpm_step at the edgeZV size of the benchmark (B = 64 samples of 100 x 40 x 18 = 72 000
     elements: 4.6 M), eta = 0 and eta = 1 (in-kernel batch-stream noise), CFG off and on.  Rounds alternate between the
     two kernels; prints the median per-launch time of each.
  2. Cascade.run(schedule="ddim", ddim_steps=N) at the benchmark workload (B = 64, S0 = 50, E = 40, dense masks, random-init
     weights, both decoders): seconds per cascade, B-reps/s and kernel launches (host launches + kernels in graph replays).
     The whole schedule runs; nothing is scaled.

    python tools/ddim_time.py            # env: DDIM_STEPS (50), CASCADES (3)
Prints the card, its power limit and the median SM clock sampled while the cascades ran.
"""
import os
import statistics
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from brepgen_b200 import _ffi as f  # noqa: E402

DDIM_STEPS = int(os.environ.get("DDIM_STEPS", 50))
CASCADES = int(os.environ.get("CASCADES", 3))


def smi(q):
    return subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()


class SmClock(threading.Thread):
    """samples clocks.sm every 0.2 s until stop(); median in MHz"""

    def __init__(self):
        super().__init__(daemon=True)
        self.rows, self.halt = [], threading.Event()

    def run(self):
        while not self.halt.is_set():
            v = smi("clocks.sm").split()
            if v and v[0].isdigit():
                self.rows.append(int(v[0]))
            self.halt.wait(0.2)

    def stop(self):
        self.halt.set()
        self.join(timeout=3)
        return statistics.median(self.rows) if self.rows else None


def step_times(B=64, per=100 * 40 * 18, iters=200, rounds=15):
    from brepgen_b200.schedulers import DDIMScheduler, DDPMScheduler
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(0)
    eps_c, eps_u, x = (torch.randn(n, generator=g, device="cuda") for _ in range(3))
    out = torch.empty_like(x)
    lib, st = f.lib(), f.current_stream()
    ddpm = DDPMScheduler(clip_sample=True, clip_sample_range=3)
    ddpm.set_timesteps(1000)
    ddim = DDIMScheduler(clip_sample=True, clip_sample_range=3)
    ddim.set_timesteps(50)
    c_ddpm = ddpm.step_coefficients(500)

    def ddpm_fn(u):
        return lambda: lib.bg_ddpm_step(eps_c.data_ptr(), f.ptr(u), 0.6, x.data_ptr(), out.data_ptr(), None, 7, 0, None, 0,
                                        500, n, *c_ddpm[:2], 3.0, *c_ddpm[2:], st)

    def ddim_fn(u, eta):
        c = ddim.step_coefficients(500, eta)
        return lambda: lib.bg_ddim_step(eps_c.data_ptr(), f.ptr(u), 0.6, x.data_ptr(), out.data_ptr(), None, 7, 0, None, 0,
                                        500, n, *c, 3.0, 0, st)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / iters
    for eta in (0.0, 1.0):
        for cfg, u in (("no CFG", None), ("CFG", eps_u)):
            fa, fb = ddpm_fn(u), ddim_fn(u, eta)
            assert fa() == 0 and fb() == 0
            for _ in range(3):
                timed(fa), timed(fb)
            ta, tb = [], []
            for _ in range(rounds):
                ta.append(timed(fa))
                tb.append(timed(fb))
            ma, mb = statistics.median(ta), statistics.median(tb)
            nbytes = n * 4 * (4 if u is not None else 3)
            print(f"step eta={eta:g} {cfg}: n = {n}  bg_ddpm_step {ma:.1f} us ({nbytes / ma / 1e3:.0f} GB/s)  bg_ddim_step "
                  f"{mb:.1f} us ({nbytes / mb / 1e3:.0f} GB/s)  ddim / ddpm = {mb / ma:.3f}  (spread {min(ta):.1f}-"
                  f"{max(ta):.1f} / {min(tb):.1f}-{max(tb):.1f} us)", flush=True)


def cascade_time(B=64, S0=50, E=40):
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
    cfg = CascadeConfig(batch_size=B, num_surfaces=S0, num_edges=E, schedule="ddim", ddim_steps=DDIM_STEPS, dense_masks=True,
                        seed=1000)
    g = torch.Generator().manual_seed(1000)
    S = 2 * S0
    init = {k: torch.randn(s, generator=g).to(dev) for k, s in
            {"surfPos": (B, S0, 6), "surfZ": (B, S, 48), "edgePos": (B, S, E, 6), "edgeZV": (B, S, E, 18)}.items()}
    out = casc.run(cfg, init_noise=init)                      # warm-up: packs weights, allocates workspaces
    torch.cuda.synchronize()
    assert all(torch.isfinite(v.float()).all() for v in out.values())
    clk = SmClock()
    clk.start()
    times = []
    for _ in range(CASCADES):
        l0 = f.lib().bg_launch_count() + f.replayed_launches
        t0 = time.perf_counter()
        casc.run(cfg, init_noise=init)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        launches = f.lib().bg_launch_count() + f.replayed_launches - l0
    mhz = clk.stop()
    s = statistics.median(times)
    print(f"cascade DDIM-{DDIM_STEPS} B={B} S0={S0} E={E} dense: {s:.3f} s per cascade (spread {min(times):.3f}-"
          f"{max(times):.3f}), {B / s:.3f} B-reps/s, {launches} launches, {4 * DDIM_STEPS} network evaluations, "
          f"median SM clock {mhz} MHz", flush=True)


if __name__ == "__main__":
    print("GPU:", smi("name,power.limit,clocks.max.sm"), flush=True)
    step_times()
    cascade_time()
