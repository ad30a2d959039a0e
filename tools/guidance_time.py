"""Time per-sample classifier-free guidance on one GPU.

  1. bg_cfg_combine against the fp32 torch expression pc * (1 + w) - pu[rows] * w at the CF edgeZV size of the benchmark
     (B = 64 samples of 60 x 40 x 18 = 43 200 elements: 2.76 M), in place, with every sample guided and with half of them
     guided.  Rounds alternate between the two; prints the median per-call time of each.
  2. Cascade.run at the benchmark's CF workload (B = 64, S0 = 60, E = 40, dense masks, random-init weights, both
     decoders) under DDIM-50 and UniPC-10: the scalar config (guidance_w 0.6) and per-sample configs with 0 %, 50 % and
     100 % unguided samples (the guided ones at w = 0.6, mixed class labels), alternated in one process: seconds per
     cascade and network rows per evaluation.  The whole schedule runs; nothing is scaled.

    python tools/guidance_time.py          # env: CASCADES (3)
Prints the card, its power limit and the median SM clock sampled while the cascades ran.  The weights are random-init,
so only costs are measured.  Needs a GPU.
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


def combine_times(B=64, per=60 * 40 * 18, iters=200, rounds=15):
    g = torch.Generator(device="cuda").manual_seed(0)
    lib, st = f.lib(), f.current_stream()

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / iters
    for guided in (B, B // 2):
        gi = torch.arange(0, B, B // guided, device="cuda")[:guided]
        rows = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        rows[gi] = torch.arange(guided, dtype=torch.int32, device="cuda")
        w = torch.where(rows >= 0, 0.6, 0.0).float()
        pc = torch.randn(B, per, generator=g, device="cuda")
        pu = torch.randn(guided, per, generator=g, device="cuda")
        wc = w[gi, None]

        def kernel():
            lib.bg_cfg_combine(pc.data_ptr(), pu.data_ptr(), rows.data_ptr(), w.data_ptr(), B, guided, per,
                               pc.data_ptr(), st)

        def torch_expr():
            pc[gi] = pc[gi] * (1 + wc) - pu * wc
        kernel(), torch_expr()
        for _ in range(3):
            timed(kernel), timed(torch_expr)
        tk, tt = [], []
        for _ in range(rounds):
            tk.append(timed(kernel))
            tt.append(timed(torch_expr))
        mk, mt = statistics.median(tk), statistics.median(tt)
        nbytes = guided * per * 4 * 3                   # guided samples: eps_c read + written, eps_u read
        print(f"combine B={B} per_sample={per} guided={guided}: bg_cfg_combine {mk:.1f} us ({nbytes / mk / 1e3:.0f} GB/s)"
              f"  torch expression {mt:.1f} us  torch / kernel = {mt / mk:.2f}  (spread {min(tk):.1f}-{max(tk):.1f} / "
              f"{min(tt):.1f}-{max(tt):.1f} us)", flush=True)


class _Rows:
    def __init__(self, m):
        self.m, self.rows = m, []

    def __call__(self, x, *a):
        self.rows.append(x.shape[0])
        return self.m(x, *a)


def cascade_times(B=64, S0=60, E=40):
    from brepgen_b200.models import NETS
    from brepgen_b200.sampler import Cascade, CascadeConfig
    from brepgen_b200.spec import denoiser_spec
    from brepgen_b200.synth import synth_state_dict
    from brepgen_b200.vae import build_synthetic_decoders
    dev = torch.device("cuda")
    models = {}
    for kind in NETS:
        m = NETS[kind](True)
        m.load_state_dict(synth_state_dict(denoiser_spec(kind, True), seed=1))
        models[kind] = _Rows(m.to(dev).eval())
    sv, ev = build_synthetic_decoders(dev)
    casc = Cascade(models, sv, ev, device=dev)
    labels = [1 + b % 10 for b in range(B)]
    arms = {}
    for sched, kw in (("DDIM-50", dict(schedule="ddim", ddim_steps=50)),
                      ("UniPC-10", dict(schedule="unipc", unipc_steps=10))):
        base = dict(batch_size=B, num_surfaces=S0, num_edges=E, dense_masks=True, seed=1000, use_cf=True, **kw)
        arms[f"{sched} scalar"] = CascadeConfig(class_label=6, guidance_w=0.6, **base)
        for pct in (0, 50, 100):
            w = [0.0 if b < B * pct // 100 else 0.6 for b in range(B)]
            arms[f"{sched} per-sample {pct}% unguided"] = CascadeConfig(class_label=labels, guidance_w=w, **base)
    g = torch.Generator().manual_seed(1000)
    init = {k: torch.randn(s, generator=g).to(dev) for k, s in
            {"surfPos": (B, S0, 6), "surfZ": (B, S0, 48), "edgePos": (B, S0, E, 6), "edgeZV": (B, S0, E, 18)}.items()}
    rows = {}
    for name, cfg in arms.items():                      # warm-up: packs weights, allocates workspaces
        for m in models.values():
            m.rows.clear()
        out = casc.run(cfg, init_noise=init)
        torch.cuda.synchronize()
        assert all(torch.isfinite(v.float()).all() for v in out.values())
        rows[name] = sorted(set(r for m in models.values() for r in m.rows))
    clk = SmClock()
    clk.start()
    times = {k: [] for k in arms}
    for _ in range(CASCADES):
        for name, cfg in arms.items():
            t0 = time.perf_counter()
            casc.run(cfg, init_noise=init)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
    mhz = clk.stop()
    for name in arms:
        s = statistics.median(times[name])
        print(f"cascade {name} B={B} S0={S0} E={E} dense: {s:.3f} s per cascade (spread {min(times[name]):.3f}-"
              f"{max(times[name]):.3f}), {B / s:.3f} B-reps/s, forward rows {rows[name]}", flush=True)
    print(f"median SM clock over the cascades: {mhz} MHz", flush=True)


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("tools/guidance_time.py measures on the GPU and needs one")
    print("GPU:", smi("name,power.limit,clocks.max.sm"), flush=True)
    combine_times()
    cascade_times()
