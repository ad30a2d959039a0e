#!/usr/bin/env python
"""Per-kernel breakdown of one edge-stage denoiser forward on the GPU.

    python tools/profile_edge_layer.py OUT_DIR [--nets edgez,edgepos] [--forwards 5] [--warmup 3] [--batch 64]

Builds EdgeZNet / EdgePosNet from synth_state_dict at the bench.py workload (B = 64, S = 100, E = 40, dense masks, token
compaction on), warms up, times forwards with CUDA events, then records forwards with torch.profiler (CUDA activities) in
a run of their own. Kernels are attributed by their position in the encoder layer sequence
LN1, QKV, attn, out_proj, LN2, linear1, linear2 (the four GEMMs share one kernel name). Per operation it prints the mean
time, the share of the forward's kernel time, TFLOP/s (from shapes, counting the hi / lo K terms the precision runs) and
HBM GB/s (from the bytes the operation must move), and writes OUT_DIR/profile_<net>.json with the card name, power limit
and median SM clock read during the profiled run. `BG_LIB` selects another build of the library (see brepgen_b200/_ffi.py).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D, FF, NLAYER = 768, 1024, 12
OPS = ("LN1", "QKV", "attn", "out_proj", "LN2", "linear1", "linear2")
PATTERN = ("layernorm", "gemm", "attn", "gemm", "layernorm", "gemm", "gemm")


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("out_dir")
    ap.add_argument("--nets", default="edgez,edgepos")
    ap.add_argument("--forwards", type=int, default=5, help="forwards recorded by the profiler (and timed with events)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--surfaces", type=int, default=100)
    ap.add_argument("--edges", type=int, default=40)
    a = ap.parse_args(argv)
    a.nets = [n for n in a.nets.split(",") if n]
    for n in a.nets:
        if n not in ("edgez", "edgepos"):
            ap.error(f"unknown net {n!r} (edgez, edgepos)")
    return a


def op_model(precision, rows):
    """flop and HBM bytes per operation of one encoder layer over `rows` token rows. K per GEMM follows the weight
    packing of csrc/denoiser.cu: precision 1 splits in_proj's v rows and out_proj into [W_hi | W_lo] (q | k column tiles
    stop after the hi half), precision 2 splits every matrix."""
    s_attn, s_ff = precision >= 1, precision >= 2
    k_qk = 2 * D if s_ff else D
    k_v = 2 * D if s_attn else D
    k_o = 2 * D if s_attn else D
    k_1 = 2 * D if s_ff else D
    k_2 = 2 * FF if s_ff else FF
    gemm = lambda n, k, a_bytes, out_bytes, resid: (2.0 * rows * n * k, rows * (a_bytes + out_bytes * (2 if resid else 1)) + n * k * 2)
    qkv_f = 2.0 * rows * (2 * D * k_qk + D * k_v)
    qkv_b = rows * (D * 2 + 3 * D * 2) + (2 * D * k_qk + D * k_v) * 2
    return {
        "LN1": (0.0, rows * (D * 4 + D * 2)),
        "QKV": (qkv_f, qkv_b),
        "attn": (None, rows * (3 * D * 2 + D * 2)),                       # flop filled in per sample length
        "out_proj": gemm(D, k_o, D * 2, D * 4, True),                     # fp32 residual read + write in place
        "LN2": (0.0, rows * (D * 4 + D * 2)),
        "linear1": gemm(FF, k_1, D * 2, FF * 2, False),
        "linear2": gemm(D, k_2, FF * 2, D * 4, True),
    }


class Clocks(threading.Thread):
    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.mhz, self._halt = index, [], threading.Event()

    def run(self):
        while not self._halt.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.index}", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out.isdigit():
                    self.mhz.append(int(out))
            except Exception:
                pass
            self._halt.wait(0.1)

    def finish(self):
        self._halt.set()
        self.join(timeout=3)
        return statistics.median(self.mhz) if self.mhz else None


def card_info(index):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
        name, power, mx = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": mx}
    except Exception as e:          # the figures are reported as unknown rather than guessed
        return {"name": None, "power_limit": None, "sm_max_clock": None, "error": str(e)}


def build_net(kind, B, S, E, dev):
    import torch
    from brepgen_b200.models import NETS
    from brepgen_b200.spec import denoiser_spec
    from brepgen_b200.synth import synth_state_dict
    m = NETS[kind](False)
    m.load_state_dict(synth_state_dict(denoiser_spec(kind, False), seed=1))
    m = m.to(dev).eval()
    m.compact = 1
    g = torch.Generator().manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g).to(dev)
    t = torch.tensor([500], device=dev)
    sP, sZ = r(B, S, 6), r(B, S, 48)
    if kind == "edgez":
        x, eP, mask = r(B, S, E, 18), r(B, S, E, 6), torch.zeros(B, S, E, dtype=torch.bool, device=dev)
        fwd = lambda: m(x, t, eP, sP, sZ, mask, None)
    else:
        x, mask = r(B, S, E, 6), torch.zeros(B, S, dtype=torch.bool, device=dev)
        fwd = lambda: m(x, t, sP, sZ, mask, None)
    return m, fwd


def kernel_trace(fwd, n):
    """[(name, ts_us, dur_us)] of every CUDA kernel of n forwards, in launch order"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.no_grad():
            for _ in range(n):
                fwd()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    ks = [(e["name"], float(e["ts"]), float(e["dur"])) for e in ev if e.get("cat") == "kernel"]
    return sorted(ks, key=lambda k: k[1])


def attribute(kernels, n_forwards):
    """per-operation durations (us) of every encoder layer found in the trace, matched by position"""
    per = {op: [] for op in OPS}
    names = [k[0] for k in kernels]
    i, layers = 0, 0
    while i + len(PATTERN) <= len(names):
        if all(p in names[i + j] for j, p in enumerate(PATTERN)):
            for j, op in enumerate(OPS):
                per[op].append(kernels[i + j][2])
            i += len(PATTERN)
            layers += 1
        else:
            i += 1
    if layers != NLAYER * n_forwards:
        raise RuntimeError(f"found {layers} encoder layers in the trace, expected {NLAYER * n_forwards}: kernel names "
                           f"changed? first kernels: {names[:12]}")
    return per


def profile_net(kind, a, dev, info):
    import torch
    B, S, E = a.batch, a.surfaces, a.edges
    L, rows = S * E, a.batch * S * E
    m, fwd = build_net(kind, B, S, E, dev)
    with torch.no_grad():
        for _ in range(a.warmup):
            fwd()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.forwards):
            fwd()
        e1.record()
        torch.cuda.synchronize()
    fwd_ms = e0.elapsed_time(e1) / a.forwards
    clocks = Clocks(dev.index or 0)
    clocks.start()
    kernels = kernel_trace(fwd, a.forwards)
    mhz = clocks.finish()
    per = attribute(kernels, a.forwards)
    kernel_ms = sum(k[2] for k in kernels) / a.forwards / 1e3
    model = op_model(m.precision, rows)
    res = {}
    print(f"\n{kind}: B={B} S={S} E={E} rows={rows} precision={m.precision}  forward {fwd_ms:.2f} ms (events), "
          f"kernel time {kernel_ms:.2f} ms per forward, median SM clock {mhz} MHz")
    print(f"{'op':>9} {'mean ms':>9} {'share':>7} {'TFLOP/s':>8} {'GB/s':>7}")
    layer_ms = 0.0
    for op in OPS:
        ms = statistics.mean(per[op]) / 1e3
        flop, byts = model[op]
        if op == "attn":
            flop = B * 3072.0 * L * L
        share = ms * NLAYER / kernel_ms
        tf = flop / (ms / 1e3) / 1e12 if flop else None
        gbs = byts / (ms / 1e3) / 1e9
        layer_ms += ms
        res[op] = {"mean_ms": ms, "min_ms": min(per[op]) / 1e3, "max_ms": max(per[op]) / 1e3, "share_of_forward": share,
                   "tflop": flop / 1e12, "tflops": tf, "hbm_bytes": byts, "gbs": gbs}
        print(f"{op:>9} {ms:9.3f} {share:7.1%} {tf if tf else 0:8.1f} {gbs:7.0f}")
    print(f"{'layer':>9} {layer_ms:9.3f} {layer_ms * NLAYER / kernel_ms:7.1%}")
    out = {"net": kind, "B": B, "S": S, "E": E, "rows": rows, "precision": m.precision, "forwards": a.forwards,
           "forward_ms_events": fwd_ms, "kernel_ms_per_forward": kernel_ms, "layer_ms": layer_ms,
           "median_sm_mhz": mhz, "card": info, "lib": os.path.abspath(os.environ.get("BG_LIB", "")) or "in-tree",
           "ops": res}
    with open(os.path.join(a.out_dir, f"profile_{kind}.json"), "w") as f:
        json.dump(out, f, indent=1)
    del m, fwd
    torch.cuda.empty_cache()
    return out


def main(argv=None):
    a = parse(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("profile_edge_layer.py: needs a CUDA device")
    os.makedirs(a.out_dir, exist_ok=True)
    dev = torch.device("cuda", torch.cuda.current_device())
    info = card_info(dev.index)
    print(f"card: {info}  lib: {os.environ.get('BG_LIB', 'in-tree')}")
    for kind in a.nets:
        profile_net(kind, a, dev, info)


if __name__ == "__main__":
    main()
