#!/usr/bin/env python
"""Times the encoder layer's GEMMs alone, this build against another build of the library, and checks their outputs are
bit-identical.

    python tools/bench_gemm.py OUT_DIR --baseline-lib PATH [--rounds 5] [--iters 20] [--batch 64] [--length 4000]
                                       [--timing-only]

Both libraries are loaded into one process (one ctypes.CDLL each; the in-tree build, or $BG_LIB, is "new") and timed
alternately with CUDA events, `--rounds` times each, at M = B L rows in the precision-1 forms the edge-stage encoder
layers run through bg_op_gemm_f16_ex:
  qkv        N 2304, K 1536 over A of 768 columns (a_kwrap 768); the q|k column tiles (n < 1536) stop at K = 768; fp16 out
  out_proj   N 768, K 1536 (a_kwrap 768), fp32 in-place residual
  linear1    N 1024, K 768, ReLU, fp16 out
  linear2    N 768, K 1024, fp32 in-place residual
  compact    the linear1 form with a device row count *m_dev = 0.8 M + 17 (token compaction)
It prints and writes OUT_DIR/bench_gemm.json: ms per launch (median, min, max over rounds), TFLOP/s, the rate at which
TMA fills shared memory from L2 (A tile + W tile bytes per k-block of every 128 x 256 tile, over kernel time), the card
name, power limit and median SM clock, and whether the two builds wrote the same bytes for every form.  `--timing-only`
skips that comparison, for diagnostic builds whose results are wrong by design (a main loop that skips loads, an
epilogue that skips stores).  Timing a build against itself gives the run-to-run spread.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

D, FF, BM, BK = 768, 1024, 128, 64


def load(path):
    from brepgen_b200 import _ffi
    lib = C.CDLL(os.path.abspath(path))
    for name in ("bg_last_error", "bg_op_gemm_f16_ex"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = _ffi.SIGNATURES[name]
    return lib


class Form:
    """one GEMM call: A [M, lda] fp16, W [N, K] fp16, out fp16 or fp32 (in place on the residual when resid)"""

    def __init__(self, name, M, N, K, a_cols, out, *, resid=False, relu=0, n_short=0, k_short=0, m_rows=None, A, W, bias):
        import torch
        self.name, self.M, self.N, self.K = name, M, N, K
        self.A, self.W, self.bias, self.out, self.resid, self.relu = A, W, bias, out, resid, relu
        self.a_kwrap = a_cols if a_cols < K else 0
        self.n_short, self.k_short = n_short, k_short
        self.m_dev = None if m_rows is None else torch.tensor([m_rows], dtype=torch.int32, device="cuda")
        self.init = out.clone()        # the residual (or NaN) the output starts from in the comparison
        rows = M if m_rows is None else min(M, m_rows)
        self.flop = 2.0 * rows * sum(self.k_of(n) for n in range(N))
        # BN as launch_gemm_f16 picks it at these sizes (many more 128 x 256 tiles than SMs)
        bn = 256 if N % 256 == 0 else 128
        tiles_m = -(-rows // BM)
        self.smem_bytes = tiles_m * sum(self.k_of(n0) // BK * (BM + bn) * BK * 2 for n0 in range(0, N, bn))

    def k_of(self, n):
        return self.k_short if n < self.n_short else self.K

    def launch(self, lib):
        import torch
        o = self.out.data_ptr()
        s = lib.bg_op_gemm_f16_ex(self.A.data_ptr(), self.A.shape[1], self.W.data_ptr(), self.K, self.M, self.N, self.K,
                                  o, self.N, int(self.out.dtype == torch.float16), self.relu, self.bias.data_ptr(),
                                  o if self.resid else None, self.N if self.resid else 0, None, 1, 0, self.a_kwrap,
                                  self.n_short, self.k_short, None if self.m_dev is None else self.m_dev.data_ptr(), None,
                                  torch.cuda.current_stream().cuda_stream)
        if s != 0:
            raise RuntimeError(f"{self.name} failed (status {s}): {lib.bg_last_error().decode(errors='replace')}")

    def result(self, lib):
        import torch
        self.out.copy_(self.init)
        self.launch(lib)
        torch.cuda.synchronize()
        r = self.out.clone()
        return r.view(torch.int16) if r.dtype == torch.float16 else r.view(torch.int32)


def forms(M):
    import torch
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda")
    x, h = rnd(M, D).half(), rnd(M, FF).half()
    resid = rnd(M, D)
    nan16 = lambda n: torch.full((M, n), float("nan"), device="cuda", dtype=torch.float16)
    w = lambda n, k, kin: (rnd(n, k) / kin ** 0.5).half()
    return [
        Form("qkv", M, 3 * D, 2 * D, D, nan16(3 * D), n_short=2 * D, k_short=D, A=x, W=w(3 * D, 2 * D, D), bias=rnd(3 * D)),
        Form("out_proj", M, D, 2 * D, D, resid.clone(), resid=True, A=x, W=w(D, 2 * D, D), bias=rnd(D)),
        Form("linear1", M, FF, D, D, nan16(FF), relu=1, A=x, W=w(FF, D, D), bias=rnd(FF)),
        Form("linear2", M, D, FF, FF, resid.clone(), resid=True, A=h, W=w(D, FF, FF), bias=rnd(D)),
        Form("compact", M, FF, D, D, nan16(FF), relu=1, m_rows=(4 * M) // 5 + 17, A=x, W=w(FF, D, D), bias=rnd(FF)),
    ]


def time_round(form, lib, iters):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    form.launch(lib)
    e0.record()
    for _ in range(iters):
        form.launch(lib)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("out_dir")
    ap.add_argument("--baseline-lib", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--length", type=int, default=4000)
    ap.add_argument("--timing-only", action="store_true")
    a = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_gemm.py: needs a CUDA device")
    from brepgen_b200 import _ffi
    from profile_edge_layer import Clocks, card_info
    os.makedirs(a.out_dir, exist_ok=True)
    libs = {"base": load(a.baseline_lib), "new": load(_ffi.LIB_PATH)}
    dev = torch.cuda.current_device()
    info = card_info(dev)
    print(f"card: {info}\nbase: {os.path.abspath(a.baseline_lib)}\nnew:  {os.path.abspath(_ffi.LIB_PATH)}")

    M = a.batch * a.length
    fs = forms(M)
    res = {"card": info, "M": M, "rounds": a.rounds, "iters": a.iters, "timing": {}, "bit_identical": {}}
    total = {k: 0.0 for k in libs}
    for f in fs:
        ms = {k: [] for k in libs}
        clocks = Clocks(dev)
        clocks.start()
        for _ in range(a.rounds):
            for k, lib in libs.items():
                ms[k].append(time_round(f, lib, a.iters))
        mhz = clocks.finish()
        row = {"median_sm_mhz": mhz, "flop": f.flop, "smem_fill_bytes": f.smem_bytes}
        for k in libs:
            med = statistics.median(ms[k])
            row[k] = {"ms_median": med, "ms_min": min(ms[k]), "ms_max": max(ms[k]), "ms_all": ms[k],
                      "tflops": f.flop / (med / 1e3) / 1e12, "smem_fill_tbs": f.smem_bytes / (med / 1e3) / 1e12}
            if f.name != "compact":
                total[k] += med
        row["speedup"] = row["base"]["ms_median"] / row["new"]["ms_median"]
        res["timing"][f.name] = row
        b, n = row["base"], row["new"]
        print(f"{f.name:>8}: base {b['ms_median']:.3f} ms [{b['ms_min']:.3f}, {b['ms_max']:.3f}] {b['tflops']:.0f} TFLOP/s "
              f"{b['smem_fill_tbs']:.2f} TB/s | new {n['ms_median']:.3f} ms [{n['ms_min']:.3f}, {n['ms_max']:.3f}] "
              f"{n['tflops']:.0f} TFLOP/s {n['smem_fill_tbs']:.2f} TB/s | x{row['speedup']:.3f}  SM clock {mhz} MHz")
    res["four_gemms_ms"] = total
    res["four_gemms_speedup"] = total["base"] / total["new"]
    print(f"qkv + out_proj + linear1 + linear2: base {total['base']:.3f} ms, new {total['new']:.3f} ms, "
          f"x{res['four_gemms_speedup']:.3f}")

    all_equal = True
    if not a.timing_only:
        for f in fs:
            same = torch.equal(f.result(libs["base"]), f.result(libs["new"]))
            res["bit_identical"][f.name] = same
            all_equal &= same
            print(f"  {'equal' if same else 'DIFFERENT'}  {f.name}")
        print(f"outputs bit-identical in every case: {all_equal}")
    res["all_bit_identical"] = all_equal if not a.timing_only else None
    with open(os.path.join(a.out_dir, "bench_gemm.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    if not all_equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
