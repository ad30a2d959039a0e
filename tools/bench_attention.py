#!/usr/bin/env python
"""Times the attention kernel alone, this build against another build of the library, and checks their outputs are
bit-identical.

    python tools/bench_attention.py OUT_DIR --baseline-lib PATH [--rounds 5] [--iters 20] [--batch 64] [--length 4000]

Both libraries are loaded into one process (one ctypes.CDLL each; the in-tree build, or $BG_LIB, is "new") and timed
alternately with CUDA events, `--rounds` times each, at B = 64, L = 4000 in the two call forms the project uses:
  varlen  variable-length mode (bg_op_attention_varlen), as the token-compacted edge-stage forwards call it;
  masked  an all-valid key-padding mask plus the per-forward block list (bg_op_attention), as bench.py's roofline does.
It prints and writes OUT_DIR/bench_attention.json: ms per launch (median, min, max over rounds), TFLOP/s (4 L^2 64 flop
per sample and head), the card name, power limit and median SM clock, and whether the two builds wrote the same bytes
on the timed inputs, on the ATTN_CASES of tests/test_gpu_ops.py and on a few ragged variable-length batches.  The
baseline library must export bg_op_attention_varlen.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def load(path):
    from brepgen_b200 import _ffi
    lib = C.CDLL(os.path.abspath(path))
    for name in ("bg_last_error", "bg_op_attention", "bg_op_attention_varlen"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = _ffi.SIGNATURES[name]
    return lib


def check(lib, status, what):
    if status != 0:
        raise RuntimeError(f"{what} failed (status {status}): {lib.bg_last_error().decode(errors='replace')}")


class Case:
    """inputs of one attention call; run(lib) launches it on the current stream into a NaN-filled output"""

    def __init__(self, B, L, qkv, mask=None, lens=None):
        import torch
        self.B, self.L, self.qkv, self.mask = B, L, qkv, mask
        self.out = torch.empty(B * L, 768, device="cuda", dtype=torch.float16)
        self.scratch = torch.zeros(B * (5 * ((L + 127) // 128) + 1), dtype=torch.int32, device="cuda")
        self.lens = self.row0 = None
        if lens is not None:
            self.lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
            self.row0 = torch.zeros_like(self.lens)
            self.row0[1:] = torch.cumsum(self.lens, 0)[:-1]

    def launch(self, lib):
        import torch
        st = torch.cuda.current_stream().cuda_stream
        if self.lens is not None:
            check(lib, lib.bg_op_attention_varlen(self.qkv.data_ptr(), self.out.data_ptr(), self.B, self.L,
                                                  self.row0.data_ptr(), self.lens.data_ptr(), st), "attention varlen")
        else:
            check(lib, lib.bg_op_attention(self.qkv.data_ptr(), self.out.data_ptr(), self.B, self.L,
                                           None if self.mask is None else self.mask.data_ptr(), 1,
                                           self.scratch.data_ptr(), st), "attention")

    def result(self, lib):
        """the output bytes of one launch (rows outside every sample in variable-length mode are not written: NaN)"""
        import torch
        self.out.fill_(float("nan"))
        self.launch(lib)
        torch.cuda.synchronize()
        return self.out.clone()


def attn_cases_of_tests():
    """the inputs of tests/test_gpu_ops.py::test_attention, built the same way"""
    import torch
    from test_gpu_ops import ATTN_CASES
    out = []
    for B, L, mkind, _ in ATTN_CASES:
        g = torch.Generator(device="cuda").manual_seed(B * 1000 + L)
        qkv = (torch.randn(B * L, 2304, generator=g, device="cuda") * 1.5).half()
        mask = None
        if mkind == "tail":
            mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
            mask[0, L // 2:] = True
        elif mkind == "rand":
            mask = torch.rand(B, L, generator=g, device="cuda") < 0.3
            mask[:, 0] = False
        elif mkind == "ragged":
            nvalid = torch.randint(1, L + 1, (B,), generator=g, device="cuda")
            nvalid[0] = L
            mask = torch.arange(L, device="cuda")[None, :] >= nvalid[:, None]
            mask |= torch.rand(B, L, generator=g, device="cuda") < 0.1
            mask[:, 0] = False
        elif mkind == "blocks":
            mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
            mask[0, 128:512] = True
            mask[1, 700:] = True
            mask[1, 5] = True
        out.append((f"test_gpu_ops B={B} L={L} mask={mkind}", Case(B, L, qkv, mask)))
    return out


def varlen_cases():
    import torch
    out = []
    for lens, L, seed in (([0, 1, 127, 128, 129, 255, 4000], 4000, 1), ([4000, 3999, 2500, 130, 1], 4000, 2),
                          (torch.randint(1, 1025, (40,), generator=torch.Generator().manual_seed(3)).tolist(), 1024, 3)):
        g = torch.Generator(device="cuda").manual_seed(seed)
        qkv = (torch.randn(len(lens) * L, 2304, generator=g, device="cuda") * 1.5).half()
        out.append((f"varlen lens={lens if len(lens) < 10 else str(len(lens)) + ' samples'} L={L}",
                    Case(len(lens), L, qkv, lens=lens)))
    return out


def time_round(case, lib, iters):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    case.launch(lib)
    e0.record()
    for _ in range(iters):
        case.launch(lib)
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
    a = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_attention.py: needs a CUDA device")
    from brepgen_b200 import _ffi
    from profile_edge_layer import Clocks, card_info
    os.makedirs(a.out_dir, exist_ok=True)
    libs = {"base": load(a.baseline_lib), "new": load(_ffi.LIB_PATH)}
    dev = torch.cuda.current_device()
    info = card_info(dev)
    print(f"card: {info}\nbase: {os.path.abspath(a.baseline_lib)}\nnew:  {os.path.abspath(_ffi.LIB_PATH)}")

    B, L = a.batch, a.length
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B * L, 2304, generator=g, device="cuda").half()
    timed = {"varlen": Case(B, L, qkv, lens=[L] * B),
             "masked": Case(B, L, qkv, mask=torch.zeros(B, L, dtype=torch.bool, device="cuda"))}
    flop = B * 3072.0 * L * L
    res = {"card": info, "B": B, "L": L, "rounds": a.rounds, "iters": a.iters, "flop_per_launch": flop, "timing": {},
           "bit_identical": {}}
    for form, case in timed.items():
        ms = {k: [] for k in libs}
        clocks = Clocks(dev)
        clocks.start()
        for _ in range(a.rounds):
            for k, lib in libs.items():
                ms[k].append(time_round(case, lib, a.iters))
        mhz = clocks.finish()
        row = {"median_sm_mhz": mhz}
        for k in libs:
            med = statistics.median(ms[k])
            row[k] = {"ms_median": med, "ms_min": min(ms[k]), "ms_max": max(ms[k]), "ms_all": ms[k],
                      "tflops": flop / (med / 1e3) / 1e12}
        row["speedup"] = row["base"]["ms_median"] / row["new"]["ms_median"]
        res["timing"][form] = row
        print(f"{form:>7}: base {row['base']['ms_median']:.3f} ms [{row['base']['ms_min']:.3f}, {row['base']['ms_max']:.3f}] "
              f"{row['base']['tflops']:.0f} TFLOP/s | new {row['new']['ms_median']:.3f} ms [{row['new']['ms_min']:.3f}, "
              f"{row['new']['ms_max']:.3f}] {row['new']['tflops']:.0f} TFLOP/s | x{row['speedup']:.3f}  SM clock {mhz} MHz")
    del qkv

    cases = [(f"timed {k} B={B} L={L}", c) for k, c in timed.items()] + attn_cases_of_tests() + varlen_cases()
    all_equal = True
    for name, case in cases:
        same = torch.equal(case.result(libs["base"]).view(torch.int16), case.result(libs["new"]).view(torch.int16))
        res["bit_identical"][name] = same
        all_equal &= same
        print(f"  {'equal' if same else 'DIFFERENT'}  {name}")
        del case
    res["all_bit_identical"] = all_equal
    with open(os.path.join(a.out_dir, "bench_attention.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"outputs bit-identical in every case: {all_equal}")
    if not all_equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
