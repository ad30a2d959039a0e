"""Time the DDPM step (bg_ddpm_step) with per-sample keys against the step with the batch stream at the edgeZV size of the
benchmark (B = 64 samples of 100 x 40 x 18 = 72 000 elements: 4.6 M), with and without the CFG combine.  Both draw
their noise in the kernel.  Rounds alternate between the two forms; prints the median per-launch time of each.
    python tools/ddpm_keyed_time.py
"""
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from brepgen_b200 import _ffi as f  # noqa: E402
from brepgen_b200.schedulers import sample_keys, sample_seed  # noqa: E402


def main(B=64, per=100 * 40 * 18, iters=200, rounds=15):
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(0)
    eps_c, eps_u, x = (torch.randn(n, generator=g, device="cuda") for _ in range(3))
    out = torch.empty_like(x)
    keys = torch.from_numpy(sample_keys([sample_seed(0, b) for b in range(B)], 3).view(np.int64)).cuda()
    lib, st = f.lib(), f.current_stream()
    coef = (0.5, 0.8, 0.3, 0.6, 0.1)

    def step(u, k):
        return lambda: lib.bg_ddpm_step(eps_c.data_ptr(), f.ptr(u), 0.6, x.data_ptr(), out.data_ptr(), None, 7, 0, f.ptr(k),
                                        per, 500, n, *coef[:2], 3.0, *coef[2:], st)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / iters
    for cfg, u in (("no CFG", None), ("CFG", eps_u)):
        fb, fk = step(u, None), step(u, keys)
        assert fb() == 0 and fk() == 0
        for _ in range(3):
            timed(fb), timed(fk)
        tb, tk = [], []
        for _ in range(rounds):
            tb.append(timed(fb))
            tk.append(timed(fk))
        mb, mk = statistics.median(tb), statistics.median(tk)
        nbytes = n * 4 * (4 if u is not None else 3)
        print(f"{cfg}: n = {n}  batch stream {mb:.1f} us ({nbytes / mb / 1e3:.0f} GB/s)  keyed {mk:.1f} us "
              f"({nbytes / mk / 1e3:.0f} GB/s)  keyed / batch = {mk / mb:.3f}  (spread {min(tb):.1f}-{max(tb):.1f} / "
              f"{min(tk):.1f}-{max(tk):.1f} us)", flush=True)


if __name__ == "__main__":
    main()
