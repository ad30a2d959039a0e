"""Run a few forwards of one denoiser at ABC-eval shapes (under a profiler of your choice).

    python tools/profile_forward.py --kind edgepos --batch 8 --iters 1
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from brepgen_b200.models import NETS  # noqa: E402
from brepgen_b200.spec import denoiser_spec  # noqa: E402
from brepgen_b200.synth import synth_state_dict  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--kind", default="edgepos")
ap.add_argument("--batch", type=int, default=8)
ap.add_argument("--surfaces", type=int, default=100)
ap.add_argument("--edges", type=int, default=40)
ap.add_argument("--iters", type=int, default=1)
ap.add_argument("--precision", type=int, default=1)
ap.add_argument("--time", action="store_true", help="print CUDA-event time per forward")
a = ap.parse_args()

m = NETS[a.kind](False)
m.load_state_dict(synth_state_dict(denoiser_spec(a.kind, False), seed=1))
m.precision = a.precision
m = m.cuda().eval()
B, S, E = a.batch, a.surfaces, a.edges
g = torch.Generator(device="cuda").manual_seed(0)
r = lambda *s: torch.randn(*s, generator=g, device="cuda")
t = torch.tensor([500], device="cuda")
fm = torch.zeros(B, S, dtype=torch.bool, device="cuda")
em = torch.zeros(B, S, E, dtype=torch.bool, device="cuda")
args = {"surfpos": (r(B, S, 6), t, None), "surfz": (r(B, S, 48), t, r(B, S, 6), fm, None),
        "edgepos": (r(B, S, E, 6), t, r(B, S, 6), r(B, S, 48), fm, None),
        "edgez": (r(B, S, E, 18), t, r(B, S, E, 6), r(B, S, 6), r(B, S, 48), em, None)}[a.kind]
with torch.no_grad():
    m(*args)   # packs weights, allocates the workspace
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        y = m(*args)
    e1.record()
    torch.cuda.synchronize()
if a.time:
    print(f"{a.kind} B={B} S={S} E={E} precision={a.precision}: {e0.elapsed_time(e1) / a.iters:.3f} ms / forward")
assert torch.isfinite(y).all()
