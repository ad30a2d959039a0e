"""Golden vectors for the initial-noise helper (SURVEY.md section 8 row 2) from the reference's OWN function.

    python tests/golden/make_golden_randn.py        # writes tests/golden/randn_golden.npz   (build container only)

utils.py cannot be imported (OpenCASCADE / chamferdist at its top), so the definition of `randn_tensor`
(utils.py:60-97) is read from the reference file and exec()ed verbatim.  sample.py calls it as randn_tensor(shape) --
no generator, no device -- i.e. the CPU global generator, fp32, then `.to(device)`; the four initial-noise draws of one
cascade happen in the order surfPos, surfZ, edgePos, edgeZV (sample.py:126,189,208,267; the DDPM step noise in between
comes from diffusers on the CUDA generator and does not touch this stream).  brepgen_b200/sampler.py draws the same four
tensors from `torch.Generator().manual_seed(seed)`; tests/test_host_logic.py checks that this reproduces the reference
function under `torch.manual_seed(seed)` bit for bit.
"""
import os
import textwrap
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SEED, B, S0, S, E = 1234, 2, 3, 6, 3
SHAPES = {"surfPos": (B, S0, 6), "surfZ": (B, S, 48), "edgePos": (B, S, E, 6), "edgeZV": (B, S, E, 18)}


def main():
    lines = open(os.path.join(os.environ.get("BREPGEN_REFERENCE", "/root/reference"), "utils.py")).read().splitlines()[60 - 1:97]
    ns = dict(torch=torch, Union=Union, Tuple=Tuple, List=List, Optional=Optional)
    exec(textwrap.dedent("\n".join(lines)), ns)
    torch.manual_seed(SEED)
    out = {k: ns["randn_tensor"](s).numpy() for k, s in SHAPES.items()}
    assert all(v.dtype == np.float32 for v in out.values())
    path = os.path.join(ROOT, "tests", "golden", "randn_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
