"""Golden vectors for the slot fill of B-rep variations from the reference's OWN pad_repeat (build container only).

    python tests/golden/make_golden_fill.py          # writes tests/golden/fill_golden.npz

utils.py cannot be imported (OpenCASCADE / chamferdist at module import), so the text of pad_repeat (utils.py:100-106,
the layout the trainers give face and edge sequences, dataset.py:262-270 and :415-421) is cut out of the file with
`ast` and exec()'d VERBATIM.  It is applied to n = 1..S valid tokens (their positions 0..n-1) for S in SLOTS; only the
outputs are stored: key "S{S}" holds an (S, S) int64 array whose row n - 1 is pad_repeat(arange(n), S).  Nothing from the
reference is copied into the repo.
"""
from __future__ import annotations

import ast
import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = os.environ.get("BREPGEN_REFERENCE", "/root/reference")
SLOTS = (30, 40, 50, 100)


def reference_pad_repeat():
    src = open(os.path.join(REF, "utils.py")).read()
    ns = {"np": np, "math": math}
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name == "pad_repeat":
            exec(compile(ast.get_source_segment(src, node), "utils.py:pad_repeat", "exec"), ns)
    return ns["pad_repeat"]


def main():
    pad_repeat = reference_pad_repeat()
    out = {f"S{S}": np.stack([pad_repeat(np.arange(n), S) for n in range(1, S + 1)]).astype(np.int64) for S in SLOTS}
    path = os.path.join(ROOT, "tests", "golden", "fill_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
