"""Generate golden vectors for the two de-duplication steps from the reference's OWN statements (build container only).

    python tests/golden/make_golden_dedup.py        # writes tests/golden/dedup_golden.npz

sample.py cannot be imported (OpenCASCADE, hard-coded .cuda()), but its de-duplication code is plain
numpy / torch: this script reads the statements at sample.py:159-183 (surfaces) and :242-261 (edges) from the reference
file at generation time, dedents them and exec()s them verbatim on seeded inputs, with `Tensor.cuda` patched to the
identity.  Nothing of the reference is copied into the repository; the committed .npz holds inputs and outputs only.
oracle/cascade.py (dedup_surfaces_np / dedup_edges_np) is then checked against these vectors
(tests/test_oracle_golden.py), and the CUDA kernels against the oracle (tests/test_gpu_cascade.py, bit-exact).
"""
import os
import textwrap

import numpy as np
import torch

REF = os.path.join(os.environ.get("BREPGEN_REFERENCE", "/root/reference"), "sample.py")
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
THR = 0.08     # bbox_threshold of every mode in eval_config.yaml


def _snippet(lo, hi):
    lines = open(REF).read().splitlines()[lo - 1:hi]
    return textwrap.dedent("\n".join(lines))


def boxes(g, B, S, dup=0.4, jitter=0.03):
    """(B,S,6) boxes in [-3,3] with near-duplicates (some with swapped corners), like the cascade produces"""
    x = (torch.rand(B, S, 6, generator=g) * 6 - 3)
    for b in range(B):
        for s in range(1, S):
            u = float(torch.rand((), generator=g))
            if u < dup:
                src = int(torch.randint(0, s, (), generator=g))
                p = x[b, src] + (torch.rand(6, generator=g) * 2 - 1) * jitter * (3.0 if u < dup / 4 else 1.0)
                if u < dup / 2:
                    p = torch.cat([p[3:], p[:3]])
                x[b, s] = p
    return x


def ref_surfaces(surfPos, num_surfaces):
    ns = dict(np=np, torch=torch, surfPos=surfPos.clone(), batch_size=surfPos.shape[0], num_surfaces=num_surfaces,
              bbox_threshold=THR)
    exec(_snippet(159, 183), ns)
    return ns["surfPos"], ns["surfMask"]


def ref_edges(edgePos, surfMask, num_edges):
    ns = dict(np=np, torch=torch, edgePos=edgePos.clone(), surfMask=surfMask.clone(), batch_size=edgePos.shape[0],
              num_edges=num_edges, bbox_threshold=THR)
    exec(_snippet(242, 261), ns)
    return ns["edgeM"]


def main():
    torch.Tensor.cuda = lambda self, *a, **k: self          # the reference moves results to the GPU; stay on the host
    out = {}
    for i, (B, S, E, seed) in enumerate([(2, 8, 6, 0), (3, 30, 20, 1), (2, 100, 40, 2), (1, 1, 1, 3), (4, 50, 30, 4)]):
        g = torch.Generator().manual_seed(seed)
        sp = boxes(g, B, S)
        pos, mask = ref_surfaces(sp, S)
        ep = boxes(g, B * S, E, dup=0.5).reshape(B, S, E, 6)
        em = ref_edges(ep, mask, E)
        out[f"c{i}_surfPos_in"] = sp.numpy()
        out[f"c{i}_surfPos_out"] = pos.numpy().astype(np.float32)
        out[f"c{i}_surfMask"] = mask.numpy()
        out[f"c{i}_edgePos_in"] = ep.numpy()
        out[f"c{i}_edgeM"] = em.numpy()
        print(f"case {i}: B={B} S={S} E={E} valid faces {(~mask).sum(1).tolist()} masked edges {int(em.sum())}/{em.numel()}")
    path = os.path.join(ROOT, "tests", "golden", "dedup_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
