"""Golden vectors for the CASCADE DRIVER (SURVEY.md section 8 row 1) from the reference's OWN statements.

    python tests/golden/make_golden_driver.py       # writes tests/golden/driver_golden.npz   (build container only)

sample.py cannot be imported or run (OpenCASCADE import, checkpoints, hard-coded .cuda()), but the body of
its sampling block -- sample.py:122-299: the six step loops, classifier-free batching and combine, the late increase, both
de-duplications, the zeroing of removed edges and the decoder input preparation -- is plain torch / numpy.  This script
reads those lines from the reference file at generation time, dedents them and exec()s them VERBATIM in a namespace where
  * the four networks are cheap stand-ins with the reference's forward signatures (below; every argument influences the
    output, so a swapped or missing argument shows),
  * the two schedulers are the oracle's (oracle/schedulers.py) behind the diffusers interface, the DDPM step noise drawn
    from a seeded generator,
  * randn_tensor draws the initial noise from a second seeded generator, the VAEs are stand-in upsamplers, tqdm is the
    identity and Tensor.cuda is patched to the identity.
Nothing of the reference is copied into the repository: the committed .npz holds the outputs only.  tests/
test_oracle_golden.py replays the same generators through oracle/cascade.py:run_cascade with the same stand-ins and
requires identical masks and matching tensors, which pins the restated driver (and with it brepgen_b200/sampler.py,
which tests/test_gpu_cascade.py compares with the oracle on the GPU) to the reference's control flow.
"""
import os
import sys
import textwrap
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = os.path.join(os.environ.get("BREPGEN_REFERENCE", "/root/reference"), "sample.py")
CASES = {  # name: (use_cf, batch, num_surfaces (before the late increase), num_edges, seed)
    "abc_like": (False, 2, 3, 3, 11),
    "furniture_like": (True, 2, 5, 4, 12),
}
W = 0.6
LABEL = 6      # 'chair'


# ------------------------------------------------------------------ stand-in networks (reference forward signatures)
def _temb(t):
    return torch.cos(t.float().reshape(-1, 1, 1) / 1000.0 * 3.0)            # (1,1,1) or (B,1,1)


def _lab(label, B):
    return 0.0 if label is None else (label.float().reshape(B, 1, 1) - 3.0) * 0.01


def _masked_mean(x, mask):                                                   # x (B,S,C), mask (B,S) True = padded
    keep = (~mask).float().unsqueeze(-1)
    return (x * keep).sum(1, keepdim=True) / keep.sum(1, keepdim=True).clamp_min(1.0)


def surfpos_net(surfPos, timesteps, class_label, is_train=False):
    B = surfPos.shape[0]
    return 0.5 * torch.tanh(0.7 * surfPos) * _temb(timesteps) + 0.1 * surfPos.roll(1, 1) + 0.05 * surfPos.mean(1, keepdim=True) \
        + _lab(class_label, B)


def surfz_net(surfZ, timesteps, surfPos, surf_mask, class_label, is_train=False):
    B = surfZ.shape[0]
    ctx = _masked_mean(surfZ, surf_mask) * 0.2 + _masked_mean(surfPos, surf_mask).mean(-1, keepdim=True) * 0.1
    return 0.6 * torch.tanh(surfZ) * _temb(timesteps) + ctx + 0.03 * surfPos.repeat(1, 1, 8) + _lab(class_label, B)


def edgepos_net(edgePos, timesteps, surfPos, surfZ, mask, class_label, is_train=False):
    B, S, E, _ = edgePos.shape
    face = (surfPos * 0.1 + surfZ[..., :6] * 0.05).unsqueeze(2)              # (B,S,1,6)
    keep = (~mask).float().reshape(B, S, 1, 1)
    ctx = (edgePos * keep).sum((1, 2), keepdim=True) / (keep.sum((1, 2), keepdim=True) * E).clamp_min(1.0)
    return 0.5 * torch.tanh(0.8 * edgePos) * _temb(timesteps).unsqueeze(-1) + face + 0.2 * ctx + 0.05 * edgePos.roll(1, 2) \
        + (_lab(class_label, B).unsqueeze(-1) if class_label is not None else 0.0)


def edgez_net(edge, timesteps, edgePos, surfPos, surfZ, mask, class_label, is_train=False):
    B, S, E, _ = edge.shape
    keep = (~mask).float().unsqueeze(-1)                                     # (B,S,E,1), per-edge mask
    ctx = (edge * keep).sum((1, 2), keepdim=True) / keep.sum((1, 2), keepdim=True).clamp_min(1.0)
    cond = edgePos.repeat(1, 1, 1, 3) * 0.05 + (surfPos * 0.02).repeat(1, 1, 3).unsqueeze(2) + surfZ[..., :18].unsqueeze(2) * 0.03
    return 0.55 * torch.tanh(edge) * _temb(timesteps).unsqueeze(-1) + 0.15 * ctx + cond \
        + (_lab(class_label, B).unsqueeze(-1) if class_label is not None else 0.0)


STANDINS = {"surfpos": surfpos_net, "surfz": surfz_net, "edgepos": edgepos_net, "edgez": edgez_net}


def surf_vae(z):          # (N,3,4,4) -> (N,3,32,32)
    return torch.tanh(z).repeat_interleave(8, -1).repeat_interleave(8, -2) * 0.5 + 0.01 * z.mean((1, 2, 3), keepdim=True)


def edge_vae(z):          # (N,3,4) -> (N,3,32)
    return torch.tanh(z).repeat_interleave(8, -1) * 0.5 + 0.02 * z.sum((1, 2), keepdim=True)


# ------------------------------------------------------------------ noise sources shared by the generator and the test
class NoiseSource:
    def __init__(self, seed):
        self.g_init = torch.Generator().manual_seed(seed)
        self.g_step = torch.Generator().manual_seed(seed + 1000)

    def init(self, shape):
        return torch.randn(tuple(shape), generator=self.g_init)

    def step(self, shape):
        return torch.randn(tuple(shape), generator=self.g_step)


class _DiffusersFacade:
    """the oracle scheduler behind the part of the diffusers interface sample.py uses"""

    def __init__(self, oracle, noise=None):
        self.o, self.noise = oracle, noise

    def set_timesteps(self, n):
        self.o.set_timesteps(n)

    @property
    def timesteps(self):
        return self.o.timesteps

    def step(self, model_output, timestep, sample):
        t = int(timestep)
        if self.noise is None:
            return SimpleNamespace(prev_sample=self.o.step(model_output, t, sample))
        nz = self.noise.step(sample.shape) if t > 0 else None
        return SimpleNamespace(prev_sample=self.o.step(model_output, t, sample, nz))


def reference_driver(use_cf, B, S0, E, seed):
    from oracle.schedulers import DDPMOracle, PNDMOracle
    lines = open(REF).read().splitlines()[122 - 1:299]
    code = textwrap.dedent("\n".join(lines))
    src = NoiseSource(seed)
    label = torch.LongTensor([LABEL] * B + [0] * B).reshape(-1, 1) if use_cf else None
    ns = dict(torch=torch, np=np, tqdm=lambda it: it, device=torch.device("cpu"),
              randn_tensor=lambda shape, *a, **k: src.init(shape),
              batch_size=B, num_surfaces=S0, num_edges=E, bbox_threshold=0.08, eval_args={"use_cf": use_cf},
              class_label=label, w=W,
              surfPos_model=surfpos_net, surfZ_model=surfz_net, edgePos_model=edgepos_net, edgeZ_model=edgez_net,
              pndm_scheduler=_DiffusersFacade(PNDMOracle()),
              ddpm_scheduler=_DiffusersFacade(DDPMOracle(clip_sample=True, clip_sample_range=3.0), src),
              surf_vae=surf_vae, edge_vae=edge_vae)
    with torch.no_grad():
        exec(code, ns)
    t = lambda v: v.numpy() if torch.is_tensor(v) else np.asarray(v)
    return {"surfPos": t(ns["surfPos"]), "surfMask": t(ns["surfMask"]), "surfZ": t(ns["surfZ"]), "edgePos": t(ns["edge_pos"]),
            "edgeM": t(ns["edge_mask"]), "edge_z": t(ns["edge_z"]), "edgeV": t(ns["edgeV"]), "surf_ncs": t(ns["surf_ncs"]),
            "edge_ncs": t(ns["edge_ncs"])}


def main():
    torch.Tensor.cuda = lambda self, *a, **k: self
    out = {}
    for name, (cf, B, S0, E, seed) in CASES.items():
        res = reference_driver(cf, B, S0, E, seed)
        for k, v in res.items():
            out[f"{name}|{k}"] = v
        print(name, {k: v.shape for k, v in res.items()}, "valid faces", (~res["surfMask"]).sum(1).tolist(),
              "masked edges", int(res["edgeM"].sum()))
    path = os.path.join(ROOT, "tests", "golden", "driver_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
