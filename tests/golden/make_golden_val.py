"""Golden vectors for the forward-only VALIDATION of the four LDM trainers from the reference's OWN statements.

    python tests/golden/make_golden_val.py        # writes tests/golden/val_golden.npz   (build container only)

trainer.py cannot be imported (wandb, diffusers), but the bodies of its four `test_val()` loops --
trainer.py:395-403, :579-596, :774-791, :997-1019: frozen-encoder latent pass, fixed-timestep noising, one forward, masked
MSE -- are plain torch.  This script reads those lines from the reference file at generation time, dedents them and exec()s
them VERBATIM in a namespace where `self.model` is the oracle denoiser (oracle/denoisers.py, itself pinned to the reference's
classes) over synthetic weights, `self.surf_vae` / `self.edge_vae` are the oracle encoders, `self.noise_scheduler` the
oracle DDPM scheduler (pinned to diffusers' known answers) and `self.device` the CPU.  The random draws come from
torch.manual_seed(seed) right before each block.  Nothing of the reference is copied into the repository: the committed
.npz holds the inputs and the resulting loss sums only.  tests/test_val_golden.py replays the same seeds through
brepgen_b200/validation.py (CPU: with the same oracle callables, tight; GPU: with the product models / encoders /
scheduler, 1e-3)."""
import os
import sys
import textwrap
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from brepgen_b200.spec import denoiser_spec, edge_encoder_spec, surf_encoder_spec      # noqa: E402
from brepgen_b200.synth import synth_state_dict                                        # noqa: E402
from oracle import denoisers as O                                                      # noqa: E402
from oracle import vae as V                                                            # noqa: E402
from oracle.schedulers import DDPMOracle                                               # noqa: E402

REF = os.path.join(os.environ.get("BREPGEN_REFERENCE", "/root/reference"), "trainer.py")
BLOCKS = {"surfpos": (395, 403), "surfz": (579, 596), "edgepos": (774, 791), "edgez": (997, 1019)}
SEEDS = {"surfpos": 101, "surfz": 102, "edgepos": 103, "edgez": 104}
B, S, E = 2, 4, 3
Z_SCALED = 1.0
WSEED = {"surfpos": 31, "surfz": 32, "edgepos": 33, "edgez": 34, "surf_enc": 7, "edge_enc": 8}


def inputs():
    g = torch.Generator().manual_seed(77)
    r = lambda *s: torch.rand(*s, generator=g) * 2 - 1
    surf_mask = torch.tensor([[False, False, False, True], [False, False, True, True]])
    edge_mask = torch.rand(B, S, E, generator=g) < 0.3
    edge_mask = edge_mask | surf_mask.unsqueeze(-1)
    edge_mask[:, :, 0] = surf_mask          # first edge of every valid face is valid
    return dict(surfPos=r(B, S, 6), surfPnt=r(B, S, 32, 32, 3), edgePos=r(B, S, E, 6), edgePnt=r(B, S, E, 32, 3),
                vertPos=r(B, S, E, 6), surf_mask=surf_mask, edge_mask=edge_mask)


def state_dicts():
    return {"surfpos": synth_state_dict(denoiser_spec("surfpos", False), seed=WSEED["surfpos"]),
            "surfz": synth_state_dict(denoiser_spec("surfz", False), seed=WSEED["surfz"]),
            "edgepos": synth_state_dict(denoiser_spec("edgepos", False), seed=WSEED["edgepos"]),
            "edgez": synth_state_dict(denoiser_spec("edgez", False), seed=WSEED["edgez"]),
            "surf_enc": synth_state_dict(surf_encoder_spec(), seed=WSEED["surf_enc"]),
            "edge_enc": synth_state_dict(edge_encoder_spec(), seed=WSEED["edge_enc"])}


def oracle_callables(sd):
    models = {"surfpos": lambda x, t, lab: O.surfpos_forward(sd["surfpos"], x, t, lab),
              "surfz": lambda z, t, pos, m, lab: O.surfz_forward(sd["surfz"], z, t, pos, m, lab),
              "edgepos": lambda e, t, pos, z, m, lab: O.edgepos_forward(sd["edgepos"], e, t, pos, z, m, lab),
              "edgez": lambda e, t, ep, pos, z, m, lab: O.edgez_forward(sd["edgez"], e, t, ep, pos, z, m, lab)}
    return models, (lambda x: V.surf_encode(sd["surf_enc"], x)), (lambda x: V.edge_encode(sd["edge_enc"], x))


CF_LABEL = torch.tensor([[6], [3]])      # (B, 1) int64 class labels of the classifier-free case ('chair', 'bench')


def state_dicts_cf():
    """the classifier-free variants of the four denoisers (class embedding table); encoders as in state_dicts()"""
    sd = state_dicts()
    for i, kind in enumerate(("surfpos", "surfz", "edgepos", "edgez")):
        sd[kind] = synth_state_dict(denoiser_spec(kind, True), seed=60 + i)
    return sd


def main():
    src = open(REF).read().splitlines()
    inp = inputs()
    sched = DDPMOracle()
    sched.config = SimpleNamespace(num_train_timesteps=1000)
    out = {k: v.numpy() for k, v in inp.items()}
    for tag, sd, label in (("", state_dicts(), None), ("_cf", state_dicts_cf(), CF_LABEL)):
        models, surf_vae, edge_vae = oracle_callables(sd)
        for name, (a, b) in BLOCKS.items():
            body = textwrap.dedent("\n".join(src[a - 1:b]))
            nsteps = 5 if name in ("surfpos", "surfz") else 3
            ns = dict(torch=torch, nn=nn, mse_loss=nn.MSELoss(reduction="none"), total_loss=[0] * nsteps, total_count=0,
                      bsz=B, class_label=None if label is None else label.clone(),
                      self=SimpleNamespace(model=models[name], surf_vae=surf_vae, edge_vae=edge_vae, noise_scheduler=sched,
                                           device="cpu", z_scaled=Z_SCALED, max_edge=E),
                      **{k: v.clone() for k, v in inp.items()})
            torch.manual_seed(SEEDS[name])
            exec(compile(body, f"trainer.py:{a}-{b}", "exec"), ns)
            out[f"loss_{name}{tag}"] = np.asarray(ns["total_loss"], dtype=np.float64)
            print(name + tag, ns["total_loss"])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "val_golden.npz"), **out)


if __name__ == "__main__":
    main()
