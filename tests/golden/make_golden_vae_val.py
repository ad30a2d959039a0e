"""Golden vectors for the two VAE trainers' validation and KL terms from the reference's OWN statements.

    python tests/golden/make_golden_vae_val.py        # writes tests/golden/vae_val_golden.npz   (build container only)

trainer.py cannot be imported (wandb, diffusers), but the statements this file pins are plain torch around
`self.model.encode(x).latent_dist` / `self.model.decode(z).sample`:
    SurfVAETrainer.test_val loop body   trainer.py:116-124      EdgeVAETrainer.test_val loop body   trainer.py:246-254
    SurfVAETrainer KL term              trainer.py:84           EdgeVAETrainer KL term (written out) trainer.py:211-214
This script reads those lines from the reference file at generation time, dedents them and exec()s them VERBATIM on the
CPU, the loop body first and the KL statement after it in the same namespace (so it reads the loop's `posterior`).
`self.model` is `OracleAutoencoder`: the oracle encoder's moments (oracle/vae_posterior.py surf_moments / edge_moments)
wrapped in the oracle's restatement of diffusers' DiagonalGaussianDistribution, and the oracle decoders, over synthetic
full-auto-encoder weights.  The posterior noise comes from torch.manual_seed(seed) right before each block.  Nothing of the
reference is copied into the repository: the committed .npz holds the inputs, the moments, z, the loss sums and the KL
values only.  tests/test_vae_posterior.py (CPU: with this stand-in, tight) and tests/test_gpu_vae_posterior.py (GPU: with
the drop-in AutoencoderKL / AutoencoderKL1D, 1e-3) replay the same seeds through brepgen_b200/validation.py."""
import os
import sys
import textwrap
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from brepgen_b200.spec import edge_decoder_spec, edge_encoder_spec, surf_decoder_spec, surf_encoder_spec   # noqa: E402
from brepgen_b200.synth import synth_state_dict                                                          # noqa: E402
from oracle import vae as V                                                                              # noqa: E402
from oracle import vae_posterior as VP                                                                    # noqa: E402

REF = os.path.join(os.environ.get("BREPGEN_REFERENCE", "/root/reference"), "trainer.py")
VAL_BLOCKS = {"surf": (116, 124), "edge": (246, 254)}
KL_BLOCKS = {"surf": (84, 84), "edge": (211, 214)}
SEEDS = {"surf": 201, "edge": 202}
WSEED = {"surf": 41, "edge": 42}
N_SURF, N_EDGE = 3, 5


def full_state_dict(kind):
    """synthetic weights of the whole auto-encoder, the layout of the reference's surfvae / edgevae checkpoints"""
    if kind == "surf":
        return {**synth_state_dict(surf_encoder_spec(), WSEED[kind]), **synth_state_dict(surf_decoder_spec(), WSEED[kind])}
    return {**synth_state_dict(edge_encoder_spec(), WSEED[kind]), **synth_state_dict(edge_decoder_spec(), WSEED[kind])}


class OracleAutoencoder:
    """stand-in for the trainers' `self.model`: encode(x).latent_dist / decode(z).sample over the CPU oracle"""

    def __init__(self, sd, two_d: bool):
        self.sd, self.two_d = sd, two_d

    def encode(self, x):
        moments = (VP.surf_moments if self.two_d else VP.edge_moments)(self.sd, x)
        return SimpleNamespace(latent_dist=VP.DiagonalGaussianDistribution(moments))

    def decode(self, z):
        return SimpleNamespace(sample=(V.surf_decode if self.two_d else V.edge_decode)(self.sd, z))


def inputs():
    g = torch.Generator().manual_seed(78)
    return dict(surf_uv=torch.rand(N_SURF, 32, 32, 3, generator=g) * 2 - 1, edge_u=torch.rand(N_EDGE, 32, 3, generator=g) * 2 - 1)


def main():
    src = open(REF).read().splitlines()
    block = lambda a, b: textwrap.dedent("\n".join(src[a - 1:b]))
    inp = inputs()
    out = {k: v.numpy() for k, v in inp.items()}
    for kind, var in (("surf", "surf_uv"), ("edge", "edge_u")):
        model = OracleAutoencoder(full_state_dict(kind), kind == "surf")
        ns = dict(torch=torch, nn=nn, mse_loss=nn.MSELoss(reduction="none"), total_loss=0, total_count=0,
                  self=SimpleNamespace(model=model, device="cpu"), **{var: inp[var].clone()})
        torch.manual_seed(SEEDS[kind])
        with torch.no_grad():
            a, b = VAL_BLOCKS[kind]
            exec(compile(block(a, b), f"trainer.py:{a}-{b}", "exec"), ns)
            a, b = KL_BLOCKS[kind]
            exec(compile(block(a, b), f"trainer.py:{a}-{b}", "exec"), ns)
        out[f"loss_{kind}"] = np.float64(ns["total_loss"])
        out[f"count_{kind}"] = np.int64(ns["total_count"])
        out[f"kl_{kind}"] = ns["kl_loss"].double().numpy()
        out[f"moments_{kind}"] = ns["posterior"].parameters.numpy()
        out[f"z_{kind}"] = ns["z"].numpy()
        print(kind, "loss sum", ns["total_loss"], "count", ns["total_count"], "kl", float(ns["kl_loss"]))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "vae_val_golden.npz"), **out)


if __name__ == "__main__":
    main()
