"""Forward-only validation of the four latent-diffusion trainers -- the reference's `test_val()` loop bodies
(trainer.py:383-407 SurfPos, :570-603 SurfZ, :764-798 EdgePos, :987-1026 EdgeZ): frozen VAE encoders ->
latents, noise at the fixed timesteps {10, 50, 100[, 200, 500]} - 1, one denoiser forward per timestep, masked MSE of the
noise prediction summed over the batch (the trainer divides the accumulated sums by the number of samples seen).

Host glue only: `model`, `surf_vae`, `edge_vae` and `noise_scheduler` are the drop-in objects of brepgen_b200 (models.py,
vae.py, schedulers.py) -- or any callables with the reference's signatures -- and carry the CUDA work.  The random draws
follow the reference statement by statement (timesteps with torch.randint on the data's device, noise with torch.randn on
the CPU generator and then moved), so a seeded run reproduces the reference's numbers (tests/golden/val_golden.npz).
The two VAE trainers' `test_val()` loop bodies (trainer.py:116-124 surface, :246-254 edge: encode -> posterior sample ->
decode -> per-sample MSE) are `surfvae_val_losses` / `edgevae_val_losses`, and `vae_val_mse` is their loop
(tests/golden/vae_val_golden.npz).
The training step itself (autograd, AdamW, GradScaler; trainer.py:497-541 etc.) is out of scope: the product is
inference-only.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from .vae import encode_edge_latents, encode_surface_latents

SURF_STEPS = (10, 50, 100, 200, 500)      # trainer.py:395, :588
EDGE_STEPS = (10, 50, 100)                # trainer.py:783, :1011


def _draw(shape, bsz: int, step: int, device, rng_device=None):
    """the reference's two draws (trainer.py:397-398): timesteps on the data's device, noise on the CPU generator.
    rng_device="cpu" draws the (constant) timesteps on the CPU generator as well, which makes a seeded run independent of
    the device -- used to replay the CPU-generated golden vectors on the GPU."""
    timesteps = torch.randint(step - 1, step, (bsz,), device=rng_device or device).long().to(device)
    noise = torch.randn(shape).to(device)
    return timesteps, noise


def _mse_rows(pred: torch.Tensor, noise: torch.Tensor) -> float:
    """nn.MSELoss(reduction='none')(pred, noise).mean(-1).sum() over the selected token rows"""
    return float(((pred - noise) ** 2).mean(-1).sum().item())


def surfpos_val_losses(model, noise_scheduler, surfPos: torch.Tensor, class_label: Optional[torch.Tensor] = None,
                       steps: Sequence[int] = SURF_STEPS, rng_device=None) -> List[float]:
    """trainer.py:395-403: per timestep, sum over the batch of the per-sample mean squared error"""
    bsz, out = len(surfPos), []
    for step in steps:
        timesteps, noise = _draw(surfPos.shape, bsz, step, surfPos.device, rng_device)
        diffused = noise_scheduler.add_noise(surfPos, noise, timesteps)
        with torch.no_grad():
            pred = model(diffused, timesteps, class_label)
        out.append(float(((pred - noise) ** 2).mean((1, 2)).sum().item()))
    return out


def surfz_val_losses(model, surf_vae, noise_scheduler, surfPos, surfPnt, surf_mask, class_label=None, z_scaled: float = 1.0,
                     steps: Sequence[int] = SURF_STEPS, rng_device=None) -> List[float]:
    """trainer.py:579-596"""
    bsz, out = len(surfPos), []
    with torch.no_grad():
        tokens = encode_surface_latents(surf_vae, surfPnt, z_scaled)
    for step in steps:
        timesteps, noise = _draw(tokens.shape, bsz, step, tokens.device, rng_device)
        diffused = noise_scheduler.add_noise(tokens, noise, timesteps)
        with torch.no_grad():
            pred = model(diffused, timesteps, surfPos, surf_mask, class_label)
        out.append(_mse_rows(pred[~surf_mask], noise[~surf_mask]))
    return out


def edgepos_val_losses(model, surf_vae, noise_scheduler, edgePos, surfPnt, surfPos, surf_mask, class_label=None,
                       z_scaled: float = 1.0, steps: Sequence[int] = EDGE_STEPS, rng_device=None) -> List[float]:
    """trainer.py:774-791 (the mask is per FACE: all edges of a padded face are dropped)"""
    bsz, out = len(surfPos), []
    with torch.no_grad():
        surfZ = encode_surface_latents(surf_vae, surfPnt, z_scaled)
    for step in steps:
        timesteps, noise = _draw(edgePos.shape, bsz, step, edgePos.device, rng_device)
        diffused = noise_scheduler.add_noise(edgePos, noise, timesteps)
        with torch.no_grad():
            pred = model(diffused, timesteps, surfPos, surfZ, surf_mask, class_label)
        out.append(_mse_rows(pred[~surf_mask], noise[~surf_mask]))
    return out


def edgez_val_losses(model, surf_vae, edge_vae, noise_scheduler, edgePnt, edgePos, edge_mask, surfPnt, surfPos, vertPos,
                     class_label=None, z_scaled: float = 1.0, steps: Sequence[int] = EDGE_STEPS, rng_device=None) -> List[float]:
    """trainer.py:997-1019: joint 18-D token = 12-D edge latent + the two end points (mask per EDGE)"""
    bsz, out = len(surfPos), []
    with torch.no_grad():
        surfZ = encode_surface_latents(surf_vae, surfPnt, z_scaled)
        edgeZ = encode_edge_latents(edge_vae, edgePnt, z_scaled)
    joint_data = torch.concat([edgeZ, vertPos], -1)
    for step in steps:
        timesteps, noise = _draw(joint_data.shape, bsz, step, joint_data.device, rng_device)
        diffused = noise_scheduler.add_noise(joint_data, noise, timesteps)
        with torch.no_grad():
            pred = model(diffused, timesteps, edgePos, surfPos, surfZ, edge_mask, class_label)
        out.append(_mse_rows(pred[~edge_mask], noise[~edge_mask]))
    return out


def _vae_val_loss(model, x: torch.Tensor, rng_device=None) -> float:
    """encode -> posterior.sample() -> decode -> per-sample MSE summed over the batch.  The drop-in auto-encoders run it as
    one fused round trip (`reconstruct`); any other model with the reference's encode / decode surface runs the statements
    one by one.  rng_device="cpu" draws the posterior noise on the CPU generator (see _draw)."""
    generator = torch.default_generator if rng_device == "cpu" else None
    with torch.no_grad():
        if hasattr(model, "reconstruct"):
            return float(model.reconstruct(x, sample_posterior=True, generator=generator)[1].sum().item())
        posterior = model.encode(x).latent_dist
        z = posterior.sample(generator=generator)
        dec = model.decode(z).sample
        return float(((dec - x) ** 2).mean(tuple(range(1, x.dim()))).sum().item())


def surfvae_val_losses(model, surf_uv: torch.Tensor, rng_device=None) -> float:
    """SurfVAETrainer.test_val loop body (trainer.py:116-124): surf_uv (N, 32, 32, 3) as the dataloader yields it -> the
    sum over the batch of the per-sample reconstruction MSE, the posterior sampled as the reference samples it"""
    return _vae_val_loss(model, surf_uv.permute(0, 3, 1, 2), rng_device)


def edgevae_val_losses(model, edge_u: torch.Tensor, rng_device=None) -> float:
    """EdgeVAETrainer.test_val loop body (trainer.py:246-254): edge_u (N, 32, 3) -> summed per-sample MSE"""
    return _vae_val_loss(model, edge_u.permute(0, 2, 1), rng_device)


def vae_val_mse(model, batches, edge: bool = False, device=None, rng_device=None) -> float:
    """SurfVAETrainer / EdgeVAETrainer.test_val (trainer.py:106-129, :236-259): total_loss / total_count over the batches of
    a validation loader"""
    fn = edgevae_val_losses if edge else surfvae_val_losses
    total_loss, total_count = 0.0, 0
    for batch in batches:
        if device is not None:
            batch = batch.to(device)
        total_loss += fn(model, batch, rng_device)
        total_count += len(batch)
    return total_loss / total_count
