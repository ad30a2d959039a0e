"""ORACLE (test infrastructure): CPU fp32 restatement of the full auto-encoders' posterior.

The VAE trainers (trainer.py:79-86, :116-124, :206-216, :246-254) use the whole posterior: moments = quant_conv(encoder(x))
wrapped in diffusers 0.27's DiagonalGaussianDistribution.  The encoder layers are those of oracle/vae.py (surf_encode /
edge_encode return the first half of these moments); diffusers publishes no known answer for DiagonalGaussianDistribution,
so the restatement below is PARITY UNPINNED at that boundary.  The trainers' own statements around it are pinned by
tests/golden/vae_val_golden.npz (tests/golden/make_golden_vae_val.py).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .vae import SD, _attn1d, _attn2d, _downsample2d, _gn, _resconv1d, _resnet2d, cubic_downsample1d


def surf_moments(sd: SD, x: torch.Tensor) -> torch.Tensor:
    """x (N,3,H,W) -> moments (N,6,H/8,W/8) = mean | logvar (surf_encode without the final [:, :3])"""
    e = "encoder"
    h = F.conv2d(x, sd[f"{e}.conv_in.weight"], sd[f"{e}.conv_in.bias"], padding=1)
    for i in range(4):
        for j in range(2):
            h = _resnet2d(sd, f"{e}.down_blocks.{i}.resnets.{j}", h)
        if i < 3:
            h = _downsample2d(sd, f"{e}.down_blocks.{i}.downsamplers.0", h, padding=0)
    h = _resnet2d(sd, f"{e}.mid_block.resnets.0", h)
    h = _attn2d(sd, f"{e}.mid_block.attentions.0", h)
    h = _resnet2d(sd, f"{e}.mid_block.resnets.1", h)
    h = F.silu(_gn(h, sd, f"{e}.conv_norm_out", 32, 1e-6))
    h = F.conv2d(h, sd[f"{e}.conv_out.weight"], sd[f"{e}.conv_out.bias"], padding=1)
    return F.conv2d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])


def edge_moments(sd: SD, x: torch.Tensor) -> torch.Tensor:
    """x (N,3,32) -> moments (N,6,4) = mean | logvar (edge_encode without the final [:, :3])"""
    e = "encoder"
    h = F.conv1d(x, sd[f"{e}.conv_in.weight"], sd[f"{e}.conv_in.bias"], padding=1)
    for i in range(3):
        h = cubic_downsample1d(h, sd[f"{e}.down_blocks.{i}.down.kernel"])
        for j in range(3):
            h = _resconv1d(sd, f"{e}.down_blocks.{i}.resnets.{j}", h)
    for i in range(6):
        h = _resconv1d(sd, f"{e}.mid_block.resnets.{i}", h)
        h = _attn1d(sd, f"{e}.mid_block.attentions.{i}", h)
    h = F.silu(_gn(h, sd, f"{e}.conv_norm_out", 32, 1e-6))
    h = F.conv1d(h, sd[f"{e}.conv_out.weight"], sd[f"{e}.conv_out.bias"], padding=1)
    return F.conv1d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])


class DiagonalGaussianDistribution:
    """diffusers 0.27 DiagonalGaussianDistribution (published structure): moments split in half along dim 1 into mean and
    logvar, logvar clamped to [-30, 20], std = exp(logvar / 2), var = exp(logvar); deterministic: std = var = 0.
    sample = mean + std * randn(mean.shape) (CPU generator); kl / nll sum over dims [1, 2, 3]."""

    def __init__(self, parameters: torch.Tensor, deterministic: bool = False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, generator=None, noise=None) -> torch.Tensor:
        """`noise` (optional): use it instead of a fresh draw (tests compare chains on the same noise)"""
        if noise is None:
            noise = torch.randn(self.mean.shape, generator=generator, dtype=self.parameters.dtype)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean

    def kl(self, other=None) -> torch.Tensor:
        if self.deterministic:
            return torch.Tensor([0.0])
        if other is None:
            return 0.5 * torch.sum(torch.pow(self.mean, 2) + self.var - 1.0 - self.logvar, dim=[1, 2, 3])
        return 0.5 * torch.sum(torch.pow(self.mean - other.mean, 2) / other.var + self.var / other.var - 1.0 - self.logvar
                               + other.logvar, dim=[1, 2, 3])

    def nll(self, sample: torch.Tensor, dims=(1, 2, 3)) -> torch.Tensor:
        if self.deterministic:
            return torch.Tensor([0.0])
        return 0.5 * torch.sum(math.log(2.0 * math.pi) + self.logvar + torch.pow(sample - self.mean, 2) / self.var,
                               dim=list(dims))
