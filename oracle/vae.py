"""ORACLE (test infrastructure): CPU fp32 restatement of the two VAE decoders.

2-D (surface) decoder leaves PINNED by diffusers' own known answers (tests/test_oracle_vae_kat.py): `_resnet2d` (with and
without conv_shortcut), `_attn2d` and `_upsample2d` reproduce the expected output slices of diffusers'
tests/models/test_layers_utils.py (ResnetBlock2DTests.test_resnet_default / test_restnet_with_use_in_shortcut,
AttentionBlockTests.test_attention_block_default, Upsample2DBlockTests.test_upsample_default / test_upsample_with_conv) to 4
decimals, and the block wiring (resnet -> upsample; resnet -> attention -> resnet) those of test_unet_2d_blocks.py
(UpDecoderBlock2DTests / UNetMidBlock2DTests); the encoder's stride-2 convolution and resnet -> downsample wiring those of
Downsample2DBlockTests.test_downsample_with_conv / DownEncoderBlock2DTests (with diffusers' default symmetric padding; the
asymmetric padding=0 variant the VAE uses differs by the one F.pad line).  1-D leaves (ResConvBlock, SelfAttention1d, Upsample1d / Downsample1d; diffusers has no known-answer test for them)
remain PARITY UNPINNED.  The arithmetic lives in diffusers==0.27 (requirements.txt:5 of the reference), which is absent from
the reference and from this environment: `Decoder`, `UNetMidBlock2D`, `UpDecoderBlock2D`, `ResnetBlock2D`, `Attention`,
`Upsample2D` (surface) and `ResConvBlock`, `SelfAttention1d`, `Upsample1d` (edge).  This file restates their published
structure (SURVEY.md Appendix A.1 / A.2) around the reference's own wrappers
    AutoencoderKLFastDecode.forward      network.py:1013-1040   (cfg sample.py:72-82)
    AutoencoderKL1DFastDecode.forward    network.py:846-858, Decoder1D :188-299, UNetMidBlock1D :51-83, UpBlock1D :30-48
                                         (cfg sample.py:86-97)
and is anchored on: input/output shapes consumed at sample.py:289-294, the state-dict key sets and the parameter counts
49 485 583 / 39 124 751 (SURVEY A.5(6); tests/test_oracle_vae.py), partition-of-unity of the cubic resampler.

Partly pinned since: the EDGE decoder's wrapper -- everything the reference itself defines (AutoencoderKL1DFastDecode,
Decoder1D, UNetMidBlock1D, UpBlock1D: block order and counts, channel wiring, head count, norms, key names) -- is checked
against outputs of those classes (tests/golden/vae1d_golden.npz, made by tests/golden/make_golden_vae1d.py from the real
network.py over module forms of the diffusers leaves), and the EDGE encoder's wrapper (AutoencoderKL1DFastEncode,
Encoder1D) the same way.  The arithmetic inside the 1-D diffusers leaves remains unpinned.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]


def _gn(x, sd, name, groups, eps):
    return F.group_norm(x, groups, sd[name + ".weight"], sd[name + ".bias"], eps)


# ------------------------------------------------------------------------------------------------ surface (2-D)
def _resnet2d(sd: SD, name: str, x, temb_add=None):
    """diffusers ResnetBlock2D (groups 32, eps 1e-6, swish).  `temb_add` (the projected time embedding, (N,C,1,1)) is None in
    the VAE (temb_channels=None); it exists so that the block can be checked against diffusers' own known answers, which use
    one (tests/test_oracle_vae_kat.py)."""
    h = F.conv2d(F.silu(_gn(x, sd, name + ".norm1", 32, 1e-6)), sd[name + ".conv1.weight"], sd[name + ".conv1.bias"], padding=1)
    if temb_add is not None:
        h = h + temb_add
    h = F.conv2d(F.silu(_gn(h, sd, name + ".norm2", 32, 1e-6)), sd[name + ".conv2.weight"], sd[name + ".conv2.bias"], padding=1)
    if name + ".conv_shortcut.weight" in sd:
        x = F.conv2d(x, sd[name + ".conv_shortcut.weight"], sd[name + ".conv_shortcut.bias"])
    return x + h


def _attn2d(sd: SD, name: str, x, n_head: int = 1):
    """diffusers mid-block attention (GroupNorm 32 / 1e-6, softmax(q k^T / sqrt(dim_head)), residual).  The VAE uses ONE head of
    dim_head = C (attention_head_dim = C); n_head exists for diffusers' known-answer test, which uses heads of dimension 1."""
    N, C, H, W = x.shape
    h = _gn(x, sd, name + ".group_norm", 32, 1e-6).view(N, C, H * W).transpose(1, 2)          # (N, HW, C)
    dh = C // n_head
    heads = lambda t: t.view(N, H * W, n_head, dh).transpose(1, 2)                            # (N, heads, HW, dh)
    q = heads(h @ sd[name + ".to_q.weight"].t() + sd[name + ".to_q.bias"])
    k = heads(h @ sd[name + ".to_k.weight"].t() + sd[name + ".to_k.bias"])
    v = heads(h @ sd[name + ".to_v.weight"].t() + sd[name + ".to_v.bias"])
    a = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh), dim=-1) @ v
    a = a.transpose(1, 2).reshape(N, H * W, C)
    a = a @ sd[name + ".to_out.0.weight"].t() + sd[name + ".to_out.0.bias"]
    return x + a.transpose(1, 2).reshape(N, C, H, W)


def _downsample2d(sd: SD, name: str, x, padding: int = 0):
    """diffusers Downsample2D(use_conv=True): 3x3 convolution with stride 2.  The VAE encoder builds it with padding=0, for
    which diffusers pads the right / bottom edge by one zero pixel first; padding=1 (diffusers' default, symmetric) exists
    for diffusers' own known-answer tests."""
    if padding == 0:
        x = F.pad(x, (0, 1, 0, 1), mode="constant", value=0)
    return F.conv2d(x, sd[name + ".conv.weight"], sd[name + ".conv.bias"], stride=2, padding=padding)


def _upsample2d(sd: SD, name: str, x):
    """diffusers Upsample2D(use_conv=True): nearest 2x, then conv 3x3 pad 1"""
    x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    return F.conv2d(x, sd[name + ".conv.weight"], sd[name + ".conv.bias"], padding=1)


def surf_decode(sd: SD, z: torch.Tensor) -> torch.Tensor:
    """z (N,3,h,w) -> (N,3,8h,8w); the cascade uses h = w = 4 (sample.py:289)"""
    d = "decoder"
    x = F.conv2d(z, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
    x = F.conv2d(x, sd[f"{d}.conv_in.weight"], sd[f"{d}.conv_in.bias"], padding=1)
    x = _resnet2d(sd, f"{d}.mid_block.resnets.0", x)
    x = _attn2d(sd, f"{d}.mid_block.attentions.0", x)
    x = _resnet2d(sd, f"{d}.mid_block.resnets.1", x)
    for i in range(4):
        for j in range(3):
            x = _resnet2d(sd, f"{d}.up_blocks.{i}.resnets.{j}", x)
        if i < 3:
            x = _upsample2d(sd, f"{d}.up_blocks.{i}.upsamplers.0", x)
    x = F.silu(_gn(x, sd, f"{d}.conv_norm_out", 32, 1e-6))
    return F.conv2d(x, sd[f"{d}.conv_out.weight"], sd[f"{d}.conv_out.bias"], padding=1)


# ------------------------------------------------------------------------------------------------ edge (1-D)
def _resconv1d(sd: SD, name: str, x):
    res = F.conv1d(x, sd[name + ".conv_skip.weight"]) if name + ".conv_skip.weight" in sd else x
    h = F.conv1d(x, sd[name + ".conv_1.weight"], sd[name + ".conv_1.bias"], padding=2)
    h = F.gelu(_gn(h, sd, name + ".group_norm_1", 1, 1e-5))
    h = F.conv1d(h, sd[name + ".conv_2.weight"], sd[name + ".conv_2.bias"], padding=2)
    h = F.gelu(_gn(h, sd, name + ".group_norm_2", 1, 1e-5))
    return h + res


def _attn1d(sd: SD, name: str, x, n_head: int = 16):
    N, C, L = x.shape
    h = _gn(x, sd, name + ".group_norm", 1, 1e-5).transpose(1, 2)                             # (N, L, C)
    dh = C // n_head
    proj = lambda t, w: (t @ sd[f"{name}.{w}.weight"].t() + sd[f"{name}.{w}.bias"]).view(N, L, n_head, dh).transpose(1, 2)
    q, k, v = proj(h, "query"), proj(h, "key"), proj(h, "value")
    scale = 1.0 / math.sqrt(math.sqrt(dh))
    a = torch.softmax((q * scale) @ (k * scale).transpose(-1, -2), dim=-1) @ v
    a = a.transpose(1, 2).reshape(N, L, C)
    a = a @ sd[name + ".proj_attn.weight"].t() + sd[name + ".proj_attn.bias"]
    return x + a.transpose(1, 2)


def cubic_upsample1d(x, kernel):
    """diffusers Upsample1d('cubic'): reflect pad 2, depthwise conv_transpose1d(stride 2, padding 7): L -> 2L"""
    C = x.shape[1]
    x = F.pad(x, (2, 2), "reflect")
    w = x.new_zeros(C, C, kernel.shape[0])
    idx = torch.arange(C)
    w[idx, idx] = kernel.to(x)
    return F.conv_transpose1d(x, w, stride=2, padding=kernel.shape[0] * 2 // 2 - 1)


def edge_decode(sd: SD, z: torch.Tensor) -> torch.Tensor:
    """z (N,3,4) -> (N,3,32)"""
    d = "decoder"
    x = F.conv1d(z, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
    x = F.conv1d(x, sd[f"{d}.conv_in.weight"], sd[f"{d}.conv_in.bias"], padding=1)
    for i in range(6):
        x = _resconv1d(sd, f"{d}.mid_block.resnets.{i}", x)
        x = _attn1d(sd, f"{d}.mid_block.attentions.{i}", x)
    for i in range(3):
        for j in range(3):
            x = _resconv1d(sd, f"{d}.up_blocks.{i}.resnets.{j}", x)
        x = cubic_upsample1d(x, sd[f"{d}.up_blocks.{i}.up.kernel"])
    x = F.silu(_gn(x, sd, f"{d}.conv_norm_out", 32, 1e-6))
    return F.conv1d(x, sd[f"{d}.conv_out.weight"], sd[f"{d}.conv_out.bias"], padding=1)


# ------------------------------------------------------------------------------------------------ encoders (config 1)
# AutoencoderKLFastEncode.forward network.py:927-945 and AutoencoderKL1DFastEncode.forward :745-783 return
# DiagonalGaussianDistribution(quant_conv(encoder(x))).mode() = the first half of the channels (2-D leaves pinned by
# tests/test_oracle_vae_kat.py; 1-D leaves unpinned).
def surf_encode(sd: SD, x: torch.Tensor) -> torch.Tensor:
    """x (N,3,H,W), H and W divisible by 8 -> latent mode (N,3,H/8,W/8)"""
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
    moments = F.conv2d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])
    return moments[:, :3]


def cubic_downsample1d(x, kernel):
    """diffusers Downsample1d('cubic'): reflect pad 3, depthwise conv1d stride 2: L -> L/2"""
    C = x.shape[1]
    x = F.pad(x, (3, 3), "reflect")
    w = x.new_zeros(C, C, kernel.shape[0])
    idx = torch.arange(C)
    w[idx, idx] = kernel.to(x)
    return F.conv1d(x, w, stride=2)


def edge_encode(sd: SD, x: torch.Tensor) -> torch.Tensor:
    """x (N,3,32) -> latent mode (N,3,4)"""
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
    moments = F.conv1d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])
    return moments[:, :3]


surf_decode_any = surf_decode     # the restated decoder is size-agnostic (convolutions + nearest upsampling)
