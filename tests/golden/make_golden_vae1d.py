"""Golden vectors for the EDGE decoder wrapper (SURVEY.md section 8 row 16) from the reference's OWN classes.

    python tests/golden/make_golden_vae1d.py        # writes tests/golden/vae1d_golden.npz   (build container only)

AutoencoderKL1DFastDecode, Decoder1D, UNetMidBlock1D and UpBlock1D are defined by the reference itself
(network.py:786-858, :188-299, :51-83, :30-48); only three leaf modules come from diffusers 0.27
(ResConvBlock, SelfAttention1d, Upsample1d -- absent here, no network).  This script imports the REAL network.py with those
three leaves replaced by the nn.Module forms below (written from the published diffusers 0.27 `unet_1d_blocks.py`
semantics, the same restatement oracle/vae.py uses in functional form), instantiates the reference's
AutoencoderKL1DFastDecode with the constructor arguments of sample.py:86-97, loads the synthetic state dict of
brepgen_b200.spec.edge_decoder_spec STRICTLY (so the key set and every shape are checked against the reference's module
tree) and stores its outputs.

What this pins: everything the reference owns -- block order and counts (6 x [ResConvBlock, SelfAttention1d] mid block,
3 up blocks of 3 ResConvBlocks + cubic upsampling), channel wiring 512 -> 512 -> 256 -> 128, head count 512 // 32,
post_quant_conv -> conv_in -> ... -> GroupNorm(32, eps 1e-6) -> SiLU -> conv_out, state-dict key names.
What it does NOT pin: the arithmetic inside the three diffusers leaves (still "parity unpinned", DESIGN.md section 2).
"""
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
CUBIC = [-0.01171875, -0.03515625, 0.11328125, 0.43359375, 0.43359375, 0.11328125, -0.03515625, -0.01171875]


class ResConvBlock(nn.Module):
    def __init__(self, in_channels, mid_channels, out_channels, is_last=False):
        super().__init__()
        self.is_last = is_last
        self.has_conv_skip = in_channels != out_channels
        if self.has_conv_skip:
            self.conv_skip = nn.Conv1d(in_channels, out_channels, 1, bias=False)
        self.conv_1 = nn.Conv1d(in_channels, mid_channels, 5, padding=2)
        self.group_norm_1 = nn.GroupNorm(1, mid_channels)
        self.gelu_1 = nn.GELU()
        self.conv_2 = nn.Conv1d(mid_channels, out_channels, 5, padding=2)
        if not self.is_last:
            self.group_norm_2 = nn.GroupNorm(1, out_channels)
            self.gelu_2 = nn.GELU()

    def forward(self, hidden_states):
        residual = self.conv_skip(hidden_states) if self.has_conv_skip else hidden_states
        hidden_states = self.gelu_1(self.group_norm_1(self.conv_1(hidden_states)))
        hidden_states = self.conv_2(hidden_states)
        if not self.is_last:
            hidden_states = self.gelu_2(self.group_norm_2(hidden_states))
        return hidden_states + residual


class SelfAttention1d(nn.Module):
    def __init__(self, in_channels, n_head=1, dropout_rate=0.0):
        super().__init__()
        self.channels = in_channels
        self.group_norm = nn.GroupNorm(1, num_channels=in_channels)
        self.num_heads = n_head
        self.query = nn.Linear(self.channels, self.channels)
        self.key = nn.Linear(self.channels, self.channels)
        self.value = nn.Linear(self.channels, self.channels)
        self.proj_attn = nn.Linear(self.channels, self.channels, bias=True)
        self.dropout = nn.Dropout(dropout_rate, inplace=True)

    def _heads(self, projection):
        n, l, _ = projection.shape
        return projection.view(n, l, self.num_heads, -1).permute(0, 2, 1, 3)

    def forward(self, hidden_states):
        residual = hidden_states
        hidden_states = self.group_norm(hidden_states).transpose(1, 2)
        q, k, v = self._heads(self.query(hidden_states)), self._heads(self.key(hidden_states)), self._heads(self.value(hidden_states))
        scale = 1 / math.sqrt(math.sqrt(k.shape[-1]))
        probs = torch.softmax(torch.matmul(q * scale, k.transpose(-1, -2) * scale), dim=-1)
        hidden_states = torch.matmul(probs, v).permute(0, 2, 1, 3).contiguous()
        hidden_states = hidden_states.view(hidden_states.shape[0], hidden_states.shape[1], self.channels)
        hidden_states = self.proj_attn(hidden_states).transpose(1, 2)
        return self.dropout(hidden_states) + residual


class Upsample1d(nn.Module):
    def __init__(self, kernel="linear", pad_mode="reflect"):
        super().__init__()
        assert kernel == "cubic"
        self.pad_mode = pad_mode
        kernel_1d = torch.tensor(CUBIC) * 2
        self.pad = kernel_1d.shape[0] // 2 - 1
        self.register_buffer("kernel", kernel_1d)

    def forward(self, hidden_states, temb=None):
        hidden_states = F.pad(hidden_states, ((self.pad + 1) // 2,) * 2, self.pad_mode)
        weight = hidden_states.new_zeros([hidden_states.shape[1], hidden_states.shape[1], self.kernel.shape[0]])
        idx = torch.arange(hidden_states.shape[1])
        weight[idx, idx] = self.kernel.to(weight)
        return F.conv_transpose1d(hidden_states, weight, stride=2, padding=self.pad * 2 + 1)


class Downsample1d(nn.Module):
    def __init__(self, kernel="linear", pad_mode="reflect"):
        super().__init__()
        assert kernel == "cubic"
        self.pad_mode = pad_mode
        kernel_1d = torch.tensor(CUBIC)
        self.pad = kernel_1d.shape[0] // 2 - 1
        self.register_buffer("kernel", kernel_1d)

    def forward(self, hidden_states):
        hidden_states = F.pad(hidden_states, (self.pad,) * 2, self.pad_mode)
        weight = hidden_states.new_zeros([hidden_states.shape[1], hidden_states.shape[1], self.kernel.shape[0]])
        idx = torch.arange(hidden_states.shape[1])
        weight[idx, idx] = self.kernel.to(weight)
        return F.conv1d(hidden_states, weight, stride=2)


class DownBlock1D(nn.Module):
    def __init__(self, out_channels, in_channels, mid_channels=None):
        super().__init__()
        mid_channels = out_channels if mid_channels is None else mid_channels
        self.down = Downsample1d("cubic")
        self.resnets = nn.ModuleList([ResConvBlock(in_channels, mid_channels, mid_channels),
                                      ResConvBlock(mid_channels, mid_channels, mid_channels),
                                      ResConvBlock(mid_channels, mid_channels, out_channels)])

    def forward(self, hidden_states, temb=None):
        hidden_states = self.down(hidden_states)
        for resnet in self.resnets:
            hidden_states = resnet(hidden_states)
        return hidden_states, (hidden_states,)


def get_down_block(down_block_type, num_layers, in_channels, out_channels, temb_channels, add_downsample):
    assert down_block_type == "DownBlock1D"
    return DownBlock1D(out_channels=out_channels, in_channels=in_channels)


class DiagonalGaussianDistribution:
    def __init__(self, parameters, deterministic=False):
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)

    def mode(self):
        return self.mean


class DecoderOutput:
    def __init__(self, sample):
        self.sample = sample


def load_reference_network_with_leaves():
    import make_golden as MG
    from oracle.reference_loader import _stub_diffusers
    _stub_diffusers()
    sys.modules["diffusers.models.unets.unet_1d_blocks"].__dict__.update(
        ResConvBlock=ResConvBlock, SelfAttention1d=SelfAttention1d, Upsample1d=Upsample1d, get_down_block=get_down_block)
    sys.modules["diffusers.models.autoencoders.vae"].__dict__.update(
        DecoderOutput=DecoderOutput, DiagonalGaussianDistribution=DiagonalGaussianDistribution)
    sys.modules["diffusers.utils"].__dict__.update(BaseOutput=object)
    sys.modules.pop("network", None)
    sys.path.insert(0, MG.REF)
    import network
    assert os.path.abspath(network.__file__).startswith(MG.REF)
    return network


def inputs(seed, n):
    return torch.randn(n, 3, 4, generator=torch.Generator().manual_seed(seed))


def enc_inputs(seed, n):
    return torch.rand(n, 3, 32, generator=torch.Generator().manual_seed(100 + seed)) * 2 - 1


def main():
    from brepgen_b200.spec import edge_decoder_spec
    from brepgen_b200.synth import synth_state_dict
    network = load_reference_network_with_leaves()
    # constructor arguments of sample.py:86-97
    vae = network.AutoencoderKL1DFastDecode(
        in_channels=3, out_channels=3,
        down_block_types=["DownBlock1D", "DownBlock1D", "DownBlock1D"], up_block_types=["UpBlock1D", "UpBlock1D", "UpBlock1D"],
        block_out_channels=[128, 256, 512], layers_per_block=2, act_fn="silu", latent_channels=3, norm_num_groups=32,
        sample_size=512)
    sd = synth_state_dict(edge_decoder_spec(), seed=2)
    ref_keys = {k: tuple(v.shape) for k, v in vae.state_dict().items()}
    assert ref_keys == {k: tuple(v.shape) for k, v in sd.items()}, set(ref_keys) ^ set(sd)
    vae.load_state_dict(sd)          # strict
    vae.eval()
    out = {}
    for seed, n in ((0, 3), (1, 7)):
        with torch.no_grad():
            out[f"s{seed}"] = vae(inputs(seed, n)).numpy().astype(np.float32)
        print("case", seed, out[f"s{seed}"].shape, float(np.abs(out[f"s{seed}"]).max()))
    # the encoder of BASELINE config 1's edge analogue: AutoencoderKL1DFastEncode (network.py:690-783) over Encoder1D
    # (:86-185, the reference's own) with the constructor arguments of trainer.py:841-852; its down blocks are diffusers'
    from brepgen_b200.spec import edge_encoder_spec
    enc = network.AutoencoderKL1DFastEncode(
        in_channels=3, out_channels=3,
        down_block_types=["DownBlock1D", "DownBlock1D", "DownBlock1D"], up_block_types=["UpBlock1D", "UpBlock1D", "UpBlock1D"],
        block_out_channels=[128, 256, 512], layers_per_block=2, act_fn="silu", latent_channels=3, norm_num_groups=32,
        sample_size=512)
    sde = synth_state_dict(edge_encoder_spec(), seed=3)
    enc_keys = {k: tuple(v.shape) for k, v in enc.state_dict().items()}
    assert enc_keys == {k: tuple(v.shape) for k, v in sde.items()}, set(enc_keys) ^ set(sde)
    enc.load_state_dict(sde)
    enc.eval()
    for seed, n in ((0, 2), (1, 5)):
        with torch.no_grad():
            out[f"enc_s{seed}"] = enc(enc_inputs(seed, n)).numpy().astype(np.float32)
        print("encoder case", seed, out[f"enc_s{seed}"].shape, float(np.abs(out[f"enc_s{seed}"]).max()))
    path = os.path.join(ROOT, "tests", "golden", "vae1d_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; keys checked:", len(ref_keys))


if __name__ == "__main__":
    main()
