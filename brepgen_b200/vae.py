"""Drop-in VAE decoders (and the encoders of BASELINE config 1) with the reference's constructor kwargs, forward
signature and state-dict keys.

    AutoencoderKLFastDecode(**cfg).forward(z)      network.py:948-1040   z (N,3,4,4) -> (N,3,32,32)   cfg sample.py:72-82
    AutoencoderKL1DFastDecode(**cfg).forward(z)    network.py:786-858    z (N,3,4)   -> (N,3,32)      cfg sample.py:86-97

`load_state_dict(torch.load(path), strict=False)` (sample.py:83,98) works on full auto-encoder checkpoints: only
`decoder.*` and `post_quant_conv.*` keys exist here, everything else is reported as unexpected and ignored, exactly as with
the reference's decoder-only modules.  Arithmetic: libbrepgen_b200.so (csrc/vae.cu).  Only the architecture the reference
instantiates is supported (block_out_channels [128,256,512,512] / [128,256,512], layers_per_block 2, latent 3, groups 32).
"""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.nn as nn

from . import _ffi
from .models import _register_tree
from .spec import (CUBIC_DOWN_KERNEL, CUBIC_UP_KERNEL, edge_decoder_spec, edge_encoder_spec, surf_decoder_spec,
                   surf_encoder_spec)
from .synth import synth_state_dict


class _VaeModule(nn.Module):
    kind = 0
    chunk = 1024          # samples per library call (bounds the im2col workspace)

    def __init__(self, spec, expect, cfg):
        super().__init__()
        for k, v in expect.items():
            if k in cfg and list(cfg[k]) != list(v):
                raise NotImplementedError(f"{type(self).__name__}: only {k}={v} (the reference's sample.py config) is built")
        for key, shape in spec:
            if key.endswith(".kernel"):       # fixed resampling taps: a registered buffer, like diffusers' Up/Downsample1d
                taps = CUBIC_UP_KERNEL if key.endswith("up.kernel") else CUBIC_DOWN_KERNEL
                _register_tree(self, key, torch.tensor(taps, dtype=torch.float32), buffer=True)
            else:
                _register_tree(self, key, torch.zeros(shape) if len(shape) == 1 else torch.randn(shape) * 0.02)
        self._handle, self._sig, self._ws = None, None, None
        self._graphs = {}
        self.use_graph = os.environ.get("BREPGEN_B200_VAE_GRAPH", "1") != "0"   # replay one captured chunk per chunk

    def _release(self):
        if self._handle is not None:
            _ffi.lib().bg_vae_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _ensure(self, device):
        sd = self.state_dict()
        sig = tuple((v.data_ptr(), v._version) for v in sd.values())
        if self._handle is not None and sig == self._sig:
            return
        self._release()
        arr = _ffi.named_tensors(sd, device)
        out = C.c_void_p()
        _ffi.check(_ffi.lib().bg_vae_create(self.kind, arr, len(arr), _ffi.current_stream(), C.byref(out)), "bg_vae_create")
        torch.cuda.current_stream().synchronize()
        self._handle, self._sig = out, sig
        self._graphs = {}

    def forward(self, z: torch.Tensor) -> torch.Tensor:
        want_dim = 4 if self.kind in (0, 2) else 3       # surface VAEs: (N,3,H,W); edge VAEs: (N,3,L)
        if z.dim() != want_dim or z.shape[1] != 3 or z.shape[0] < 1:
            raise RuntimeError(f"{type(self).__name__}: expected a non-empty {want_dim}-D tensor with 3 channels, "
                               f"got {tuple(z.shape)}")
        if not z.is_cuda:
            raise RuntimeError("brepgen_b200 has no CPU path: z must be a CUDA tensor on an sm_90 (H100) device")
        dev = z.device
        z = z.detach().float().contiguous()
        N = z.shape[0]
        encode = self.kind >= 2
        hw = z.shape[-1]
        if z.dim() == 4 and z.shape[2] != z.shape[3]:
            raise NotImplementedError("only square grids")
        spatial = tuple((s // 8) if encode else (s * 8) for s in z.shape[2:])
        out = torch.empty((N, 3) + spatial, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            self._ensure(dev)
            step = min(self.chunk, N)
            need = _ffi.lib().bg_vae_workspace_bytes(self._handle, step)
            if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
                self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
                self._graphs = {}            # captured chunks point into the old workspace
            fn = _ffi.lib().bg_vae_encode if encode else _ffi.lib().bg_vae_decode_hw
            what = "bg_vae_encode" if encode else "bg_vae_decode"

            def run(zp, n, op):
                _ffi.check(fn(self._handle, zp, n, hw, op, self._ws.data_ptr(), self._ws.numel(), _ffi.current_stream()), what)

            full = N // step
            use_graph = self.use_graph and full >= 3 and not torch.cuda.is_current_stream_capturing()
            if use_graph:
                # A chunk is ~350 stream-ordered launches; with dozens of chunks per call (25 600 faces, 1 M edges at
                # B = 256) the host side dominates and, with 8 ranks on one host, contends.  One chunk is captured in a CUDA
                # graph over static staging buffers and replayed per chunk (two device copies around each replay).
                key = (self._handle.value, step, hw, tuple(z.shape[1:]), dev.index)
                g = self._graphs.get(key)
                if g is None:
                    zs, os_ = torch.empty_like(z[:step]), torch.empty_like(out[:step])
                    run(z[:step].data_ptr(), step, os_.data_ptr())           # warm-up outside the capture
                    graph = torch.cuda.CUDAGraph()
                    l0 = _ffi.lib().bg_launch_count()
                    with torch.cuda.graph(graph):
                        run(zs.data_ptr(), step, os_.data_ptr())
                    g = self._graphs[key] = (graph, zs, os_, _ffi.lib().bg_launch_count() - l0)
                graph, zs, os_, per_replay = g
                for c in range(full):
                    zs.copy_(z[c * step:(c + 1) * step])
                    graph.replay()
                    out[c * step:(c + 1) * step].copy_(os_)
                _ffi.note_replay(per_replay, full)
                lo0 = full * step
            else:
                lo0 = 0
            for lo in range(lo0, N, step):
                n = min(step, N - lo)
                run(z[lo:lo + n].data_ptr(), n, out[lo:lo + n].data_ptr())
        return out


class AutoencoderKLFastDecode(_VaeModule):
    kind = 0
    chunk = 1024

    def __init__(self, in_channels=3, out_channels=3, down_block_types=None, up_block_types=None,
                 block_out_channels=(128, 256, 512, 512), layers_per_block=2, act_fn="silu", latent_channels=3,
                 norm_num_groups=32, sample_size=512, **unused):
        cfg = dict(block_out_channels=block_out_channels)
        if (in_channels, out_channels, layers_per_block, act_fn, latent_channels, norm_num_groups) != (3, 3, 2, "silu", 3, 32):
            raise NotImplementedError("AutoencoderKLFastDecode: only the configuration of sample.py:72-82 is built")
        super().__init__(surf_decoder_spec(), dict(block_out_channels=[128, 256, 512, 512]), cfg)


class AutoencoderKL1DFastDecode(_VaeModule):
    kind = 1
    chunk = 32768

    def __init__(self, in_channels=3, out_channels=3, down_block_types=None, up_block_types=None,
                 block_out_channels=(128, 256, 512), layers_per_block=2, act_fn="silu", latent_channels=3,
                 norm_num_groups=32, sample_size=512, **unused):
        cfg = dict(block_out_channels=block_out_channels)
        if (in_channels, out_channels, layers_per_block, act_fn, latent_channels, norm_num_groups) != (3, 3, 2, "silu", 3, 32):
            raise NotImplementedError("AutoencoderKL1DFastDecode: only the configuration of sample.py:86-97 is built")
        super().__init__(edge_decoder_spec(), dict(block_out_channels=[128, 256, 512]), cfg)


class AutoencoderKLFastEncode(_VaeModule):
    """network.py:861-945: forward(x (N,3,H,W)) -> DiagonalGaussianDistribution(quant_conv(encoder(x))).mode()"""
    kind = 2
    chunk = 1024

    def __init__(self, in_channels=3, out_channels=3, down_block_types=None, up_block_types=None,
                 block_out_channels=(128, 256, 512, 512), layers_per_block=2, act_fn="silu", latent_channels=3,
                 norm_num_groups=32, sample_size=512, **unused):
        if (in_channels, layers_per_block, act_fn, latent_channels, norm_num_groups) != (3, 2, "silu", 3, 32):
            raise NotImplementedError("AutoencoderKLFastEncode: only the reference's surface-VAE configuration is built")
        super().__init__(surf_encoder_spec(), dict(block_out_channels=[128, 256, 512, 512]),
                         dict(block_out_channels=block_out_channels))


class AutoencoderKL1DFastEncode(_VaeModule):
    """network.py:690-783: forward(x (N,3,32)) -> latent mode (N,3,4)"""
    kind = 3
    chunk = 32768

    def __init__(self, in_channels=3, out_channels=3, down_block_types=None, up_block_types=None,
                 block_out_channels=(128, 256, 512), layers_per_block=2, act_fn="silu", latent_channels=3,
                 norm_num_groups=32, sample_size=512, **unused):
        if (in_channels, layers_per_block, act_fn, latent_channels, norm_num_groups) != (3, 2, "silu", 3, 32):
            raise NotImplementedError("AutoencoderKL1DFastEncode: only the reference's edge-VAE configuration is built")
        super().__init__(edge_encoder_spec(), dict(block_out_channels=[128, 256, 512]),
                         dict(block_out_channels=block_out_channels))


def build_synthetic_decoders(device, seed: int = 2):
    """random-init decoders (there are no checkpoints offline) for the bench and the tests"""
    s, e = AutoencoderKLFastDecode(), AutoencoderKL1DFastDecode()
    s.load_state_dict(synth_state_dict(surf_decoder_spec(), seed), strict=False)
    e.load_state_dict(synth_state_dict(edge_decoder_spec(), seed), strict=False)
    return s.to(device).eval(), e.to(device).eval()


# ------------------------------------------------------------------------------------------------ training-side latent pass
def encode_surface_latents(surf_vae, surfPnt: torch.Tensor, z_scaled: float = 1.0) -> torch.Tensor:
    """The frozen-encoder pass that feeds LDM training (trainer.py:518-524, :704-709, :918-927): surfPnt (B, S, 32, 32, 3)
    -> surfZ (B, S, 48) = flattened 4 x 4 x 3 latent of every face (position-major, channel-minor) times z_scaled."""
    bsz = surfPnt.shape[0]
    surf_uv = surfPnt.flatten(0, 1).permute(0, 3, 1, 2)
    surf_z = surf_vae(surf_uv.contiguous())
    surf_z = surf_z.unflatten(0, (bsz, -1)).flatten(-2, -1).permute(0, 1, 3, 2)
    return surf_z.flatten(-2, -1) * z_scaled


def encode_edge_latents(edge_vae, edgePnt: torch.Tensor, z_scaled: float = 1.0) -> torch.Tensor:
    """trainer.py:922-928: edgePnt (B, S, E, 32, 3) -> edgeZ (B, S, E, 12) = flattened 4 x 3 latent of every edge times z_scaled"""
    bsz, _, max_edge = edgePnt.shape[:3]
    edge_u = edgePnt.flatten(0, 1).flatten(0, 1).permute(0, 2, 1)
    edge_z = edge_vae(edge_u.contiguous())
    edge_z = edge_z.unflatten(0, (-1, max_edge)).unflatten(0, (bsz, -1)).permute(0, 1, 2, 4, 3)
    return edge_z.flatten(-2, -1) * z_scaled
