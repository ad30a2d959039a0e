"""Drop-in VAE decoders (and the encoders of BASELINE config 1) with the reference's constructor kwargs, forward
signature and state-dict keys.

    AutoencoderKLFastDecode(**cfg).forward(z)      network.py:948-1040   z (N,3,4,4) -> (N,3,32,32)   cfg sample.py:72-82
    AutoencoderKL1DFastDecode(**cfg).forward(z)    network.py:786-858    z (N,3,4)   -> (N,3,32)      cfg sample.py:86-97

`load_state_dict(torch.load(path), strict=False)` (sample.py:83,98) works on full auto-encoder checkpoints: only
`decoder.*` and `post_quant_conv.*` keys exist here, everything else is reported as unexpected and ignored, exactly as with
the reference's decoder-only modules.

    AutoencoderKL(**cfg)      diffusers AutoencoderKL as trainer.py:20-30 builds it      x (N,3,H,W), H = W in {8,16,24,32}
    AutoencoderKL1D(**cfg)    network.py:316-687 as trainer.py:146-157 builds it          x (N,3,32)

are the full auto-encoders of the VAE trainers: the whole checkpoint (encoder, quant_conv, decoder, post_quant_conv) with
strict=True, `encode(x).latent_dist` (DiagonalGaussianDistribution), `decode(z).sample` and `forward`.  Arithmetic:
libbrepgen_b200.so (csrc/vae.cu).  Only the architecture the reference
instantiates is supported (block_out_channels [128,256,512,512] / [128,256,512], layers_per_block 2, latent 3, groups 32).
"""
from __future__ import annotations

import ctypes as C
import math
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


    # ---- shared by the encoders and the full auto-encoders
    def _input(self, x: torch.Tensor, two_d: bool) -> torch.Tensor:
        """x as the library reads it: a contiguous fp32 CUDA tensor (N,3,H,W) with H == W (two_d) or (N,3,L)"""
        want_dim = 4 if two_d else 3
        if x.dim() != want_dim or x.shape[1] != 3 or x.shape[0] < 1:
            raise RuntimeError(f"{type(self).__name__}: expected a non-empty {want_dim}-D tensor with 3 channels, "
                               f"got {tuple(x.shape)}")
        if not x.is_cuda:
            raise RuntimeError("brepgen_b200 has no CPU path: inputs must be CUDA tensors on an sm_90 (H100) device")
        if two_d and x.shape[2] != x.shape[3]:
            raise NotImplementedError("only square grids")
        return x.detach().float().contiguous()

    def _workspace(self, need: int, dev) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
            self._graphs = {}            # captured chunks point into the old workspace
        return self._ws

    def _run_chunks(self, key, ins, outs, call):
        """call(ins, n, outs) over slices of at most `chunk` samples of the tensors `ins` / `outs` (None entries stay None).
        With three or more full chunks, one chunk is captured in a CUDA graph over static buffers and replayed per chunk
        (inputs copied in, outputs copied out), as forward() does."""
        N = ins[0].shape[0]
        step = min(self.chunk, N)
        full = N // step
        part = lambda ts, lo, hi: [None if t is None else t[lo:hi] for t in ts]
        lo0 = 0
        if self.use_graph and full >= 3 and not torch.cuda.is_current_stream_capturing():
            key = key + (step, tuple(None if t is None else tuple(t.shape[1:]) for t in ins + outs), ins[0].device.index)
            g = self._graphs.get(key)
            if g is None:
                si = [None if t is None else torch.empty_like(t[:step]) for t in ins]
                so = [None if t is None else torch.empty_like(t[:step]) for t in outs]
                call(part(ins, 0, step), step, so)                          # warm-up outside the capture
                graph = torch.cuda.CUDAGraph()
                l0 = _ffi.lib().bg_launch_count()
                with torch.cuda.graph(graph):
                    call(si, step, so)
                g = self._graphs[key] = (graph, si, so, _ffi.lib().bg_launch_count() - l0)
            graph, si, so, per_replay = g
            for c in range(full):
                for s, t in zip(si, ins):
                    if t is not None:
                        s.copy_(t[c * step:(c + 1) * step])
                graph.replay()
                for s, t in zip(so, outs):
                    if t is not None:
                        t[c * step:(c + 1) * step].copy_(s)
            _ffi.note_replay(per_replay, full)
            lo0 = full * step
        for lo in range(lo0, N, step):
            hi = min(N, lo + step)
            call(part(ins, lo, hi), hi - lo, part(outs, lo, hi))

    def _encode(self, x: torch.Tensor, return_dict: bool):
        """encoder handles: x -> AutoencoderKLOutput(latent_dist=DiagonalGaussianDistribution(quant_conv(encoder(x))))"""
        x = self._input(x, self.kind == 2)
        N, hw = x.shape[0], x.shape[-1]
        moments = torch.empty((N, 6) + tuple(s // 8 for s in x.shape[2:]), device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            self._ensure(x.device)
            ws = self._workspace(_ffi.lib().bg_vae_workspace_bytes(self._handle, min(self.chunk, N)), x.device)

            def call(i, n, o):
                _ffi.check(_ffi.lib().bg_vae_encode_moments(self._handle, i[0].data_ptr(), n, hw, o[0].data_ptr(),
                                                            ws.data_ptr(), ws.numel(), _ffi.current_stream()),
                           "bg_vae_encode_moments")
            self._run_chunks(("encode", self._handle.value, hw), [x], [moments], call)
        posterior = DiagonalGaussianDistribution(moments)
        return AutoencoderKLOutput(latent_dist=posterior) if return_dict else (posterior,)


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

    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """network.py:753-762: x (N,3,32) -> AutoencoderKLOutput(latent_dist=DiagonalGaussianDistribution((N,6,4) moments))"""
        return self._encode(x, return_dict)


# ------------------------------------------------------------------------------------------------ full auto-encoders
class AutoencoderKLOutput:
    """diffusers' AutoencoderKLOutput: `.latent_dist`; out[0] is the posterior"""

    def __init__(self, latent_dist):
        self.latent_dist = latent_dist

    def __getitem__(self, i):
        return (self.latent_dist,)[i]


class DecoderOutput:
    """diffusers' DecoderOutput: `.sample`; out[0] is the decoded tensor"""

    def __init__(self, sample):
        self.sample = sample

    def __getitem__(self, i):
        return (self.sample,)[i]


def randn_tensor(shape, generator=None, device=None, dtype=None) -> torch.Tensor:
    """diffusers 0.27 `randn_tensor`: drawn on `device`, or on the CPU and then moved when `generator` is a CPU generator
    (a list of generators draws one sample each), so a seeded call gives the reference's noise"""
    device = torch.device(device) if device is not None else torch.device("cpu")
    if isinstance(generator, list) and len(generator) == 1:
        generator = generator[0]
    gens = generator if isinstance(generator, list) else [generator]
    rand_device = device
    if gens[0] is not None and gens[0].device.type != device.type:
        if gens[0].device.type != "cpu":
            raise ValueError(f"Cannot generate a {device} tensor from a generator of type {gens[0].device.type}.")
        rand_device = torch.device("cpu")
    if isinstance(generator, list):
        draws = [torch.randn((1,) + tuple(shape[1:]), generator=g, device=rand_device, dtype=dtype) for g in generator]
        return torch.cat(draws, dim=0).to(device)
    return torch.randn(tuple(shape), generator=generator, device=rand_device, dtype=dtype).to(device)


class DiagonalGaussianDistribution:
    """diffusers 0.27 `DiagonalGaussianDistribution` over device moments (N, 6, ...) = mean | logvar, the posterior that
    `encode(x).latent_dist` returns.  `sample()` and `kl()` run bg_vae_posterior; `kl(other)` and `nll` are plain tensor
    expressions (nothing on the trainers' path calls them).  The attributes are those of diffusers: `parameters`, `mean`,
    `logvar` (clamped to [-30, 20]), `std`, `var`, `deterministic`."""

    def __init__(self, parameters: torch.Tensor, deterministic: bool = False):
        self.parameters = parameters
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.deterministic = deterministic
        self._logvar_raw, self._logvar, self._std, self._var = logvar, None, None, None

    # std / var / logvar are computed on first use: the trainers' validation path never reads them
    @property
    def logvar(self) -> torch.Tensor:
        if self._logvar is None:
            self._logvar = torch.clamp(self._logvar_raw, -30.0, 20.0)
        return self._logvar

    @property
    def std(self) -> torch.Tensor:
        if self._std is None:
            self._std = torch.zeros_like(self.mean) if self.deterministic else torch.exp(0.5 * self.logvar)
        return self._std

    @property
    def var(self) -> torch.Tensor:
        if self._var is None:
            self._var = torch.zeros_like(self.mean) if self.deterministic else torch.exp(self.logvar)
        return self._var

    def _posterior(self, noise, want_z: bool, want_kl: bool):
        p = self.parameters
        if not p.is_cuda:
            raise RuntimeError("brepgen_b200 has no CPU path: the moments must be a CUDA tensor on an sm_90 (H100) device")
        if p.dim() < 3 or p.shape[1] != 6:
            raise NotImplementedError("only the reference's 3-channel latent (6 moment channels) is built")
        p = p.detach().float().contiguous()
        N, P = p.shape[0], p[0, 0].numel()
        z = torch.empty((N, 3) + tuple(p.shape[2:]), device=p.device, dtype=torch.float32) if want_z else None
        kl = torch.empty(N, device=p.device, dtype=torch.float32) if want_kl else None
        if noise is not None:
            noise = noise.float().contiguous()
        with torch.cuda.device(p.device):
            _ffi.check(_ffi.lib().bg_vae_posterior(p.data_ptr(), _ffi.ptr(noise), N, P, int(bool(self.deterministic)),
                                                   _ffi.ptr(z), _ffi.ptr(kl), _ffi.current_stream()), "bg_vae_posterior")
        return z, kl

    def sample(self, generator=None) -> torch.Tensor:
        noise = randn_tensor(self.mean.shape, generator=generator, device=self.parameters.device,
                             dtype=self.parameters.dtype)
        return self._posterior(noise, True, False)[0]

    def mode(self) -> torch.Tensor:
        return self.mean

    def kl(self, other: "DiagonalGaussianDistribution" = None) -> torch.Tensor:
        if self.deterministic:
            return torch.Tensor([0.0])
        if other is None:
            if self.parameters.dim() != 4:        # diffusers sums over dim=[1, 2, 3]
                d = self.parameters.dim()
                raise IndexError(f"Dimension out of range (expected to be in range of [{-d}, {d - 1}], but got 3)")
            return self._posterior(None, False, True)[1]
        return 0.5 * torch.sum(torch.pow(self.mean - other.mean, 2) / other.var + self.var / other.var - 1.0 - self.logvar
                               + other.logvar, dim=[1, 2, 3])

    def nll(self, sample: torch.Tensor, dims=(1, 2, 3)) -> torch.Tensor:
        if self.deterministic:
            return torch.Tensor([0.0])
        return 0.5 * torch.sum(math.log(2.0 * math.pi) + self.logvar + torch.pow(sample - self.mean, 2) / self.var,
                               dim=list(dims))


class _AutoencoderKLModule(_VaeModule):
    """encoder -> posterior -> decoder with the reference's state dict (`encoder.*`, `quant_conv.*`, `decoder.*`,
    `post_quant_conv.*`): two native handles, the encoder (`kind`) and the decoder (`dec_kind`), packed from this module's
    parameters and re-packed when one of them changes.  Inference only; slicing does not change the result (accepted),
    tiling is not built.  The decoder handle runs three-term compensated products for both families: the edge decoder's
    default two terms (AutoencoderKL1DFastDecode) measure up to 1.1e-3 against the fp32 oracle on some weights, which the
    round trip of the trainers would carry into its losses."""
    dec_kind = 0

    def __init__(self, spec, expect, cfg):
        super().__init__(spec, expect, cfg)
        self._dec = None
        self.use_slicing = False
        self.use_tiling = False

    def _release(self):
        super()._release()
        if getattr(self, "_dec", None) is not None:
            _ffi.lib().bg_vae_destroy(self._dec)
            self._dec = None

    def _ensure(self, device):
        super()._ensure(device)          # the encoder handle; a changed parameter releases both handles first
        if self._dec is None:
            arr = _ffi.named_tensors(self.state_dict(), device)
            out = C.c_void_p()
            _ffi.check(_ffi.lib().bg_vae_create_ex(self.dec_kind, 3, arr, len(arr), _ffi.current_stream(), C.byref(out)),
                       "bg_vae_create_ex")
            torch.cuda.current_stream().synchronize()
            self._dec = out

    def enable_slicing(self):
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    def enable_tiling(self, use_tiling: bool = True):
        if use_tiling:
            raise NotImplementedError(f"{type(self).__name__}: tiled encode / decode is not built")
        self.use_tiling = False

    def disable_tiling(self):
        self.use_tiling = False

    def encode(self, x: torch.Tensor, return_dict: bool = True):
        return self._encode(x, return_dict)

    def decode(self, z: torch.Tensor, return_dict: bool = True):
        two_d = self.kind == 2
        z = self._input(z, two_d)
        N, hw = z.shape[0], z.shape[-1]
        dec = torch.empty((N, 3) + tuple(8 * s for s in z.shape[2:]), device=z.device, dtype=torch.float32)
        with torch.cuda.device(z.device):
            self._ensure(z.device)
            ws = self._workspace(_ffi.lib().bg_vae_workspace_bytes(self._dec, min(self.chunk, N)), z.device)

            def call(i, n, o):
                _ffi.check(_ffi.lib().bg_vae_decode_hw(self._dec, i[0].data_ptr(), n, hw, o[0].data_ptr(), ws.data_ptr(),
                                                       ws.numel(), _ffi.current_stream()), "bg_vae_decode")
            self._run_chunks(("decode", self._dec.value, hw), [z], [dec], call)
        return DecoderOutput(sample=dec) if return_dict else (dec,)

    def reconstruct(self, sample: torch.Tensor, sample_posterior: bool = True, generator=None):
        """The fused round trip: (dec, mse) with dec = forward(sample, sample_posterior, generator=generator).sample and
        mse (N,) = the per-sample mean of (dec - sample)^2, one bg_vae_reconstruct per chunk (encoder, posterior, decoder
        and error without leaving the device).  The noise is drawn as diffusers' posterior.sample(generator) draws it."""
        x = self._input(sample, self.kind == 2)
        N, hw = x.shape[0], x.shape[-1]
        noise = None
        if sample_posterior:
            latent = (N, 3) + tuple(s // 8 for s in x.shape[2:])
            noise = randn_tensor(latent, generator=generator, device=x.device, dtype=torch.float32).contiguous()
        dec, mse = torch.empty_like(x), torch.empty(N, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            self._ensure(x.device)
            need = _ffi.lib().bg_vae_reconstruct_workspace_bytes(self._handle, self._dec, min(self.chunk, N))
            ws = self._workspace(need, x.device)

            def call(i, n, o):
                _ffi.check(_ffi.lib().bg_vae_reconstruct(self._handle, self._dec, i[0].data_ptr(), n, hw, _ffi.ptr(i[1]),
                                                         None, None, None, o[0].data_ptr(), o[1].data_ptr(), ws.data_ptr(),
                                                         ws.numel(), _ffi.current_stream()), "bg_vae_reconstruct")
            self._run_chunks(("reconstruct", self._handle.value, self._dec.value, hw, noise is not None), [x, noise],
                             [dec, mse], call)
        return dec, mse

    def forward(self, sample: torch.Tensor, sample_posterior: bool = False, return_dict: bool = True, generator=None):
        """network.py:660-687 / diffusers AutoencoderKL.forward: encode, posterior sample (or mode), decode"""
        dec = self.reconstruct(sample, sample_posterior, generator)[0]
        return DecoderOutput(sample=dec) if return_dict else (dec,)


def _check_full_cfg(name, got, want):
    if got != want:
        raise NotImplementedError(f"{name}: only the configuration of the reference's VAE trainer is built")


class AutoencoderKL(_AutoencoderKLModule):
    """diffusers AutoencoderKL as SurfVAETrainer builds it (trainer.py:20-30): x (N,3,H,W), H = W in {8,16,24,32}"""
    kind, dec_kind = 2, 0
    chunk = 1024

    def __init__(self, in_channels=3, out_channels=3, down_block_types=None, up_block_types=None,
                 block_out_channels=(128, 256, 512, 512), layers_per_block=2, act_fn="silu", latent_channels=3,
                 norm_num_groups=32, sample_size=512, **unused):
        _check_full_cfg("AutoencoderKL", (in_channels, out_channels, layers_per_block, act_fn, latent_channels,
                                          norm_num_groups), (3, 3, 2, "silu", 3, 32))
        cfg = dict(block_out_channels=block_out_channels, down_block_types=down_block_types, up_block_types=up_block_types)
        super().__init__(surf_encoder_spec() + surf_decoder_spec(),
                         dict(block_out_channels=[128, 256, 512, 512], down_block_types=["DownEncoderBlock2D"] * 4,
                              up_block_types=["UpDecoderBlock2D"] * 4),
                         {k: v for k, v in cfg.items() if v is not None})


class AutoencoderKL1D(_AutoencoderKLModule):
    """network.py:316-687 as EdgeVAETrainer builds it (trainer.py:146-157): x (N,3,32)"""
    kind, dec_kind = 3, 1
    chunk = 32768

    def __init__(self, in_channels=3, out_channels=3, down_block_types=None, up_block_types=None,
                 block_out_channels=(128, 256, 512), layers_per_block=2, act_fn="silu", latent_channels=3,
                 norm_num_groups=32, sample_size=512, **unused):
        _check_full_cfg("AutoencoderKL1D", (in_channels, out_channels, layers_per_block, act_fn, latent_channels,
                                            norm_num_groups), (3, 3, 2, "silu", 3, 32))
        cfg = dict(block_out_channels=block_out_channels, down_block_types=down_block_types, up_block_types=up_block_types)
        super().__init__(edge_encoder_spec() + edge_decoder_spec(),
                         dict(block_out_channels=[128, 256, 512], down_block_types=["DownBlock1D"] * 3,
                              up_block_types=["UpBlock1D"] * 3),
                         {k: v for k, v in cfg.items() if v is not None})


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
