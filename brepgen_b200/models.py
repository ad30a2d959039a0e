"""Drop-in denoisers: same constructor, forward signature and state-dict keys as the reference classes.

    SurfPosNet(use_cf).forward(surfPos, timesteps, class_label, is_train=False)              network.py:1066-1126
    SurfZNet(use_cf).forward(surfZ, timesteps, surfPos, surf_mask, class_label, ...)          network.py:1129-1200
    EdgePosNet(use_cf).forward(edgePos, timesteps, surfPos, surfZ, mask, class_label, ...)    network.py:1203-1286
    EdgeZNet(use_cf).forward(edge, timesteps, edgePos, surfPos, surfZ, mask, class_label,...) network.py:1289-1393

so `sample.py:56-70` (`Net(use_cf); load_state_dict(torch.load(p)); .to(device).eval()`) and every call in the six
sampling loops work unchanged.  The parameters live in an nn.Module tree whose state_dict keys equal the
reference's; the arithmetic runs in libbrepgen_b200.so (wgmma GEMM + flash attention, see csrc/).  Inference
only: there is no autograd and no CPU path -- calling forward on a CPU tensor or with is_train=True raises.
Returned predictions are fp32 (the reference returns fp16 under its autocast context, sample.py:121).
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Dict

import torch
import torch.nn as nn

from . import _ffi
from .spec import D, denoiser_spec

_KIND_ID = {"surfpos": 0, "surfz": 1, "edgepos": 2, "edgez": 3}


def reference_sincos_table(n: int = 1000, dim: int = D) -> torch.Tensor:
    """sincos_embedding(t, 768) for t = 0..n-1, computed on the host with the same fp32 torch ops as
    network.py:1043-1063 (cos block first)."""
    half = dim // 2
    freqs = torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
    args = torch.arange(n).unsqueeze(-1).float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def _register_tree(root: nn.Module, key: str, tensor: torch.Tensor) -> None:
    parts = key.split(".")
    mod = root
    for p in parts[:-1]:
        if not hasattr(mod, p):
            mod.add_module(p, nn.Module())
        mod = getattr(mod, p)
    mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))


def _default_init(key: str, shape) -> torch.Tensor:
    """torch-default-like init (uniform +-1/sqrt(fan_in) weights and biases, unit norms); checkpoints overwrite it."""
    if len(shape) >= 2:
        bound = 1.0 / math.sqrt(shape[1])
        return (torch.rand(shape) * 2 - 1) * bound
    if key.endswith("weight"):
        return torch.ones(shape)
    if ".1." in key or "norm" in key:
        return torch.zeros(shape)
    return (torch.rand(shape) * 2 - 1) / math.sqrt(D)


class _Denoiser(nn.Module):
    kind = ""

    def __init__(self, use_cf):
        super().__init__()
        self.embed_dim = D
        self.use_cf = bool(use_cf)
        for key, shape in denoiser_spec(self.kind, self.use_cf):
            _register_tree(self, key, _default_init(key, shape))
        # 0 / 1 / 2, see include/brepgen_b200.h (bg_denoiser_create); 1 meets the 1e-3 parity bar with margin
        self.precision = int(os.environ.get("BREPGEN_B200_PRECISION", "1"))
        # mask-aware token compaction (BgDenoiserArgs.compact): on whenever a mask is passed; 0 = dense layout with masking only
        self.compact = int(os.environ.get("BREPGEN_B200_COMPACT", "1"))
        self._handle = None
        self._packed_sig = None
        self._dirty = True           # parameters may have changed since the last pack (set by load_state_dict / .to() / ...)
        self._ws: Dict[tuple, torch.Tensor] = {}

    # ---------------------------------------------------------------- native handle management
    def _signature(self):
        return (self.precision,) + tuple((p.data_ptr(), p._version) for p in self.parameters())

    # The packed device copy is rebuilt when the parameters change.  Walking ~190 parameters on every forward (1600+ forwards
    # per cascade) is pure host overhead on the latency-critical small-batch path, so the walk only happens after an event
    # that can change them: load_state_dict, any _apply (.to / .cuda / .float ...), or a changed `precision`.  Code that
    # writes into parameters in place some other way calls `mark_dirty()`.
    def mark_dirty(self):
        self._dirty = True

    def _apply(self, fn, *a, **k):
        self._dirty = True
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._dirty = True
        return super().load_state_dict(*a, **k)

    def __deepcopy__(self, memo):
        import copy
        new = type(self)(self.use_cf)
        new.load_state_dict(copy.deepcopy(self.state_dict(), memo))
        new.precision = self.precision
        return new

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_handle"], d["_packed_sig"], d["_dirty"], d["_ws"] = None, None, True, {}
        return d

    def _release(self):
        if self._handle is not None:
            _ffi.lib().bg_denoiser_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _ensure_packed(self, device):
        if self._handle is not None and not self._dirty and self._packed_sig[0] == self.precision:
            return
        sig = self._signature()
        if self._handle is not None and sig == self._packed_sig:
            self._dirty = False
            return
        self._release()
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        for k, v in sd.items():
            if v.device != device or v.dtype != torch.float32 or not v.is_contiguous():
                raise RuntimeError(f"parameter {k} must be contiguous fp32 on {device} (call .to(device) first)")
        names = [k.encode() for k in sd]
        arr = (_ffi.BgNamedTensor * len(sd))()
        for i, (k, v) in enumerate(sd.items()):
            arr[i].name, arr[i].data, arr[i].numel = names[i], v.data_ptr(), v.numel()
        sincos = reference_sincos_table().to(device)
        out = C.c_void_p()
        st = _ffi.current_stream()
        _ffi.check(_ffi.lib().bg_denoiser_create(_KIND_ID[self.kind], int(self.use_cf), int(self.precision), arr, len(sd),
                                                sincos.data_ptr(), st, C.byref(out)), "bg_denoiser_create")
        torch.cuda.current_stream().synchronize()   # weights / sincos may now be released or modified
        self._handle, self._packed_sig, self._dirty = out, sig, False

    def _workspace(self, B, S, E, device):
        key = (B, S, E, device.index)
        ws = self._ws.get(key)
        if ws is None:
            n = _ffi.lib().bg_denoiser_workspace_bytes(self._handle, B, S, E)
            self._ws = {key: torch.empty(n, dtype=torch.uint8, device=device)}   # keep only the latest shape
            ws = self._ws[key]
        return ws

    # the C ABI takes raw pointers: every shape is checked here, against the reference's forward signatures
    _X_WIDTH = {"surfpos": 6, "surfz": 48, "edgepos": 6, "edgez": 18}

    def _check_shapes(self, x, surfPos, surfZ, edgePos, mask):
        edge = self.kind in ("edgepos", "edgez")
        want_dim = 4 if edge else 3
        if x.dim() != want_dim or x.shape[-1] != self._X_WIDTH[self.kind]:
            raise RuntimeError(f"{type(self).__name__}: expected a {want_dim}-D input with last dimension "
                               f"{self._X_WIDTH[self.kind]}, got {tuple(x.shape)}")
        B, S = x.shape[0], x.shape[1]
        E = x.shape[2] if edge else 0
        if B < 1 or S < 1 or (edge and E < 1):
            raise RuntimeError(f"{type(self).__name__}: empty batch / face / edge dimension in {tuple(x.shape)}")

        def need(name, t, shape):
            if t is None:
                raise RuntimeError(f"{type(self).__name__}: {name} is required")
            if tuple(t.shape) != shape:
                raise RuntimeError(f"{type(self).__name__}: {name} must have shape {shape}, got {tuple(t.shape)}")

        if self.kind != "surfpos":
            need("surfPos", surfPos, (B, S, 6))
        if edge:
            need("surfZ", surfZ, (B, S, 48))
        if self.kind == "edgez":
            need("edgePos", edgePos, (B, S, E, 6))
        if mask is not None:
            want = (B, S, E) if self.kind == "edgez" else (B, S)
            if self.kind == "surfpos" or tuple(mask.shape) != want:
                raise RuntimeError(f"{type(self).__name__}: mask must have shape {want}, got {tuple(mask.shape)}")

    # ---------------------------------------------------------------- shared forward plumbing
    def _run(self, x, timesteps, surfPos=None, surfZ=None, edgePos=None, mask=None, class_label=None, is_train=False):
        if is_train:
            raise RuntimeError("brepgen_b200 denoisers are inference-only (is_train=True is the reference's training path)")
        self._check_shapes(x, surfPos, surfZ, edgePos, mask)
        if not x.is_cuda:
            raise RuntimeError("brepgen_b200 has no CPU path: inputs must be CUDA tensors on an sm_90 (H100) device")
        dev = x.device
        with torch.cuda.device(dev):
            self._ensure_packed(dev)
            f32 = lambda t: None if t is None else t.detach().to(device=dev, dtype=torch.float32).contiguous()
            x = f32(x)
            surfPos, surfZ, edgePos = f32(surfPos), f32(surfZ), f32(edgePos)
            ts = timesteps.detach().to(device=dev, dtype=torch.int64).reshape(-1).contiguous()
            B, S = x.shape[0], x.shape[1]
            E = x.shape[2] if x.dim() == 4 else 0
            if ts.numel() not in (1, B):
                raise RuntimeError(f"timesteps must have 1 or {B} elements, got {ts.numel()}")
            if mask is not None:
                mask = mask.detach().to(device=dev).to(torch.bool).contiguous()
            if self.use_cf:
                if class_label is None:
                    raise RuntimeError("class_label is required for use_cf=True")
                class_label = class_label.detach().to(device=dev, dtype=torch.int64).reshape(-1).contiguous()
                if class_label.numel() != B:
                    raise RuntimeError("class_label must have one entry per sample")
            else:
                class_label = None
            out = torch.empty_like(x)
            a = _ffi.BgDenoiserArgs(B, S, E, x.data_ptr(), ts.data_ptr(), ts.numel(), _ffi.ptr(surfPos), _ffi.ptr(surfZ),
                                    _ffi.ptr(edgePos), _ffi.ptr(mask), _ffi.ptr(class_label), out.data_ptr(),
                                    int(self.compact))
            ws = self._workspace(B, S, E, dev)
            _ffi.check(_ffi.lib().bg_denoiser_forward(self._handle, C.byref(a), ws.data_ptr(), ws.numel(),
                                                     _ffi.current_stream()), "bg_denoiser_forward")
        return out


class SurfPosNet(_Denoiser):
    kind = "surfpos"

    def forward(self, surfPos, timesteps, class_label, is_train=False):
        return self._run(surfPos, timesteps, class_label=class_label, is_train=is_train)


class SurfZNet(_Denoiser):
    kind = "surfz"

    def forward(self, surfZ, timesteps, surfPos, surf_mask, class_label, is_train=False):
        return self._run(surfZ, timesteps, surfPos=surfPos, mask=surf_mask, class_label=class_label, is_train=is_train)


class EdgePosNet(_Denoiser):
    kind = "edgepos"

    def forward(self, edgePos, timesteps, surfPos, surfZ, mask, class_label, is_train=False):
        return self._run(edgePos, timesteps, surfPos=surfPos, surfZ=surfZ, mask=mask, class_label=class_label,
                         is_train=is_train)


class EdgeZNet(_Denoiser):
    kind = "edgez"

    def forward(self, edge, timesteps, edgePos, surfPos, surfZ, mask, class_label, is_train=False):
        return self._run(edge, timesteps, surfPos=surfPos, surfZ=surfZ, edgePos=edgePos, mask=mask,
                         class_label=class_label, is_train=is_train)


NETS = {"surfpos": SurfPosNet, "surfz": SurfZNet, "edgepos": EdgePosNet, "edgez": EdgeZNet}
