"""ORACLE-side helper (test infrastructure, not product code): import the reference's OWN `network.py`.

Only tests/, tests/golden/make_golden*.py, __graft_entry__ (build / smoke) and bench.py's CPU legs (`cpu_baseline`,
`--impl reference`) use this module; brepgen_b200/ never does.

The reference (samxuxiang/BrepGen) is a script collection without packaging, and `import network` needs `diffusers`
(absent offline) at module import time although the four denoisers (network.py:1066-1393), `sincos_embedding` (:1043) and
`Embedder` (:17) use torch only.  So the reference module is imported UNMODIFIED with inert stand-ins registered for the
`diffusers` names it imports; its denoiser classes then run their stock code path (nn.TransformerEncoder etc.).

Where the file comes from:
  * the reference checkout named by $BREPGEN_REFERENCE (default /root/reference),
    when it is readable;
  * oracle/_ref/network.py: `install_reference()` (called by __graft_entry__.build() whenever the reference checkout is
    readable) places an unmodified copy there, so that a copy of the built tree carries it to machines without the
    checkout.  oracle/_ref/ is git-ignored: the reference's source never enters this repository's history.
"""
from __future__ import annotations

import importlib.util
import os
import shutil
import sys
import types
from typing import Optional

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SRC = os.environ.get("BREPGEN_REFERENCE", "/root/reference")
REF_INSTALL = os.path.join(ROOT, "oracle", "_ref")
_FILES = ("network.py",)            # the only reference module the denoiser path needs


def install_reference() -> Optional[str]:
    """copy the reference module(s) of this path, unmodified, into oracle/_ref/ (no-op without a readable checkout)"""
    if not REF_SRC or not all(os.access(os.path.join(REF_SRC, f), os.R_OK) for f in _FILES):
        return REF_INSTALL if os.path.exists(os.path.join(REF_INSTALL, _FILES[0])) else None
    os.makedirs(REF_INSTALL, exist_ok=True)
    for f in _FILES:
        shutil.copyfile(os.path.join(REF_SRC, f), os.path.join(REF_INSTALL, f))
    return REF_INSTALL


def reference_dir() -> Optional[str]:
    for d in (REF_SRC, REF_INSTALL):
        if d and os.access(os.path.join(d, _FILES[0]), os.R_OK):
            return d
    return None


def _stub_diffusers() -> None:
    import torch

    class _Any:  # inert base / placeholder
        def __init__(self, *a, **k):
            pass

    def _identity_decorator(fn):
        return fn

    names = {
        "diffusers": {},
        "diffusers.configuration_utils": {"ConfigMixin": _Any, "register_to_config": _identity_decorator},
        "diffusers.utils": {"BaseOutput": _Any, "is_torch_version": lambda *a, **k: True},
        "diffusers.utils.accelerate_utils": {"apply_forward_hook": _identity_decorator},
        "diffusers.models": {},
        "diffusers.models.attention_processor": {"AttentionProcessor": _Any, "AttnProcessor": _Any, "SpatialNorm": _Any},
        "diffusers.models.modeling_utils": {"ModelMixin": torch.nn.Module},
        "diffusers.models.autoencoders": {},
        "diffusers.models.autoencoders.vae": {"Decoder": _Any, "DecoderOutput": _Any,
                                              "DiagonalGaussianDistribution": _Any, "Encoder": _Any},
        "diffusers.models.unets": {},
        "diffusers.models.unets.unet_1d_blocks": {"ResConvBlock": _Any, "SelfAttention1d": _Any, "get_down_block": _Any,
                                                  "get_up_block": _Any, "Upsample1d": _Any},
    }
    for name, attrs in names.items():
        if name in sys.modules:
            continue
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m


_cached = None


def load_reference_network(required: bool = True):
    """the reference's network module (its real file, executed unmodified), or None / RuntimeError when unavailable"""
    global _cached
    if _cached is not None:
        return _cached
    d = reference_dir()
    if d is None:
        if required:
            raise RuntimeError("reference network.py not found (neither $BREPGEN_REFERENCE nor oracle/_ref): "
                               "run __graft_entry__.build() where the reference checkout is readable")
        return None
    _stub_diffusers()
    spec = importlib.util.spec_from_file_location("brepgen_reference_network", os.path.join(d, "network.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod          # @dataclass looks its module up in sys.modules while the file executes
    spec.loader.exec_module(mod)
    assert os.path.abspath(mod.__file__).startswith(d)
    _cached = mod
    return mod
