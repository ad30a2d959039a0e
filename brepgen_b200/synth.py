"""Deterministic synthetic weights, keyed by state-dict name.

There are no checkpoints offline (SURVEY.md §6), so tests, the bench and the golden-vector
generator all need the *same* random-init weights without shipping ~200 MB per network.
Every tensor is drawn from its own generator seeded by crc32(key) + seed, so the result does
not depend on module construction order or on which framework class holds the parameter.

Magnitudes follow torch's default inits used by the reference
(network.py:1066-1393 builds stock nn.Linear / nn.LayerNorm /
nn.TransformerEncoderLayer): 2-D weights U(+-1/sqrt(fan_in)), LayerNorm/GroupNorm weights
1 + 0.1 N(0,1) (non-trivial on purpose so the affine path is exercised), biases 0.05 N(0,1).
"""
from __future__ import annotations

import math
import zlib
from typing import Dict, Iterable, Tuple

import torch


def _gen(key: str, seed: int) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((zlib.crc32(key.encode()) + 1000003 * seed) & 0x7FFFFFFF)
    return g


def synth_tensor(key: str, shape: Tuple[int, ...], seed: int = 0) -> torch.Tensor:
    g = _gen(key, seed)
    shape = tuple(shape)
    if key.endswith("up.kernel"):   # fixed resampling buffer of diffusers Upsample1d("cubic"), not a learnt weight
        from .spec import CUBIC_UP_KERNEL
        return torch.tensor(CUBIC_UP_KERNEL, dtype=torch.float32)
    if key.endswith("down.kernel"):
        from .spec import CUBIC_DOWN_KERNEL
        return torch.tensor(CUBIC_DOWN_KERNEL, dtype=torch.float32)
    if len(shape) >= 2:
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        bound = 1.0 / math.sqrt(max(fan_in, 1))
        return (torch.rand(shape, generator=g, dtype=torch.float32) * 2.0 - 1.0) * bound
    if key.endswith("weight"):  # 1-D weight == normalisation scale
        return 1.0 + 0.1 * torch.randn(shape, generator=g, dtype=torch.float32)
    return 0.05 * torch.randn(shape, generator=g, dtype=torch.float32)


def synth_state_dict(spec: Iterable[Tuple[str, Tuple[int, ...]]], seed: int = 0) -> Dict[str, torch.Tensor]:
    """spec: iterable of (key, shape). Returns {key: fp32 CPU tensor}."""
    return {k: synth_tensor(k, s, seed) for k, s in spec}
