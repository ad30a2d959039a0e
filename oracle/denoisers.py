"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of BrepGen's four denoisers.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module; the product path (brepgen_b200/) never does.

Restates, as plain functions over a state dict (no nn.Module, so nothing is shared with the
reference's class structure):
  sincos_embedding   network.py:1043-1063  (cos first, then sin; fp32)
  embed MLPs         network.py:1080-1099 etc.  Linear -> LayerNorm(eps 1e-5) -> SiLU -> Linear
  encoder            network.py:1076-1078 = torch nn.TransformerEncoder(12 x pre-norm layer, final LN):
                     x += out_proj(softmax(q k^T / 8 + kpm) v);  x += W2 relu(W1 LN2(x) + b1) + b2
  SurfPosNet.forward network.py:1107-1126
  SurfZNet.forward   network.py:1176-1200
  EdgePosNet.forward network.py:1257-1286   (faces x edges flattened to ONE sequence; face mask repeated)
  EdgeZNet.forward   network.py:1357-1393   (token = 12 edge latent + 6 vertex coords)

Pinned: tests/golden/denoisers_*.npz hold outputs of the reference's OWN classes (imported from
the reference with `diffusers` stubbed, see tests/golden/make_golden.py) on the same synthetic
weights; tests/test_oracle_golden.py checks this restatement against them.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]
D, NHEAD, NLAYER = 768, 12, 12


def sincos_embedding(t: torch.Tensor, dim: int = D, max_period: float = 10000.0) -> torch.Tensor:
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half).to(t.device)
    args = t.to(torch.float32).unsqueeze(-1) * freqs
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def _ln(x, sd: SD, name: str, eps: float = 1e-5):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], eps)


def _lin(x, sd: SD, name: str):
    return x @ sd[name + ".weight"].t() + sd[name + ".bias"]


def embed_mlp(sd: SD, name: str, x: torch.Tensor) -> torch.Tensor:
    h = _lin(x, sd, name + ".0")
    h = F.silu(_ln(h, sd, name + ".1"))
    return _lin(h, sd, name + ".3")


def encoder(sd: SD, x: torch.Tensor, key_padding_mask: Optional[torch.Tensor], prefix: str = "net") -> torch.Tensor:
    """x: (B, L, 768) batch-first (the reference permutes to seq-first and back; same math)."""
    B, L, _ = x.shape
    dh = D // NHEAD
    bias = None
    if key_padding_mask is not None:
        bias = torch.zeros(B, 1, 1, L, dtype=x.dtype, device=x.device)
        bias.masked_fill_(key_padding_mask.view(B, 1, 1, L), float("-inf"))
    for i in range(NLAYER):
        p = f"{prefix}.layers.{i}"
        h = _ln(x, sd, p + ".norm1")
        qkv = h @ sd[p + ".self_attn.in_proj_weight"].t() + sd[p + ".self_attn.in_proj_bias"]
        q, k, v = qkv.split(D, dim=-1)
        q = q.view(B, L, NHEAD, dh).transpose(1, 2)
        k = k.view(B, L, NHEAD, dh).transpose(1, 2)
        v = v.view(B, L, NHEAD, dh).transpose(1, 2)
        # softmax(q k^T / sqrt(dh) + kpm) v through torch's fused CPU kernel: the same arithmetic without the
        # (B, 12, L, L) score tensor (768 MB per layer at L = 4000), which is also how the reference's
        # nn.MultiheadAttention evaluates it -- the materialised form was 6x slower and not representative as a baseline
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=bias)
        a = a.transpose(1, 2).reshape(B, L, D)
        x = x + _lin(a, sd, p + ".self_attn.out_proj")
        h = _ln(x, sd, p + ".norm2")
        x = x + _lin(torch.relu(_lin(h, sd, p + ".linear1")), sd, p + ".linear2")
    return _ln(x, sd, prefix + ".norm")


def _cond(sd: SD, timesteps: torch.Tensor, class_label: Optional[torch.Tensor]) -> torch.Tensor:
    """time (+ class) embedding, shape (1|B, 1, 768)."""
    c = embed_mlp(sd, "time_embed", sincos_embedding(timesteps)).unsqueeze(1)
    if "class_embed.embed.weight" in sd:
        c = c + sd["class_embed.embed.weight"][class_label]      # (B,1) -> (B,1,768)
    return c


def surfpos_forward(sd: SD, surfPos, timesteps, class_label=None):
    tokens = embed_mlp(sd, "p_embed", surfPos) + _cond(sd, timesteps, class_label)
    return embed_mlp(sd, "fc_out", encoder(sd, tokens, None))


def surfz_forward(sd: SD, surfZ, timesteps, surfPos, surf_mask, class_label=None):
    tokens = embed_mlp(sd, "z_embed", surfZ) + embed_mlp(sd, "p_embed", surfPos) + _cond(sd, timesteps, class_label)
    return embed_mlp(sd, "fc_out", encoder(sd, tokens, surf_mask))


def edgepos_forward(sd: SD, edgePos, timesteps, surfPos, surfZ, mask, class_label=None):
    B, S, E, _ = edgePos.shape
    surf = embed_mlp(sd, "surfp_embed", surfPos) + embed_mlp(sd, "surfz_embed", surfZ)       # (B,S,768)
    tokens = (surf.unsqueeze(2) + embed_mlp(sd, "edgep_embed", edgePos)).reshape(B, S * E, D)
    tokens = tokens + _cond(sd, timesteps, class_label)
    kpm = mask.unsqueeze(-1).expand(B, S, E).reshape(B, S * E)
    out = embed_mlp(sd, "fc_out", encoder(sd, tokens, kpm))
    return out.view(B, S, E, -1)


def edgez_forward(sd: SD, edge, timesteps, edgePos, surfPos, surfZ, mask, class_label=None):
    B, S, E, _ = edgePos.shape
    edgeZ, vertPos = edge[..., :12], edge[..., 12:]
    surf = embed_mlp(sd, "surfp_embed", surfPos) + embed_mlp(sd, "surfz_embed", surfZ)
    tok = surf.unsqueeze(2) + embed_mlp(sd, "edgep_embed", edgePos) + embed_mlp(sd, "edgez_embed", edgeZ) \
        + embed_mlp(sd, "vertp_fc", vertPos)
    tokens = tok.reshape(B, S * E, D) + _cond(sd, timesteps, class_label)
    out = embed_mlp(sd, "fc_out", encoder(sd, tokens, mask.reshape(B, S * E)))
    return out.view(B, S, E, -1)


FORWARDS = {"surfpos": surfpos_forward, "surfz": surfz_forward, "edgepos": edgepos_forward, "edgez": edgez_forward}
