"""ORACLE (test infrastructure): per-sample classifier-free guidance as a stack of single-sample runs.

The oracle drivers are per-sample in their arithmetic: sample b of a batch only ever meets its own rows (the denoisers
run per sample, the CFG combine p[:B] * (1 + w) - p[B:] * w is elementwise, the de-duplication loops are per sample).  So
the reference for a mixed batch -- sample b with its own class label, guidance scale w_b and negative label -- is the
stack of B = 1 runs of the existing drivers (oracle.cascade.run_cascade, oracle.ddim, oracle.dpm, oracle.unipc,
oracle.repaint, oracle.completion, oracle.variation, oracle.inversion), each with scalar fields and its own slice of the
explicit initial and step noise.  The drivers label the unconditional half of their CFG-doubled batch 0 ("uncond", as
the reference does, sample.py:46-51); `negative_forwards` relabels that half with the sample's negative label, and is
the identity for a negative label of 0.  A w = 0 sample still evaluates its unconditional row here; its result is
e * 1 - e_u * 0 = e, which is what the product computes without that row.
"""
from __future__ import annotations

from dataclasses import fields, is_dataclass, replace

import torch

from . import denoisers as O

NETS = ("surfpos", "surfz", "edgepos", "edgez")


def oracle_forwards(sds):
    """the drivers' default forwards: the oracle denoisers on the state dicts sds"""
    return {"surfpos": lambda *a: O.surfpos_forward(sds["surfpos"], *a),
            "surfz": lambda *a: O.surfz_forward(sds["surfz"], *a),
            "edgepos": lambda *a: O.edgepos_forward(sds["edgepos"], *a),
            "edgez": lambda *a: O.edgez_forward(sds["edgez"], *a)}


def negative_forwards(forwards, negative_label: int):
    """forwards whose class-label tensor (last argument, (2B, 1): B conditional rows, then B unconditional rows) has its
    second half set to negative_label"""
    if int(negative_label) == 0:
        return forwards

    def wrap(f):
        def g(*a):
            label = a[-1].clone()
            label[label.shape[0] // 2:] = int(negative_label)
            return f(*a[:-1], label)
        return g
    return {k: wrap(f) for k, f in forwards.items()}


def take(v, b: int, B: int):
    """sample b of a batch-shaped value: tensors with B rows, sequences of B entries and dataclasses (Completion,
    Variation, Interpolation) field by field; dicts entry by entry; anything else as it is"""
    if torch.is_tensor(v):
        return v[b:b + 1] if v.dim() > 0 and v.shape[0] == B else v
    if isinstance(v, dict):
        return {k: take(x, b, B) for k, x in v.items()}
    if is_dataclass(v) and not isinstance(v, type):
        return replace(v, **{f.name: take(getattr(v, f.name), b, B) for f in fields(v)})
    if isinstance(v, (list, tuple)) and len(v) == B:
        return type(v)([v[b]])
    return v


def run_stacked(driver, sds, cfg, classes, negatives, weights, args_of, forwards=None):
    """the stack over b of driver(sds, cfg_b, *args, forwards=..., **kwargs), (args, kwargs) = args_of(b), with cfg_b =
    cfg at batch_size 1 with class_label classes[b], guidance_w weights[b] and negative label negatives[b] (use_cf
    configs).  Outputs are concatenated along the batch; every sample must give the same shapes (CFG: S = num_surfaces)."""
    B = cfg.batch_size
    if not (len(classes) == len(negatives) == len(weights) == B):
        raise ValueError(f"per-sample fields need {B} entries each")
    base = oracle_forwards(sds) if forwards is None else forwards
    outs = []
    for b in range(B):
        cfg_b = replace(cfg, batch_size=1, class_label=int(classes[b]), guidance_w=float(weights[b]), negative_label=0)
        args, kwargs = args_of(b)
        outs.append(driver(sds, cfg_b, *args, forwards=negative_forwards(base, negatives[b]), **kwargs))
    return {k: torch.cat([o[k] for o in outs], 0) for k in outs[0]}
