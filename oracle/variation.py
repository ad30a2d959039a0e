"""ORACLE (test infrastructure): B-rep variations (SDEdit, diffusers' img2img `strength`) of the cascade driver.

run_cascade_variation restates the DDPM, DDIM and DPM-Solver++ drivers of oracle/cascade.py, oracle/ddim.py and
oracle/dpm.py on the tail of each stage's list that a strength selects (diffusers' get_timesteps:
timesteps[N - min(int(N * s), N):]).  A varied stage starts at add_noise(scale * gathered source, z, first timestep) in
fp32 torch; a stage with strength 0 is not run and returns the source.  The slot layout is written with plain Python
loops: the valid tokens of a source row repeated as the trainers' pad_repeat (utils.py:100-106) repeats them (pinned by
tests/golden/fill_golden.npz, which tests/golden/make_golden_fill.py computes by exec()'ing the reference's own
function), and the survivor list of the face de-duplication, recorded by the loop of dedup_surfaces_np
(sample.py:159-183).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import denoisers as O
from .cascade import dedup_edges_np
from .ddim import DDIMOracle
from .dpm import DPMOracle
from .schedulers import DDPMOracle, linear_alphas_cumprod

STAGES = ("surfPos", "surfZ", "edgePos", "edgeZV")


def pad_repeat_positions(n_valid: int, out_slots: int) -> list:
    """for each of out_slots slots, the position in a list of n_valid tokens that pad_repeat puts there: with
    r = floor(out / n) and sep = out - r n, each of the first sep tokens r + 1 times in a row, each later one r times"""
    r = math.floor(out_slots / n_valid)
    sep = out_slots - r * n_valid
    pos = []
    for k in range(n_valid):
        for _ in range(r + 1 if k < sep else r):
            pos.append(k)
    return pos


def fill_rows(mask: np.ndarray, out_slots: int, row_map=None) -> list:
    """mask (n_src_rows, in_slots) bool, True = padded; row_map: source row of each output row (-1 = none), default the
    identity -> per output row, out_slots flat source-token indices (-1: no source or no valid slot)"""
    n_src, in_slots = mask.shape
    rows = list(range(n_src)) if row_map is None else [int(r) for r in row_map]
    out = []
    for sr in rows:
        valid = [] if sr == -1 else [i for i in range(in_slots) if not mask[sr, i]]
        if not valid:
            out.append([-1] * out_slots)
            continue
        assert len(valid) <= out_slots, "more valid slots than output slots"
        out.append([sr * in_slots + valid[k] for k in pad_repeat_positions(len(valid), out_slots)])
    return out


def dedup_surfaces_survivors(surfPos: np.ndarray, thr: float):
    """dedup_surfaces_np (sample.py:159-183) that also returns, per sample, the input slot of every kept box"""
    B, S, _ = surfPos.shape
    out = np.zeros_like(surfPos)
    mask = np.ones((B, S), dtype=bool)
    slots = []
    for ii in range(B):
        bboxes = np.round(surfPos[ii].reshape(S, 2, 3), 4)
        non_repeat = bboxes[:1]
        kept = [0]
        for j, bbox in enumerate(bboxes):
            diff = np.max(np.max(np.abs(non_repeat - bbox), -1), -1)
            same = diff < thr
            diff_rev = np.max(np.max(np.abs(non_repeat - bbox[::-1]), -1), -1)
            same_rev = diff_rev < thr
            if same.sum() >= 1 or same_rev.sum() >= 1:
                continue
            non_repeat = np.concatenate([non_repeat, bbox[np.newaxis]], 0)
            kept.append(j)
        n = len(non_repeat)
        out[ii, :n] = non_repeat.reshape(n, -1)
        mask[ii, :n] = False
        slots.append(kept)
    return out, mask, slots


def strengths(source) -> list:
    s = source.strength
    return [float(v) for v in ([s] * 4 if isinstance(s, (int, float)) else s)]


def run_cascade_variation(sds, cfg, source, init_noise, step_noise, forwards=None):
    """A variation of `source` (brepgen_b200.sampler.Variation-like) under cfg.schedule "ddpm", "ddim" or "dpm".
    init_noise: name -> start noise z of each varied stage, in its starting shape; step_noise(stage, k, shape): the noise
    of step k of the stage's tail, drawn where oracle.cascade / ddim / dpm draw it.  Returns the tensors
    oracle.cascade.run_cascade returns (no decode)."""
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    S = S0 if cfg.use_cf else 2 * S0
    w = cfg.guidance_w
    st = strengths(source)
    label2 = None
    if cfg.use_cf:
        label2 = torch.tensor([cfg.class_label] * B + [0] * B).reshape(-1, 1)
    rep2 = (lambda t: torch.cat([t, t], 0)) if cfg.use_cf else (lambda t: t)
    acp = linear_alphas_cumprod()
    if cfg.schedule == "ddpm":
        sched = DDPMOracle(clip_sample=True, clip_sample_range=3.0)
        n_steps = cfg.ddpm_steps
    elif cfg.schedule == "ddim":
        sched = DDIMOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True)
        n_steps = cfg.ddim_steps
    else:
        sched = DPMOracle(solver_order=cfg.dpm_order, algorithm_type=cfg.dpm_algorithm, clip_sample=True,
                          clip_sample_range=3.0)
        n_steps = cfg.dpm_steps
    sched.set_timesteps(n_steps)
    full = sched.timesteps
    N = len(full)
    tails = {name: full[N - min(int(N * s), N):] for name, s in zip(STAGES, st)}
    eta = float(cfg.ddim_eta)
    sde = cfg.dpm_algorithm == "sde-dpmsolver++"

    def predict(fwd, x, t):
        tt = torch.tensor([int(t)])
        if cfg.use_cf:
            p = fwd(torch.cat([x, x], 0), tt)
            return p[:B] * (1 + w) - p[B:] * w
        return fwd(x, tt)

    def step(name, k, t, x, eps):
        if cfg.schedule == "ddpm":
            return sched.step(eps, int(t), x, step_noise(name, k, x.shape) if int(t) > 0 else None)
        if cfg.schedule == "ddim":
            return sched.step(eps, int(t), x, eta, noise=step_noise(name, k, x.shape) if eta > 0 else None)
        return sched.step(eps, int(t), x, noise=step_noise(name, k, x.shape) if sde else None)

    def stage(name, x, fwd, late=None):
        if cfg.schedule == "dpm":
            sched.set_timesteps(n_steps)          # an empty history: the tail's first step is first order
        for k, t in enumerate(tails[name]):
            if late is not None:
                shape = x.shape
                x = late(int(t), x)
                if x.shape != shape and cfg.schedule == "dpm":
                    sched.restart()
            x = step(name, k, t, x, predict(fwd, x, t))
        return x

    def add_noise(name, src_tokens, index, scale, shape):
        """sa*(scale*src[index]) + sb*z at the tail's first timestep; index -1: z"""
        dim = shape[-1]
        a = acp[int(tails[name][0])]
        sa, sb = a ** 0.5, (1 - a) ** 0.5
        g = torch.stack([src_tokens[i] if i >= 0 else torch.zeros(dim) for i in index]).reshape(shape)
        has = torch.tensor([i >= 0 for i in index]).reshape(shape[:-1])[..., None]
        z = init_noise[name]
        assert tuple(z.shape) == tuple(shape), (name, tuple(z.shape), shape)
        return torch.where(has, sa * (scale * g) + sb * z, z)

    if forwards is None:
        forwards = {"surfpos": lambda *a: O.surfpos_forward(sds["surfpos"], *a),
                    "surfz": lambda *a: O.surfz_forward(sds["surfz"], *a),
                    "edgepos": lambda *a: O.edgepos_forward(sds["edgepos"], *a),
                    "edgez": lambda *a: O.edgez_forward(sds["edgez"], *a)}
    F = forwards
    src = {k: getattr(source, k).detach().cpu() for k in ("surfPos", "surfMask", "surfZ", "edgePos", "edgeM", "edge_z",
                                                          "edgeV")}
    src = {k: v if v.dtype == torch.bool else v.float() for k, v in src.items()}
    thr = np.float32(cfg.bbox_threshold)

    with torch.no_grad():
        # surface positions, then the face de-duplication
        if st[0] == 0:
            surfPos, surfMask = src["surfPos"] * 3.0, src["surfMask"]
            rows = [b * S + f if not bool(surfMask[b, f]) else -1 for b in range(B) for f in range(S)]
        else:
            S1 = S0 if (not cfg.use_cf and int(tails["surfPos"][0]) > 249) else S
            fill = fill_rows(src["surfMask"].numpy(), S1)
            x = add_noise("surfPos", src["surfPos"].reshape(-1, 6), [i for r in fill for i in r], 3.0, (B, S1, 6))
            state = {"late": S1 == S}

            def late_increase(t, x):          # sample.py:140-142: double the face slots at the first t <= 249
                if not state["late"] and t <= 249:
                    state["late"] = True
                    return x.repeat(1, 2, 1)
                return x
            surfPos = stage("surfPos", x, lambda x, t: F["surfpos"](x, t, label2), late_increase)
            if not state["late"]:
                surfPos = surfPos.repeat(1, 2, 1)
            p, m, kept = dedup_surfaces_survivors(surfPos.numpy(), thr)
            surfPos, surfMask = torch.from_numpy(p), torch.from_numpy(m)
            rows = []
            for b in range(B):
                for k in range(S):
                    rows.append(fill[b][kept[b][k] % S1] if k < len(kept[b]) else -1)
        sP, sM = rep2(surfPos), rep2(surfMask)

        if st[1] == 0:
            surfZ = src["surfZ"]
        else:
            x = add_noise("surfZ", src["surfZ"].reshape(-1, 48), rows, 1.0, (B, S, 48))
            surfZ = stage("surfZ", x, lambda x, t: F["surfz"](x, t, sP, sM, label2))
        sZ = rep2(surfZ)

        if st[2] == 0:
            edgePos, edgeM = src["edgePos"] * 3.0, src["edgeM"]
            edges = list(range(B * S * E))
        else:
            edges = [i for r in fill_rows(src["edgeM"].reshape(-1, E).numpy(), E, rows) for i in r]
            x = add_noise("edgePos", src["edgePos"].reshape(-1, 6), edges, 3.0, (B, S, E, 6))
            edgePos = stage("edgePos", x, lambda x, t: F["edgepos"](x, t, sP, sZ, sM, label2))
            edgeM = torch.from_numpy(dedup_edges_np(edgePos.numpy(), surfMask.numpy(), thr))
        eP, eM = rep2(edgePos), rep2(edgeM)

        if st[3] == 0:
            edge_z, edgeV = src["edge_z"], src["edgeV"]
        else:
            zv = torch.cat([src["edge_z"], src["edgeV"]], -1).reshape(-1, 18)
            x = add_noise("edgeZV", zv, edges, 1.0, (B, S, E, 18))
            edgeZV = stage("edgeZV", x, lambda x, t: F["edgez"](x, t, eP, sP, sZ, eM, label2))
            edgeZV = edgeZV.masked_fill(edgeM.unsqueeze(-1), 0.0)
            edge_z, edgeV = edgeZV[..., :12], edgeZV[..., 12:]
    out = {"surfPos": surfPos / 3.0, "surfMask": surfMask, "surfZ": surfZ, "edgePos": edgePos / 3.0, "edgeM": edgeM,
           "edge_z": edge_z, "edgeV": edgeV}
    if st[0] == 0:
        out["surfPos"] = src["surfPos"]
    if st[2] == 0:
        out["edgePos"] = src["edgePos"]
    return out
