"""ORACLE (test infrastructure): CPU fp32 restatement of B-rep completion, the cascade driver of oracle/cascade.py ("ddpm")
and oracle/ddim.py ("ddim") with known tokens replaced before the first step and after every step of each stage.

The replacement is inpainting by replacement (no retraining): after the step at t, the tokens of the known parts are set
to sqrt(abar_prev(t)) * known + sqrt(1 - abar_prev(t)) * z, abar_prev following each scheduler's own step convention
(1 past the last step); before a stage's first step at t_first, to sqrt(abar_t_first) * known + sqrt(1 - abar_t_first) * z.
Known faces occupy slots 0..n_faces[b]-1 (both copies after the late face-count increase), their edges all E slots; the
de-duplication's edge masks of known faces are the given ones, and the known parts are returned as given.

run_cascade_completion with known=None runs the statements of oracle.cascade.run_cascade (schedule "ddpm") and
oracle.ddim.run_cascade_ddim (schedule "ddim") unchanged; tests/test_completion.py checks that it returns their outputs.
The reference has no completion, so nothing pins the completion itself beyond this restatement.
"""
from __future__ import annotations

import numpy as np
import torch

from . import denoisers as O
from .cascade import dedup_edges_np, dedup_surfaces_np
from .ddim import DDIMOracle
from .schedulers import DDPMOracle


def _known_layout(known, cfg, S0, S):
    """{stage: {slots: (values, bool token mask)}}, the face mask (B, S) and the given outputs, in model units"""
    B, E = cfg.batch_size, cfg.num_edges
    n = torch.as_tensor(known.n_faces, dtype=torch.int64).reshape(-1)
    K = known.surfPos.shape[1]

    def pad(t, slots):
        p = torch.zeros((B, slots) + tuple(t.shape[2:]), dtype=t.dtype)
        p[:, :K] = t
        return p

    def face(slots):
        return torch.arange(slots)[None, :] < n[:, None]
    f32 = lambda t: t.detach().cpu().float()
    pos = f32(known.surfPos) * 3.0
    lay = {"face": face(S), "out": {"surfPos": pad(f32(known.surfPos), S)},
           "surfPos": {S0: (pad(pos, S0), face(S0)), 2 * S0: (pad(pos, S0).repeat(1, 2, 1), face(S0).repeat(1, 2))}}
    if known.surfZ is not None:
        lay["surfZ"] = {S: (pad(f32(known.surfZ), S), face(S))}
        lay["out"]["surfZ"] = lay["surfZ"][S][0]
    if known.edgePos is not None:
        em = face(S)[..., None].expand(B, S, E)
        lay["edgePos"] = {S: (pad(f32(known.edgePos) * 3.0, S), em)}
        lay["edgeZV"] = {S: (pad(torch.cat([f32(known.edge_z), f32(known.edgeV)], -1), S), em)}
        lay["edgeM"] = pad(known.edge_mask.cpu().bool(), S)
        lay["out"].update(edgePos=pad(f32(known.edgePos), S), edgeM=lay["edgeM"], edge_z=pad(f32(known.edge_z), S),
                          edgeV=pad(f32(known.edgeV), S))
    return lay


def run_cascade_completion(sds, cfg, init_noise, step_noise, known=None, replace_noise=None, forwards=None):
    """cfg.schedule "ddpm" (cfg.ddpm_steps DDPM steps per stage) or "ddim" (cfg.ddim_steps, eta = cfg.ddim_eta) with the
    schedulers of brepgen_b200.sampler.Cascade; init_noise / step_noise / forwards as oracle.cascade.run_cascade.
    known: a brepgen_b200.sampler.Completion-like object or None; replace_noise(stage, k, shape) -> the explicit noise z
    of the replacement after step k (k = -1: before the first step).  Returns the tensors run_cascade returns (no decode)."""
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    w = cfg.guidance_w
    label2 = None
    if cfg.use_cf:
        label2 = torch.tensor([cfg.class_label] * B + [0] * B).reshape(-1, 1)
    rep2 = (lambda t: torch.cat([t, t], 0)) if cfg.use_cf else (lambda t: t)
    S = S0 if cfg.use_cf else 2 * S0
    lay = _known_layout(known, cfg, S0, S) if known is not None else {}
    if cfg.schedule == "ddim":
        sch = DDIMOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True)
        sch.set_timesteps(cfg.ddim_steps)
        final = sch.final_acp
    elif cfg.schedule == "ddpm":
        sch = DDPMOracle(clip_sample=True, clip_sample_range=3.0)
        sch.set_timesteps(cfg.ddpm_steps)
        final = torch.tensor(1.0)
    else:
        raise NotImplementedError("the completion oracle restates the 'ddpm' and 'ddim' schedules")
    eta = float(cfg.ddim_eta)

    def predict(fwd, x, t):
        tt = torch.tensor([int(t)])
        if cfg.use_cf:
            p = fwd(torch.cat([x, x], 0), tt)
            return p[:B] * (1 + w) - p[B:] * w
        return fwd(x, tt)

    def step(name, k, t, x, eps):
        if cfg.schedule == "ddim":
            return sch.step(eps, t, x, eta, noise=step_noise(name, k, x.shape) if eta > 0 else None)
        return sch.step(eps, t, x, step_noise(name, k, x.shape) if t > 0 else None)

    def replace(name, k, t, x, initial=False):
        values, mask = lay[name][x.shape[1]]
        if initial:
            a = sch.acp[t]
        else:
            prev_t = t - sch.n_train // sch.n_inf
            a = sch.acp[prev_t] if prev_t >= 0 else final
        z = replace_noise(name, k, x.shape)
        return torch.where(mask[..., None], a ** 0.5 * values + (1 - a) ** 0.5 * z, x)

    def stage(name, x, fwd, late=None):
        kn = name in lay
        if kn:
            x = replace(name, -1, int(sch.timesteps[0]), x, initial=True)
        for k, t in enumerate(sch.timesteps):
            t = int(t)
            if late is not None:
                x = late(t, x)
            x = step(name, k, t, x, predict(fwd, x, t))
            if kn:
                x = replace(name, k, t, x)
        return x

    state = {"late": cfg.use_cf}

    def late_increase(t, x):          # sample.py:140-142: double the face slots at the first t <= 249
        if not state["late"] and t <= 249:
            state["late"] = True
            return x.repeat(1, 2, 1)
        return x

    if forwards is None:
        forwards = {"surfpos": lambda *a: O.surfpos_forward(sds["surfpos"], *a),
                    "surfz": lambda *a: O.surfz_forward(sds["surfz"], *a),
                    "edgepos": lambda *a: O.edgepos_forward(sds["edgepos"], *a),
                    "edgez": lambda *a: O.edgez_forward(sds["edgez"], *a)}
    F = forwards

    with torch.no_grad():
        surfPos = stage("surfPos", init_noise["surfPos"].clone(), lambda x, t: F["surfpos"](x, t, label2), late_increase)
        if not state["late"]:
            surfPos = surfPos.repeat(1, 2, 1)
        if cfg.dense_masks:
            surfMask = torch.zeros(B, S, dtype=torch.bool)
        else:
            p, m = dedup_surfaces_np(surfPos.numpy(), np.float32(cfg.bbox_threshold))
            surfPos, surfMask = torch.from_numpy(p), torch.from_numpy(m)
        sP, sM = rep2(surfPos), rep2(surfMask)
        surfZ = stage("surfZ", init_noise["surfZ"].clone(), lambda x, t: F["surfz"](x, t, sP, sM, label2))
        sZ = rep2(surfZ)
        edgePos = stage("edgePos", init_noise["edgePos"].clone(), lambda x, t: F["edgepos"](x, t, sP, sZ, sM, label2))
        if cfg.dense_masks:
            edgeM = torch.zeros(B, S, E, dtype=torch.bool)
        else:
            edgeM = torch.from_numpy(dedup_edges_np(edgePos.numpy(), surfMask.numpy(), np.float32(cfg.bbox_threshold)))
        if "edgeM" in lay:
            edgeM = torch.where(lay["face"][..., None], lay["edgeM"], edgeM)
        eP, eM = rep2(edgePos), rep2(edgeM)
        edgeZV = stage("edgeZV", init_noise["edgeZV"].clone(), lambda x, t: F["edgez"](x, t, eP, sP, sZ, eM, label2))
        edgeZV = edgeZV.masked_fill(edgeM.unsqueeze(-1), 0.0)
    out = {"surfPos": surfPos / 3.0, "surfMask": surfMask, "surfZ": surfZ, "edgePos": edgePos / 3.0, "edgeM": edgeM,
           "edge_z": edgeZV[..., :12], "edgeV": edgeZV[..., 12:]}
    for k, v in lay.get("out", {}).items():
        out[k] = torch.where(lay["face"].reshape(lay["face"].shape + (1,) * (v.dim() - 2)), v, out[k])
    return out
