"""ORACLE (test infrastructure): CPU fp32 restatement of diffusers 0.27 RePaintScheduler (scheduling_repaint.py) and of
the RePaint loop of pipeline_repaint.py, and the cascade driver run with a RePaint list per stage.

diffusers is absent from this image (see oracle/schedulers.py).  RePaintOracle restates set_timesteps, step and
undo_step for epsilon prediction; the one change is the clip range (clip_sample_range, diffusers clips to +-1; the
cascade clips to +-3 as its other schedulers do).  The statements are pinned by equivalence to parts that are pinned
already (tests/test_repaint.py): with jump_n_sample = 1 the list is DDIMOracle's, a step with nothing known is
DDIMOracle.step, and the cascade runner with jump_n_sample = 1, eta = 0 and nothing known returns
oracle.ddim.run_cascade_ddim's outputs.

run_cascade_repaint restates the cascade driver (stage order, late face-count increase, CFG combine, de-duplication,
final masking; oracle/cascade.py) with each stage's loop replaced by the RePaint loop, and the known parts of a completion
laid out as oracle/completion.py lays them out.  Without trained weights nothing here says whether resampling improves a
completion; only the arithmetic and the invariants are pinned.
"""
from __future__ import annotations

import numpy as np
import torch

from . import denoisers as O
from .cascade import dedup_edges_np, dedup_surfaces_np
from .completion import _known_layout


class RePaintOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, eta=0.0, clip_sample=True,
                 clip_sample_range=1.0):
        self.n_train = num_train_timesteps
        self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.acp = torch.cumprod(1.0 - self.betas, dim=0)
        self.final_acp = torch.tensor(1.0)
        self.eta = float(eta)
        self.clip_sample, self.clip_range = clip_sample, float(clip_sample_range)

    def set_timesteps(self, n: int, jump_length: int = 10, jump_n_sample: int = 10):
        n = min(self.n_train, n)
        self.n_inf = n
        timesteps = []
        jumps = {}
        for j in range(0, n - jump_length, jump_length):
            jumps[j] = jump_n_sample - 1
        t = n
        while t >= 1:
            t = t - 1
            timesteps.append(t)
            if jumps.get(t, 0) > 0:
                jumps[t] = jumps[t] - 1
                for _ in range(jump_length):
                    t = t + 1
                    timesteps.append(t)
        self.timesteps = torch.from_numpy(np.array(timesteps) * (self.n_train // n))

    def _variance(self, t):
        prev_t = t - self.n_train // self.n_inf
        a_t = self.acp[t]
        a_prev = self.acp[prev_t] if prev_t >= 0 else self.final_acp
        return ((1 - a_prev) / (1 - a_t)) * (1 - a_t / a_prev)

    def step(self, eps, t, x, original, mask, noise):
        """mask: float 0/1 broadcastable to x (1 = known), or None with original None (nothing known); noise: the one z"""
        t = int(t)
        prev_t = t - self.n_train // self.n_inf
        a_t = self.acp[t]
        a_prev = self.acp[prev_t] if prev_t >= 0 else self.final_acp
        b_t = 1 - a_t
        x0 = (x - b_t ** 0.5 * eps) / a_t ** 0.5
        if self.clip_sample:
            x0 = torch.clamp(x0, -self.clip_range, self.clip_range)
        std_dev_t = self.eta * self._variance(t) ** 0.5
        variance = 0
        if t > 0 and self.eta > 0:
            variance = std_dev_t * noise
        direction = (1 - a_prev - std_dev_t ** 2) ** 0.5 * eps
        unknown = a_prev ** 0.5 * x0 + direction + variance
        if mask is None:
            return unknown
        known = (a_prev ** 0.5) * original + ((1 - a_prev) ** 0.5) * noise
        return mask * known + (1.0 - mask) * unknown

    def undo_step(self, x, t_last, noise):
        """noise: (n, *x.shape), one normal tensor per transition"""
        n = self.n_train // self.n_inf
        for i in range(n):
            beta = self.betas[int(t_last) + i]
            x = (1 - beta) ** 0.5 * x + beta ** 0.5 * noise[i]
        return x


def run_cascade_repaint(sds, cfg, init_noise, step_noise, undo_noise, known=None, forwards=None):
    """cfg.schedule "repaint": per stage the RePaint list of set_timesteps(cfg.repaint_steps, cfg.repaint_jump_length,
    cfg.repaint_jump_n_sample) with eta = cfg.repaint_eta, clip +-3.  step_noise(stage, k, shape) -> the z of the step at
    list entry k (drawn at every step); undo_noise(stage, k, (n, *shape)) -> the normals of the undo at entry k.
    known: a brepgen_b200.sampler.Completion-like object or None.  init_noise / forwards as oracle.cascade.run_cascade.
    Returns the tensors run_cascade returns (no decode)."""
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    w = cfg.guidance_w
    label2 = None
    if cfg.use_cf:
        label2 = torch.tensor([cfg.class_label] * B + [0] * B).reshape(-1, 1)
    rep2 = (lambda t: torch.cat([t, t], 0)) if cfg.use_cf else (lambda t: t)
    S = S0 if cfg.use_cf else 2 * S0
    lay = _known_layout(known, cfg, S0, S) if known is not None else {}
    sch = RePaintOracle(eta=cfg.repaint_eta, clip_sample=True, clip_sample_range=3.0)
    sch.set_timesteps(cfg.repaint_steps, cfg.repaint_jump_length, cfg.repaint_jump_n_sample)
    n_undo = sch.n_train // sch.n_inf

    def predict(fwd, x, t):
        tt = torch.tensor([int(t)])
        if cfg.use_cf:
            p = fwd(torch.cat([x, x], 0), tt)
            return p[:B] * (1 + w) - p[B:] * w
        return fwd(x, tt)

    def stage(name, x, fwd, late=None):
        t_last = int(sch.timesteps[0]) + 1
        for k, t in enumerate(sch.timesteps):
            t = int(t)
            if late is not None:
                x = late(t, x)
            if t < t_last:
                original = mask = None
                if name in lay:
                    original, m = lay[name][x.shape[1]]
                    mask = m[..., None].float()
                x = sch.step(predict(fwd, x, t), t, x, original, mask, step_noise(name, k, x.shape))
            else:
                x = sch.undo_step(x, t_last, undo_noise(name, k, (n_undo,) + tuple(x.shape)))
            t_last = t
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
