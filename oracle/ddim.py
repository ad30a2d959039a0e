"""ORACLE (test infrastructure): CPU fp32 restatement of diffusers 0.27 DDIMScheduler, and the cascade driver of
oracle/cascade.py run with N DDIM steps per stage.

diffusers 0.27 is absent from the reference and from this image (see oracle/schedulers.py).  DDIMOracle restates
`scheduling_ddim.py` for the configuration brepgen_b200.schedulers.DDIMScheduler supports (prediction_type='epsilon',
timestep_spacing='leading', no thresholding).  PINNED by the known answers of diffusers' tests/schedulers/
test_scheduler_ddim.py full loops (tests/test_ddim.py).

run_cascade_ddim restates the same driver as oracle.cascade.run_cascade (sample.py:120-299: stage order, late face-count
increase, CFG combine, de-duplication, final masking) with the DDPM loop of each stage replaced by N DDIM steps.  The
reference has no DDIM schedule, so the driver part is pinned only through oracle.cascade (driver_golden.npz); the DDIM
steps through DDIMOracle.
"""
from __future__ import annotations

import numpy as np
import torch

from . import denoisers as O
from .cascade import dedup_edges_np, dedup_surfaces_np
from .schedulers import linear_alphas_cumprod


class DDIMOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, clip_sample=True, clip_sample_range=1.0,
                 set_alpha_to_one=True, steps_offset=0):
        self.n_train = num_train_timesteps
        self.acp = linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        self.final_acp = torch.tensor(1.0) if set_alpha_to_one else self.acp[0]
        self.clip_sample, self.clip_range = clip_sample, float(clip_sample_range)
        self.steps_offset = steps_offset
        self.set_timesteps(num_train_timesteps)

    def set_timesteps(self, n: int):
        self.n_inf = n
        ratio = self.n_train // n
        ts = (np.arange(0, n) * ratio).round()[::-1].copy().astype(np.int64) + self.steps_offset
        self.timesteps = torch.from_numpy(ts)

    def coeffs(self, t: int, eta: float = 0.0):
        """(sqrt(1-abar_t), sqrt(abar_t), sqrt(abar_prev), c_dir, sigma) as fp32 torch scalars"""
        prev_t = t - self.n_train // self.n_inf
        a_t = self.acp[t]
        a_prev = self.acp[prev_t] if prev_t >= 0 else self.final_acp
        b_t = 1 - a_t
        variance = ((1 - a_prev) / b_t) * (1 - a_t / a_prev)
        std_dev_t = eta * variance ** 0.5
        return b_t ** 0.5, a_t ** 0.5, a_prev ** 0.5, (1 - a_prev - std_dev_t ** 2) ** 0.5, std_dev_t

    def step(self, eps, t, x, eta: float = 0.0, use_clipped_model_output: bool = False, noise=None):
        sb, sa, sa_prev, c_dir, sigma = self.coeffs(int(t), eta)
        x0 = (x - sb * eps) / sa
        if self.clip_sample:
            x0 = x0.clamp(-self.clip_range, self.clip_range)
        if use_clipped_model_output:
            eps = (x - sa * x0) / sb
        prev = sa_prev * x0 + c_dir * eps
        if eta > 0:
            assert noise is not None, "eta > 0 needs the step noise (diffusers draws randn of eps.shape on every step)"
            prev = prev + sigma * noise
        return prev


def run_cascade_ddim(sds, cfg, init_noise, step_noise, forwards=None):
    """oracle.cascade.run_cascade for cfg.schedule == 'ddim': cfg.ddim_steps DDIM steps (eta = cfg.ddim_eta) per stage with
    DDIMScheduler(clip_sample=True, clip_sample_range=3, set_alpha_to_one=True); step_noise(stage, i, shape) is injected
    at every step i when eta > 0 (diffusers draws it on every step).  Returns the tensors run_cascade returns (no decode)."""
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    w = cfg.guidance_w
    eta = float(cfg.ddim_eta)
    label2 = None
    if cfg.use_cf:
        label2 = torch.tensor([cfg.class_label] * B + [0] * B).reshape(-1, 1)
    rep2 = (lambda t: torch.cat([t, t], 0)) if cfg.use_cf else (lambda t: t)
    ddim = DDIMOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True)
    ddim.set_timesteps(cfg.ddim_steps)

    def predict(fwd, x, t):
        tt = torch.tensor([int(t)])
        if cfg.use_cf:
            p = fwd(torch.cat([x, x], 0), tt)
            return p[:B] * (1 + w) - p[B:] * w
        return fwd(x, tt)

    def stage(name, x, fwd, late=None):
        for k, t in enumerate(ddim.timesteps):
            if late is not None:
                x = late(int(t), x)
            x = ddim.step(predict(fwd, x, t), int(t), x, eta, noise=step_noise(name, k, x.shape) if eta > 0 else None)
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
        S = surfPos.shape[1]
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
        eP, eM = rep2(edgePos), rep2(edgeM)
        edgeZV = stage("edgeZV", init_noise["edgeZV"].clone(), lambda x, t: F["edgez"](x, t, eP, sP, sZ, eM, label2))
        edgeZV = edgeZV.masked_fill(edgeM.unsqueeze(-1), 0.0)
    return {"surfPos": surfPos / 3.0, "surfMask": surfMask, "surfZ": surfZ, "edgePos": edgePos / 3.0, "edgeM": edgeM,
            "edge_z": edgeZV[..., :12], "edgeV": edgeZV[..., 12:]}
