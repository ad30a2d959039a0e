"""ORACLE (test infrastructure): CPU fp32 restatement of diffusers 0.27 DPMSolverMultistepScheduler, and the cascade driver
of oracle/cascade.py run with N DPM-Solver++ steps per stage, with or without known tokens (B-rep completion).

diffusers 0.27 is absent from the reference and from this image (see oracle/schedulers.py).  DPMOracle restates
`scheduling_dpmsolver_multistep.py` for the configuration brepgen_b200.schedulers.DPMSolverMultistepScheduler supports
(prediction_type='epsilon', solver_order 1 or 2, algorithm_type 'dpmsolver++' or 'sde-dpmsolver++', solver_type
'midpoint', final_sigmas_type 'zero' (the product's only one; 'sigma_min' here for diffusers' known answer), timestep_spacing 'linspace' / 'leading' / 'trailing', no thresholding, no Karras or Lu
sigmas), plus the product's clip extra (clip_sample: the data prediction is clamped before it is used and stored).  Pinned
by tests/test_dpm.py: the timestep tables written out from diffusers' formulas, first order = DDIM (eta = 0), second-order
convergence on a Gaussian problem with a closed-form solution, and the full-loop answer of diffusers' own test.

run_cascade_dpm restates the driver of oracle.cascade.run_cascade (sample.py:120-299) and, with `known`, of
oracle.completion.run_cascade_completion, with each stage's loop replaced by N DPM-Solver++ steps.  The late face-count
increase (sample.py:140-142) restarts the solver: the step after the face slots are doubled is first order, because the
history holds a data prediction of the sample before the increase.
"""
from __future__ import annotations

import numpy as np
import torch

from . import denoisers as O
from .cascade import dedup_edges_np, dedup_surfaces_np
from .completion import _known_layout
from .schedulers import linear_alphas_cumprod


class DPMOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, solver_order=2,
                 algorithm_type="dpmsolver++", lower_order_final=True, euler_at_final=False, timestep_spacing="linspace",
                 steps_offset=0, final_sigmas_type="zero", clip_sample=False, clip_sample_range=1.0):
        self.n_train = num_train_timesteps
        self.acp = linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        self.order, self.algorithm = solver_order, algorithm_type
        self.lower_order_final, self.euler_at_final = lower_order_final, euler_at_final
        self.spacing, self.steps_offset = timestep_spacing, steps_offset
        self.final_sigmas_type = final_sigmas_type
        self.clip_sample, self.clip_range = clip_sample, float(clip_sample_range)
        self.set_timesteps(num_train_timesteps)

    def set_timesteps(self, n: int):
        last = self.n_train
        if self.spacing == "linspace":
            ts = np.linspace(0, last - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif self.spacing == "leading":
            ratio = last // (n + 1)
            ts = (np.arange(0, n + 1) * ratio).round()[::-1][:-1].copy().astype(np.int64) + self.steps_offset
        else:
            ts = np.arange(last, 0, -self.n_train / n).round().copy().astype(np.int64) - 1
        sig = (((1 - self.acp) / self.acp) ** 0.5).numpy()
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        last_sigma = ((1 - self.acp[0]) / self.acp[0]) ** 0.5 if self.final_sigmas_type == "sigma_min" else 0
        self.sigmas = torch.from_numpy(np.concatenate([sig, [last_sigma]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts)
        self.n_inf = len(ts)
        self.restart()
        self.step_index = None

    def restart(self):
        """empty history: the next step is first order"""
        self.model_outputs = [None] * self.order
        self.lower_order_nums = 0

    def _index(self, t):
        cand = (self.timesteps == int(t)).nonzero().flatten()
        if len(cand) == 0:
            return len(self.timesteps) - 1
        return int(cand[1] if len(cand) > 1 else cand[0])

    def _alpha_sigma(self, k):
        s = self.sigmas[k]
        a = 1 / ((s ** 2 + 1) ** 0.5)
        return a, s * a

    def abar_after(self, k):
        """abar of the level step k leaves x at, 1 / (1 + sigma_{k+1}^2)"""
        s = self.sigmas[k + 1]
        return 1.0 / (1.0 + s * s)

    def step(self, eps, t, x, noise=None):
        if self.step_index is None:
            self.step_index = self._index(t)
        k = self.step_index
        N = len(self.timesteps)
        lower_order_final = k == N - 1 and (self.euler_at_final or (self.lower_order_final and N < 15) or
                                            self.final_sigmas_type == "zero")
        alpha_s0, sigma_s0 = self._alpha_sigma(k)
        x0 = (x - sigma_s0 * eps) / alpha_s0
        if self.clip_sample:
            x0 = x0.clamp(-self.clip_range, self.clip_range)
        for i in range(self.order - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
        self.model_outputs[-1] = x0
        sde = self.algorithm == "sde-dpmsolver++"
        if sde:
            assert noise is not None, "sde-dpmsolver++ needs the step noise (diffusers draws randn on every step)"
        alpha_t, sigma_t = self._alpha_sigma(k + 1)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        if self.order == 1 or self.lower_order_nums < 1 or lower_order_final:
            if not sde:
                prev = (sigma_t / sigma_s0) * x - (alpha_t * (torch.exp(-h) - 1.0)) * x0
            else:
                prev = (sigma_t / sigma_s0 * torch.exp(-h)) * x + (alpha_t * (1 - torch.exp(-2.0 * h))) * x0 + \
                    sigma_t * torch.sqrt(1.0 - torch.exp(-2 * h)) * noise
        else:
            alpha_s1, sigma_s1 = self._alpha_sigma(k - 1)
            lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
            m0, m1 = self.model_outputs[-1], self.model_outputs[-2]
            h_0 = lambda_s0 - lambda_s1
            r0 = h_0 / h
            D0, D1 = m0, (1.0 / r0) * (m0 - m1)
            if not sde:
                prev = (sigma_t / sigma_s0) * x - (alpha_t * (torch.exp(-h) - 1.0)) * D0 - \
                    0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1
            else:
                prev = (sigma_t / sigma_s0 * torch.exp(-h)) * x + (alpha_t * (1 - torch.exp(-2.0 * h))) * D0 + \
                    0.5 * (alpha_t * (1 - torch.exp(-2.0 * h))) * D1 + \
                    sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h)) * noise
        if self.lower_order_nums < self.order:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev


def run_cascade_dpm(sds, cfg, init_noise, step_noise, forwards=None, known=None, replace_noise=None):
    """oracle.cascade.run_cascade for cfg.schedule == 'dpm': cfg.dpm_steps steps per stage of
    DPMSolverMultistepScheduler(solver_order=cfg.dpm_order, algorithm_type=cfg.dpm_algorithm, clip_sample=True,
    clip_sample_range=3); step_noise(stage, i, shape) is injected at every step i of the SDE form (diffusers draws it on
    every step).  known / replace_noise: as oracle.completion.run_cascade_completion (replacement before the first step and
    after every step, at the level 1 / (1 + sigma_next^2) the step leaves x at).  Returns the tensors run_cascade returns
    (no decode)."""
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    w = cfg.guidance_w
    sde = cfg.dpm_algorithm == "sde-dpmsolver++"
    label2 = None
    if cfg.use_cf:
        label2 = torch.tensor([cfg.class_label] * B + [0] * B).reshape(-1, 1)
    rep2 = (lambda t: torch.cat([t, t], 0)) if cfg.use_cf else (lambda t: t)
    S = S0 if cfg.use_cf else 2 * S0
    lay = _known_layout(known, cfg, S0, S) if known is not None else {}
    dpm = DPMOracle(solver_order=cfg.dpm_order, algorithm_type=cfg.dpm_algorithm, clip_sample=True, clip_sample_range=3.0)

    def predict(fwd, x, t):
        tt = torch.tensor([int(t)])
        if cfg.use_cf:
            p = fwd(torch.cat([x, x], 0), tt)
            return p[:B] * (1 + w) - p[B:] * w
        return fwd(x, tt)

    def replace(name, k, x, a):
        values, mask = lay[name][x.shape[1]]
        z = replace_noise(name, k, x.shape)
        return torch.where(mask[..., None], a ** 0.5 * values + (1 - a) ** 0.5 * z, x)

    def stage(name, x, fwd, late=None):
        dpm.set_timesteps(cfg.dpm_steps)
        kn = name in lay
        if kn:
            x = replace(name, -1, x, dpm.acp[int(dpm.timesteps[0])])
        for k, t in enumerate(dpm.timesteps):
            if late is not None:
                shape = x.shape
                x = late(int(t), x)
                if x.shape != shape:
                    dpm.restart()
            x = dpm.step(predict(fwd, x, t), int(t), x, noise=step_noise(name, k, x.shape) if sde else None)
            if kn:
                x = replace(name, k, x, dpm.abar_after(k))
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
