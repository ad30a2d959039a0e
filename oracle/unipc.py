"""ORACLE (test infrastructure): CPU fp32 restatement of diffusers' UniPCMultistepScheduler (Zhao et al. 2023, UniPC), and
the cascade drivers of oracle/dpm.py and oracle/variation.py run with it.

diffusers is absent from the reference and from this image (see oracle/schedulers.py).  UniPCOracle restates
`scheduling_unipc_multistep.py` (0.27, plus the later final_sigmas_type) for the configuration
brepgen_b200.schedulers.UniPCMultistepScheduler supports: predict_x0=True, prediction_type 'epsilon', solver_order 1-3,
solver_type 'bh1' / 'bh2', lower_order_final, disable_corrector, timestep_spacing 'linspace' / 'leading' / 'trailing',
final_sigmas_type 'sigma_min' (0.27's only behaviour) or 'zero', no thresholding, Karras sigmas or solver_p; plus the
product's clip extra (clip_sample: the data prediction is clamped before it is used and stored).  Every tensor expression
is diffusers', in its order.  One departure: a first-order predictor into sigma = 0 is x0 (the limit of the expression,
whose B(h) * 0 term diffusers evaluates as inf * 0 under bh1).  Pinned by tests/test_unipc.py: diffusers' published
full-loop answer, the timestep tables, order 1 = DDIM (eta = 0), order 2 bh2 without corrector = DPM-Solver++ 2M.

run_cascade_unipc and run_cascade_variation_unipc run the drivers of oracle/dpm.py and oracle/variation.py unchanged,
with UniPCOracle in place of DPMOracle: both call set_timesteps at a stage's start (an empty history), restart() at the
late face-count increase, step(eps, t, x) and abar_after(k), which UniPCOracle provides with the same meaning.
"""
from __future__ import annotations

import contextlib
from dataclasses import replace

import numpy as np
import torch

from . import dpm as _dpm
from . import variation as _variation
from .schedulers import linear_alphas_cumprod


class UniPCOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, solver_order=2, solver_type="bh2",
                 lower_order_final=True, disable_corrector=(), timestep_spacing="linspace", steps_offset=0,
                 final_sigmas_type="sigma_min", clip_sample=False, clip_sample_range=1.0):
        self.n_train = num_train_timesteps
        self.acp = linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        self.order, self.solver_type = solver_order, solver_type
        self.lower_order_final = lower_order_final
        self.disable_corrector = list(disable_corrector)
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
        if self.final_sigmas_type == "sigma_min":
            sigma_last = ((1 - self.acp[0]) / self.acp[0]) ** 0.5
        else:
            sigma_last = 0
        self.sigmas = torch.from_numpy(np.concatenate([sig, [sigma_last]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts)
        self.n_inf = len(ts)
        self.restart()
        self.step_index = None

    def restart(self):
        """empty history and no last_sample: the next step is first order without a corrector"""
        self.model_outputs = [None] * self.order
        self.lower_order_nums = 0
        self.last_sample = None
        self.this_order = None

    def _index(self, t):
        cand = (self.timesteps == int(t)).nonzero().flatten()
        if len(cand) == 0:
            return len(self.timesteps) - 1
        return int(cand[1] if len(cand) > 1 else cand[0])

    def _alpha_sigma(self, k):
        s = self.sigmas[k]
        a = 1 / ((s ** 2 + 1) ** 0.5)
        return a, s * a

    def _lambda(self, k):
        a, s = self._alpha_sigma(k)
        return torch.log(a) - torch.log(s)

    def abar_after(self, k):
        """abar of the level step k leaves x at, 1 / (1 + sigma_{k+1}^2)"""
        s = self.sigmas[k + 1]
        return 1.0 / (1.0 + s * s)

    def _rb(self, h, rks, order):
        """diffusers' R and b (the h_phi_k / factorial recursion) and B(h)"""
        hh = -h
        h_phi_1 = torch.expm1(hh)
        h_phi_k = h_phi_1 / hh - 1
        factorial_i = 1
        B_h = hh if self.solver_type == "bh1" else torch.expm1(hh)
        R, b = [], []
        for i in range(1, order + 1):
            R.append(torch.pow(rks, i - 1))
            b.append(h_phi_k * factorial_i / B_h)
            factorial_i *= i + 1
            h_phi_k = h_phi_k / hh - 1 / factorial_i
        return torch.stack(R), torch.tensor(b), h_phi_1, B_h

    def predictor(self, x, order):
        """multistep_uni_p_bh_update (predict_x0)"""
        k = self.step_index
        m0 = self.model_outputs[-1]
        alpha_t, sigma_t = self._alpha_sigma(k + 1)
        alpha_s0, sigma_s0 = self._alpha_sigma(k)
        lambda_s0 = self._lambda(k)
        h = self._lambda(k + 1) - lambda_s0
        rks, D1s = [], []
        for i in range(1, order):
            mi = self.model_outputs[-(i + 1)]
            rk = (self._lambda(k - i) - lambda_s0) / h
            rks.append(rk)
            D1s.append((mi - m0) / rk)
        rks.append(1.0)
        R, b, h_phi_1, B_h = self._rb(h, torch.tensor(rks), order)
        x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
        if not D1s:
            return x_t_                   # diffusers subtracts alpha_t * B_h * 0: the limit, finite under bh1 too
        rhos_p = torch.tensor([0.5]) if order == 2 else torch.linalg.solve(R[:-1, :-1], b[:-1])
        pred_res = torch.einsum("k,bk...->b...", rhos_p, torch.stack(D1s, dim=1))
        return x_t_ - alpha_t * B_h * pred_res

    def corrector(self, model_t, last_sample, order):
        """multistep_uni_c_bh_update (predict_x0), before the history shift"""
        k = self.step_index
        m0 = self.model_outputs[-1]
        alpha_t, sigma_t = self._alpha_sigma(k)
        alpha_s0, sigma_s0 = self._alpha_sigma(k - 1)
        lambda_s0 = self._lambda(k - 1)
        h = self._lambda(k) - lambda_s0
        rks, D1s = [], []
        for i in range(1, order):
            mi = self.model_outputs[-(i + 1)]
            rk = (self._lambda(k - (i + 1)) - lambda_s0) / h
            rks.append(rk)
            D1s.append((mi - m0) / rk)
        rks.append(1.0)
        R, b, h_phi_1, B_h = self._rb(h, torch.tensor(rks), order)
        rhos_c = torch.tensor([0.5]) if order == 1 else torch.linalg.solve(R, b)
        x_t_ = sigma_t / sigma_s0 * last_sample - alpha_t * h_phi_1 * m0
        corr_res = torch.einsum("k,bk...->b...", rhos_c[:-1], torch.stack(D1s, dim=1)) if D1s else 0
        D1_t = model_t - m0
        return x_t_ - alpha_t * B_h * (corr_res + rhos_c[-1] * D1_t)

    def step(self, eps, t, x, noise=None):
        if self.step_index is None:
            self.step_index = self._index(t)
        k = self.step_index
        alpha_s, sigma_s = self._alpha_sigma(k)
        x0 = (x - sigma_s * eps) / alpha_s
        if self.clip_sample:
            x0 = x0.clamp(-self.clip_range, self.clip_range)
        if k > 0 and (k - 1) not in self.disable_corrector and self.last_sample is not None:
            x = self.corrector(x0, self.last_sample, self.this_order)
        for i in range(self.order - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
        self.model_outputs[-1] = x0
        order = min(self.order, len(self.timesteps) - k) if self.lower_order_final else self.order
        self.this_order = min(order, self.lower_order_nums + 1)
        self.last_sample = x
        prev = self.predictor(x, self.this_order)
        if self.lower_order_nums < self.order:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev


def _factory(cfg):
    """UniPCOracle built where the drivers build DPMOracle, with the cascade's settings"""
    return lambda **_: UniPCOracle(solver_order=cfg.unipc_order, solver_type=cfg.unipc_solver_type,
                                   final_sigmas_type="zero", clip_sample=True, clip_sample_range=3.0)


@contextlib.contextmanager
def _as_dpm(module, cfg):
    saved = module.DPMOracle
    module.DPMOracle = _factory(cfg)
    try:
        yield replace(cfg, schedule="dpm", dpm_steps=cfg.unipc_steps, dpm_algorithm="dpmsolver++")
    finally:
        module.DPMOracle = saved


def run_cascade_unipc(sds, cfg, init_noise, forwards=None, known=None, replace_noise=None):
    """oracle.dpm.run_cascade_dpm for cfg.schedule == 'unipc': cfg.unipc_steps UniPC steps per stage of
    UniPCMultistepScheduler(solver_order=cfg.unipc_order, solver_type=cfg.unipc_solver_type, final_sigmas_type='zero',
    clip_sample=True, clip_sample_range=3); no step noise.  The late face-count increase restarts the solver (first
    order, no corrector).  known / replace_noise: as run_cascade_dpm."""
    with _as_dpm(_dpm, cfg) as c:
        return _dpm.run_cascade_dpm(sds, c, init_noise, None, forwards, known, replace_noise)


def run_cascade_variation_unipc(sds, cfg, source, init_noise, forwards=None):
    """oracle.variation.run_cascade_variation for cfg.schedule == 'unipc': each varied stage runs the tail of the UniPC
    list from an empty history (its first step first order, without a corrector)"""
    with _as_dpm(_variation, cfg) as c:
        return _variation.run_cascade_variation(sds, c, source, init_noise, None, forwards)
