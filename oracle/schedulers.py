"""ORACLE (test infrastructure): CPU restatement of diffusers 0.27 DDPMScheduler / PNDMScheduler arithmetic.

diffusers==0.27 (requirements.txt:5 of the reference) is a third-party dependency that is absent from the reference and
from this image, so its code cannot be executed here and the reference itself holds no golden vector for it.
PINNED by the known answers of diffusers' own scheduler tests (tests/test_oracle_sched_kat.py): the full 1000-step DDPM
loop with injected noise (|x| sum 258.9606) and the PRK + PLMS loops of PNDM (198.1318; beta_start = 0.01: 186.9482) over the
deterministic dummy model of tests/schedulers/test_scheduler_{ddpm,pndm}.py are reproduced to diffusers' own tolerances.
Further anchors: the reference's call sites
  ctor kwargs           sample.py:101-117 (PNDM: linear betas 1e-4..0.02, epsilon; DDPM: + clip_sample, range 3)
  set_timesteps(200)    sample.py:128,191,210,269   -> 209 PNDM entries, [:158] ends 255 -> 250
  set_timesteps(1000)   sample.py:144,224           -> [-250:] starts at t=249
  step(pred,t,x).prev_sample   sample.py:137,153,202,222,236,282
  add_noise             trainer.py:348 etc.
and structural invariants (tests/test_host_logic.py): x0-recovery, posterior-mean identity, DDIM identity for PNDM's
transfer formula, PRK/PLMS table shape.
"""
from __future__ import annotations

import numpy as np
import torch


def linear_alphas_cumprod(n: int = 1000, beta_start: float = 1e-4, beta_end: float = 0.02) -> torch.Tensor:
    betas = torch.linspace(beta_start, beta_end, n, dtype=torch.float32)
    return torch.cumprod(1.0 - betas, dim=0)


class DDPMOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, clip_sample=True,
                 clip_sample_range=3.0):
        self.n_train = num_train_timesteps
        self.acp = linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        self.clip_sample, self.clip_range = clip_sample, float(clip_sample_range)
        self.set_timesteps(num_train_timesteps)

    def set_timesteps(self, n: int):
        self.n_inf = n
        ratio = self.n_train // n
        self.timesteps = torch.from_numpy((np.arange(0, n) * ratio).round()[::-1].copy().astype(np.int64))

    def coeffs(self, t: int):
        """(sqrt(1-abar_t), 1/sqrt(abar_t) as divisor abar_t**0.5, c_x0, c_x, sigma) as fp32 torch scalars."""
        prev_t = t - self.n_train // self.n_inf
        a_t = self.acp[t]
        a_prev = self.acp[prev_t] if prev_t >= 0 else torch.tensor(1.0)
        b_t, b_prev = 1 - a_t, 1 - a_prev
        cur_alpha = a_t / a_prev
        cur_beta = 1 - cur_alpha
        c_x0 = (a_prev ** 0.5 * cur_beta) / b_t
        c_x = cur_alpha ** 0.5 * b_prev / b_t
        var = torch.clamp(b_prev / b_t * cur_beta, min=1e-20)
        sigma = var ** 0.5 if t > 0 else torch.tensor(0.0)
        return b_t ** 0.5, a_t ** 0.5, c_x0, c_x, sigma

    def step(self, eps: torch.Tensor, t: int, x: torch.Tensor, noise: torch.Tensor | None = None) -> torch.Tensor:
        t = int(t)
        sb, sa, c_x0, c_x, sigma = self.coeffs(t)
        x0 = (x - sb * eps) / sa
        if self.clip_sample:
            x0 = x0.clamp(-self.clip_range, self.clip_range)
        prev = c_x0 * x0 + c_x * x
        if t > 0:
            assert noise is not None, "t>0 needs the step noise (diffusers draws randn of eps.shape)"
            prev = prev + sigma * noise
        return prev

    def add_noise(self, x0, noise, t):
        a = self.acp[t].to(x0.dtype)
        while a.dim() < x0.dim():
            a = a.unsqueeze(-1)
        return a ** 0.5 * x0 + (1 - a) ** 0.5 * noise


class PNDMOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02):
        self.n_train = num_train_timesteps
        self.acp = linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        self.final_acp = self.acp[0]          # set_alpha_to_one=False
        self.order = 4
        self.set_timesteps(num_train_timesteps)

    def set_timesteps(self, n: int):
        self.n_inf = n
        ratio = self.n_train // n
        _t = (np.arange(0, n) * ratio).round().astype(np.int64)     # steps_offset = 0
        prk = np.array(_t[-self.order:]).repeat(2) + np.tile(np.array([0, ratio // 2]), self.order)
        self.prk = (prk[:-1].repeat(2)[1:-1])[::-1].copy()
        self.plms = _t[:-3][::-1].copy()
        self.timesteps = torch.from_numpy(np.concatenate([self.prk, self.plms]).astype(np.int64))
        self.ets, self.counter, self.cur_model_output, self.cur_sample = [], 0, 0, None

    def _prev_sample(self, x, t, prev_t, eps):
        a_t = self.acp[t]
        a_p = self.acp[prev_t] if prev_t >= 0 else self.final_acp
        b_t, b_p = 1 - a_t, 1 - a_p
        sample_coeff = (a_p / a_t) ** 0.5
        denom = a_t * b_p ** 0.5 + (a_t * b_t * a_p) ** 0.5
        return sample_coeff * x - (a_p - a_t) * eps / denom

    def step(self, eps, t, x):
        t = int(t)
        if self.counter < len(self.prk):
            return self._step_prk(eps, t, x)
        return self._step_plms(eps, t, x)

    def _step_prk(self, eps, t, x):
        ratio = self.n_train // self.n_inf
        diff = 0 if self.counter % 2 else ratio // 2
        prev_t = t - diff
        t = int(self.prk[self.counter // 4 * 4])
        r = self.counter % 4
        if r == 0:
            self.cur_model_output = self.cur_model_output + eps / 6
            self.ets.append(eps)
            self.cur_sample = x
        elif r == 1:
            self.cur_model_output = self.cur_model_output + eps / 3
        elif r == 2:
            self.cur_model_output = self.cur_model_output + eps / 3
        else:
            eps = self.cur_model_output + eps / 6
            self.cur_model_output = 0
        out = self._prev_sample(self.cur_sample, t, prev_t, eps)
        self.counter += 1
        return out

    def _step_plms(self, eps, t, x):
        prev_t = t - self.n_train // self.n_inf
        self.ets = self.ets[-3:] + [eps]
        e = self.ets
        if len(e) == 1:
            eps = e[-1]
        elif len(e) == 2:
            eps = (3 * e[-1] - e[-2]) / 2
        elif len(e) == 3:
            eps = (23 * e[-1] - 16 * e[-2] + 5 * e[-3]) / 12
        else:
            eps = (1 / 24) * (55 * e[-1] - 59 * e[-2] + 37 * e[-3] - 9 * e[-4])
        out = self._prev_sample(x, t, prev_t, eps)
        self.counter += 1
        return out
