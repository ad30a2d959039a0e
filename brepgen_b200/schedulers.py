"""Drop-in DDPMScheduler / PNDMScheduler with the diffusers 0.27 interface used by the reference.

Call sites mirrored (all in the reference): constructors sample.py:101-117 and trainer.py:285-292;
`set_timesteps(n)` + `.timesteps[...]` slicing sample.py:128-129,144-145; `.step(pred, t, x).prev_sample`
sample.py:137,153,202,222,236,282; `.add_noise(x, noise, t)` trainer.py:348; `.config.num_train_timesteps` trainer.py:330.

Host side (this file): the beta / alphas_cumprod tables and the per-step scalar coefficients, computed with the same
fp32 torch-CPU operations diffusers uses (SURVEY.md Appendix A.3/A.4).  Device side: ONE fused kernel per step
(bg_ddpm_step / bg_pndm_step in csrc/sched.cu) instead of ~15 scalar-broadcast launches.  No CPU tensor path:
`step` on a CPU sample raises.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch

from . import _ffi


class SchedulerOutput:
    def __init__(self, prev_sample: torch.Tensor, pred_original_sample: Optional[torch.Tensor] = None):
        self.prev_sample = prev_sample
        self.pred_original_sample = pred_original_sample

    def __iter__(self):   # diffusers' return_dict=False tuple form
        yield self.prev_sample


def _betas(num_train_timesteps, beta_start, beta_end, beta_schedule):
    if beta_schedule == "linear":
        return torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    if beta_schedule == "scaled_linear":
        return torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    raise NotImplementedError(f"beta_schedule={beta_schedule!r} (the reference uses 'linear', sample.py:103,111)")


def mix_seed(*parts: int) -> int:
    """64-bit key from a tuple of integers (splitmix64 finaliser per part): distinct tuples -> independent Philox keys"""
    h = 0x9E3779B97F4A7C15
    for p in parts:
        z = (h ^ (int(p) & 0xFFFFFFFFFFFFFFFF)) + 0x9E3779B97F4A7C15 & 0xFFFFFFFFFFFFFFFF
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
        h = z ^ (z >> 31)
    return h


def _as_int(t) -> int:
    return int(t.item()) if torch.is_tensor(t) else int(t)


def _require_cuda(x: torch.Tensor, what: str):
    if not x.is_cuda:
        raise RuntimeError(f"brepgen_b200 schedulers have no CPU path: {what} must be a CUDA tensor")


class DDPMScheduler:
    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", prediction_type: str = "epsilon", clip_sample: bool = True,
                 clip_sample_range: float = 1.0, variance_type: str = "fixed_small", **unused):
        if prediction_type != "epsilon" or variance_type != "fixed_small":
            raise NotImplementedError("only prediction_type='epsilon', variance_type='fixed_small' (sample.py:109-117)")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, prediction_type=prediction_type,
                                      clip_sample=clip_sample, clip_sample_range=clip_sample_range,
                                      variance_type=variance_type)
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.one = torch.tensor(1.0)
        self.init_noise_sigma = 1.0
        self._philox_seed = None       # None: derived from torch.initial_seed() at first use (follows torch.manual_seed)
        self._philox_offset = 0
        self.set_timesteps(num_train_timesteps)

    def set_noise_seed(self, seed: int, *stream: int):
        """Key of the in-kernel Philox stream that `step` draws its noise from when neither `noise` nor `generator` is
        given: a 64-bit mix of `seed` and any further integers (rank, stage, ...).  Resets the stream offset, so a run is
        reproducible from the seed alone and different (seed, rank, stage) tuples give independent streams
        (SURVEY.md 8(e): per-rank independent RNG streams)."""
        self._philox_seed = mix_seed(seed, *stream)
        self._philox_offset = 0

    def set_timesteps(self, num_inference_steps: int, device=None):
        n_train = self.config.num_train_timesteps
        if num_inference_steps > n_train:
            raise ValueError("num_inference_steps cannot exceed num_train_timesteps")
        self.num_inference_steps = num_inference_steps
        ratio = n_train // num_inference_steps                      # timestep_spacing = "leading"
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(ts)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step_coefficients(self, t: int):
        """(sqrt(1-abar_t), sqrt(abar_t), c_x0, c_x, sigma) as Python floats (fp32 arithmetic like diffusers)."""
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one
        b_t, b_prev = 1 - a_t, 1 - a_prev
        cur_alpha = a_t / a_prev
        cur_beta = 1 - cur_alpha
        c_x0 = (a_prev ** 0.5 * cur_beta) / b_t
        c_x = cur_alpha ** 0.5 * b_prev / b_t
        sigma = 0.0
        if t > 0:
            sigma = float(torch.clamp(b_prev / b_t * cur_beta, min=1e-20) ** 0.5)
        return float(b_t ** 0.5), float(a_t ** 0.5), float(c_x0), float(c_x), sigma

    def coefficient_table(self, timesteps) -> torch.Tensor:
        """[len(timesteps), 5] fp32 (CPU): step_coefficients(t) for every t of a denoising loop -- the device table that
        bg_ddpm_step_tab indexes with its step counter when the loop is captured in a CUDA graph."""
        rows = [self.step_coefficients(_as_int(t)) for t in timesteps]
        return torch.tensor(rows, dtype=torch.float32).reshape(-1, 5)

    def philox_stream(self, n: int):
        """(seed, offset0, stride) of the in-kernel noise stream for a loop of steps over n elements; advances the
        scheduler's offset past `steps` later via advance_philox."""
        if self._philox_seed is None:
            self._philox_seed = mix_seed(torch.initial_seed())
        return self._philox_seed, self._philox_offset, (n + 3) // 4

    def advance_philox(self, n: int, steps: int):
        self._philox_offset += steps * ((n + 3) // 4)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None, return_dict: bool = True,
             noise: Optional[torch.Tensor] = None, model_output_uncond: Optional[torch.Tensor] = None,
             guidance_w: float = 0.0, out: Optional[torch.Tensor] = None):
        """x_{t-1}.  Extras over diffusers (all optional): `noise` = explicit N(0,1) tensor (parity runs),
        `model_output_uncond` + `guidance_w` = classifier-free combine fused into the step (sample.py:134),
        `out` = destination (may be `sample` for an in-place update)."""
        # the C ABI takes raw pointers and one element count: every tensor must cover exactly sample.numel() elements
        for name, ten in (("model_output", model_output), ("model_output_uncond", model_output_uncond), ("noise", noise),
                          ("out", out)):
            if ten is not None and tuple(ten.shape) != tuple(sample.shape):
                raise RuntimeError(f"DDPMScheduler.step: {name} has shape {tuple(ten.shape)}, sample has {tuple(sample.shape)}")
        if out is not None and (out.dtype != torch.float32 or not out.is_contiguous() or out.device != sample.device):
            raise RuntimeError("DDPMScheduler.step: `out` must be a contiguous fp32 tensor on the sample's device")
        _require_cuda(sample, "sample")
        _require_cuda(model_output, "model_output")
        t = _as_int(timestep)
        sb, sa, c_x0, c_x, sigma = self.step_coefficients(t)
        x = sample if (sample.dtype == torch.float32 and sample.is_contiguous()) else sample.float().contiguous()
        eps = model_output.float().contiguous()
        eps_u = None if model_output_uncond is None else model_output_uncond.float().contiguous()
        if noise is None and generator is not None and sigma != 0.0:
            # diffusers' randn_tensor: a CPU generator samples on the CPU and the result is moved to the device
            gdev = generator.device if hasattr(generator, "device") else torch.device("cpu")
            noise = torch.randn(x.shape, generator=generator, device=x.device if gdev.type == "cuda" else "cpu",
                                dtype=torch.float32)
        if noise is not None:
            noise = noise.to(device=x.device, dtype=torch.float32).contiguous()
        n = x.numel()
        seed, offset = 0, 0
        if noise is None and sigma != 0.0:
            if self._philox_seed is None:
                self._philox_seed = mix_seed(torch.initial_seed())
            seed = self._philox_seed
            offset = self._philox_offset
            self._philox_offset += (n + 3) // 4
        dst = torch.empty_like(x) if out is None else out
        clip = float(self.config.clip_sample_range) if self.config.clip_sample else 0.0
        with torch.cuda.device(x.device):
            _ffi.check(_ffi.lib().bg_ddpm_step(eps.data_ptr(), _ffi.ptr(eps_u), float(guidance_w), x.data_ptr(),
                                              dst.data_ptr(), _ffi.ptr(noise), seed, offset, n, sb, sa, clip, c_x0, c_x,
                                              sigma, _ffi.current_stream()), "bg_ddpm_step")
        return SchedulerOutput(dst) if return_dict else (dst,)

    def add_noise(self, original_samples, noise, timesteps):
        acp = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
        timesteps = timesteps.to(original_samples.device)
        sa = acp[timesteps] ** 0.5
        sb = (1 - acp[timesteps]) ** 0.5
        while sa.dim() < original_samples.dim():
            sa, sb = sa.unsqueeze(-1), sb.unsqueeze(-1)
        return sa * original_samples + sb * noise

    def __len__(self):
        return self.config.num_train_timesteps


class PNDMScheduler:
    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", prediction_type: str = "epsilon", skip_prk_steps: bool = False,
                 set_alpha_to_one: bool = False, steps_offset: int = 0, **unused):
        if prediction_type != "epsilon" or skip_prk_steps or steps_offset != 0:
            raise NotImplementedError("only the configuration of sample.py:101-107 (epsilon, PRK steps, offset 0)")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, prediction_type=prediction_type,
                                      skip_prk_steps=skip_prk_steps, set_alpha_to_one=set_alpha_to_one,
                                      steps_offset=steps_offset)
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.pndm_order = 4
        self.set_timesteps(num_train_timesteps)

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.config.num_train_timesteps // num_inference_steps
        _t = (np.arange(0, num_inference_steps) * ratio).round().astype(np.int64)
        prk = np.array(_t[-self.pndm_order:]).repeat(2) + np.tile(np.array([0, ratio // 2]), self.pndm_order)
        self.prk_timesteps = (prk[:-1].repeat(2)[1:-1])[::-1].copy()
        self.plms_timesteps = _t[:-3][::-1].copy()
        self.timesteps = torch.from_numpy(np.concatenate([self.prk_timesteps, self.plms_timesteps]).astype(np.int64))
        self.ets: List[torch.Tensor] = []
        self.counter = 0
        self.cur_model_output = None
        self.cur_sample = None

    def scale_model_input(self, sample, timestep=None):
        return sample

    def transfer_coefficients(self, t: int, prev_t: int):
        """x_prev = c_sample * x - c_eps * eps  (diffusers `_get_prev_sample`, formula (9) of the PNDM paper)."""
        a_t = self.alphas_cumprod[t]
        a_p = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        b_t, b_p = 1 - a_t, 1 - a_p
        c_sample = (a_p / a_t) ** 0.5
        denom = a_t * b_p ** 0.5 + (a_t * b_t * a_p) ** 0.5
        return float(c_sample), float((a_p - a_t) / denom)

    def _launch(self, x, c_sample, c_eps, terms):
        """terms: list of (tensor, weight), at most 4"""
        dst = torch.empty_like(x)
        args = []
        for i in range(4):
            if i < len(terms):
                args += [terms[i][0].data_ptr(), float(terms[i][1])]
            else:
                args += [None, 0.0]
        with torch.cuda.device(x.device):
            _ffi.check(_ffi.lib().bg_pndm_step(x.data_ptr(), dst.data_ptr(), x.numel(), c_sample, c_eps, *args,
                                              _ffi.current_stream()), "bg_pndm_step")
        return dst

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, return_dict: bool = True):
        if tuple(model_output.shape) != tuple(sample.shape):
            raise RuntimeError(f"PNDMScheduler.step: model_output has shape {tuple(model_output.shape)}, "
                               f"sample has {tuple(sample.shape)}")
        _require_cuda(sample, "sample")
        _require_cuda(model_output, "model_output")
        t = _as_int(timestep)
        eps = model_output.float().contiguous()
        x = sample.float().contiguous()
        if self.counter < len(self.prk_timesteps):
            prev = self._step_prk(eps, t, x)
        else:
            prev = self._step_plms(eps, t, x)
        return SchedulerOutput(prev) if return_dict else (prev,)

    def _step_prk(self, eps, t, x):
        ratio = self.config.num_train_timesteps // self.num_inference_steps
        diff = 0 if self.counter % 2 else ratio // 2
        prev_t = t - diff
        t = int(self.prk_timesteps[self.counter // 4 * 4])
        r = self.counter % 4
        acc = self.cur_model_output            # list of (tensor, weight) forming the running RK sum
        if r == 0:
            acc = (acc or []) + [(eps, 1 / 6)]
            self.ets.append(eps)
            self.cur_sample = x
            terms = [(eps, 1.0)]
        elif r in (1, 2):
            acc = acc + [(eps, 1 / 3)]
            terms = [(eps, 1.0)]
        else:
            terms = acc + [(eps, 1 / 6)]        # eps' = k1/6 + k2/3 + k3/3 + k4/6, folded into the transfer kernel
            acc = None
        self.cur_model_output = acc
        c_sample, c_eps = self.transfer_coefficients(t, prev_t)
        out = self._launch(self.cur_sample, c_sample, c_eps, terms)
        self.counter += 1
        return out

    def _step_plms(self, eps, t, x):
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        self.ets = self.ets[-3:] + [eps]
        e = self.ets
        if len(e) == 1:
            terms = [(e[-1], 1.0)]
        elif len(e) == 2:
            terms = [(e[-1], 3 / 2), (e[-2], -1 / 2)]
        elif len(e) == 3:
            terms = [(e[-1], 23 / 12), (e[-2], -16 / 12), (e[-3], 5 / 12)]
        else:
            terms = [(e[-1], 55 / 24), (e[-2], -59 / 24), (e[-3], 37 / 24), (e[-4], -9 / 24)]
        c_sample, c_eps = self.transfer_coefficients(t, prev_t)
        out = self._launch(x, c_sample, c_eps, terms)
        self.counter += 1
        return out

    def add_noise(self, original_samples, noise, timesteps):
        return DDPMScheduler.add_noise(self, original_samples, noise, timesteps)

    def __len__(self):
        return self.config.num_train_timesteps
