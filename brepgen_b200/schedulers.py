"""Drop-in DDPMScheduler / PNDMScheduler with the diffusers 0.27 interface used by the reference, DDIMScheduler and
DPMSolverMultistepScheduler (diffusers' few-step samplers for the same epsilon-prediction models) and RePaintScheduler
(diffusers' inpainting with resampling; none of these three is used by the reference).

Call sites mirrored (all in the reference): constructors sample.py:101-117 and trainer.py:285-292;
`set_timesteps(n)` + `.timesteps[...]` slicing sample.py:128-129,144-145; `.step(pred, t, x).prev_sample`
sample.py:137,153,202,222,236,282; `.add_noise(x, noise, t)` trainer.py:348; `.config.num_train_timesteps` trainer.py:330.

Host side (this file): the beta / alphas_cumprod tables and the per-step scalar coefficients, computed with the same
fp32 torch-CPU operations diffusers uses (SURVEY.md Appendix A.3/A.4).  Device side: ONE fused kernel per step
(bg_ddpm_step / bg_ddim_step / bg_dpm_step / bg_repaint_step / bg_pndm_step in csrc/sched.cu) instead of ~15 scalar-broadcast launches.  No CPU tensor path:
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


def sample_seed(seed: int, index: int) -> int:
    """64-bit seed of the sample at global index `index` of a run seeded with `seed` (per-sample noise mode).  A mix rather
    than seed + index, so that runs with neighbouring seeds share no sample."""
    return mix_seed(seed, index)


def sample_keys(seeds, stage: int) -> np.ndarray:
    """uint64 [len(seeds)]: the Philox key of each sample's noise streams in one cascade stage (bg_randn_keyed and the
    sample_keys of the fused steps)"""
    return np.array([mix_seed(s, stage) for s in seeds], dtype=np.uint64)


def randn_generators(shape, generators, device=None, dtype=torch.float32) -> torch.Tensor:
    """diffusers' randn_tensor for a list of generators, one per batch element: element i of the batch is drawn from
    generators[i] on the generators' device (CPU generators sample on the host) and the result is moved to `device`"""
    shape = tuple(shape)
    if len(generators) != shape[0]:
        raise ValueError(f"got {len(generators)} generators for a batch of {shape[0]}")
    gdev = generators[0].device if hasattr(generators[0], "device") else torch.device("cpu")
    rows = [torch.randn((1,) + shape[1:], generator=g, device=gdev, dtype=dtype) for g in generators]
    return torch.cat(rows, 0).to(device if device is not None else gdev)


def _as_int(t) -> int:
    return int(t.item()) if torch.is_tensor(t) else int(t)


def _require_cuda(x: torch.Tensor, what: str):
    if not x.is_cuda:
        raise RuntimeError(f"brepgen_b200 schedulers have no CPU path: {what} must be a CUDA tensor")


def _step_tensors(what, model_output, sample, model_output_uncond, noise, out):
    """Checks the tensors of a fused step; returns (x, eps, eps_uncond, destination) as contiguous fp32."""
    # the C ABI takes raw pointers and one element count: every tensor must cover exactly sample.numel() elements
    for name, ten in (("model_output", model_output), ("model_output_uncond", model_output_uncond), ("noise", noise),
                      ("out", out)):
        if ten is not None and tuple(ten.shape) != tuple(sample.shape):
            raise RuntimeError(f"{what}: {name} has shape {tuple(ten.shape)}, sample has {tuple(sample.shape)}")
    if out is not None and (out.dtype != torch.float32 or not out.is_contiguous() or out.device != sample.device):
        raise RuntimeError(f"{what}: `out` must be a contiguous fp32 tensor on the sample's device")
    _require_cuda(sample, "sample")
    _require_cuda(model_output, "model_output")
    x = sample if (sample.dtype == torch.float32 and sample.is_contiguous()) else sample.float().contiguous()
    eps = model_output.float().contiguous()
    eps_u = None if model_output_uncond is None else model_output_uncond.float().contiguous()
    return x, eps, eps_u, (torch.empty_like(x) if out is None else out)


def _generator_noise(x: torch.Tensor, generator) -> torch.Tensor:
    """N(0, 1) of x's shape drawn as diffusers' randn_tensor draws it from `generator` (one, or a list with one per batch
    element)"""
    if isinstance(generator, (list, tuple)):
        # diffusers' randn_tensor with one generator per batch element (the reference's utils.py:62-97)
        return randn_generators(x.shape, generator, x.device)
    # diffusers' randn_tensor: a CPU generator samples on the CPU and the result is moved to the device
    gdev = generator.device if hasattr(generator, "device") else torch.device("cpu")
    return torch.randn(x.shape, generator=generator, device=x.device if gdev.type == "cuda" else "cpu", dtype=torch.float32)


class _NoiseStreams:
    """The in-kernel noise sources shared by the fused DDPM, DDIM and DPM-Solver++ steps: one batch-wide Philox stream
    (set_noise_seed) or per-sample streams (set_sample_keys)."""

    def _init_noise_streams(self):
        self._philox_seed = None       # None: derived from torch.initial_seed() at first use (follows torch.manual_seed)
        self._philox_offset = 0
        self._sample_seeds = None      # per-sample noise mode: None (batch-wide stream) or (seed, first, stage, seeds)
        self._key_cache = {}

    def set_noise_seed(self, seed: int, *stream: int):
        """Key of the in-kernel Philox stream that `step` draws its noise from when neither `noise` nor `generator` is
        given: a 64-bit mix of `seed` and any further integers (rank, stage, ...).  Resets the stream offset, so a run is
        reproducible from the seed alone and different (seed, rank, stage) tuples give independent streams
        (SURVEY.md 8(e): per-rank independent RNG streams).  Leaves per-sample mode."""
        self._philox_seed = mix_seed(seed, *stream)
        self._philox_offset = 0
        self._sample_seeds = None

    def set_sample_keys(self, seed: int = 0, first: int = 0, stage: int = 0, sample_seeds=None):
        """Per-sample noise mode: sample i of the batch `step` is given draws its noise from its own Philox stream, keyed by
        mix_seed(s_i, stage) and counted by (element // 4, t, 0), so its noise depends on neither the batch size nor its
        position in the batch.  s_i = sample_seed(seed, first + i) (`first` = global index of the batch's first sample), or
        sample_seeds[i] when given.  `noise=` and `generator=` still take precedence; set_noise_seed leaves this mode."""
        self._sample_seeds = (int(seed), int(first), int(stage),
                              None if sample_seeds is None else [int(s) for s in sample_seeds])
        self._key_cache = {}

    @property
    def per_sample_noise(self) -> bool:
        return self._sample_seeds is not None

    def sample_key_tensor(self, batch: int, device) -> torch.Tensor:
        """device int64 [batch] holding the uint64 keys of the per-sample mode set by set_sample_keys"""
        if self._sample_seeds is None:
            raise RuntimeError(f"{type(self).__name__}: per-sample noise mode is not set (call set_sample_keys)")
        seed, first, stage, seeds = self._sample_seeds
        if seeds is None:
            seeds = [sample_seed(seed, first + i) for i in range(batch)]
        elif len(seeds) != batch:
            raise ValueError(f"{type(self).__name__}: {len(seeds)} sample seeds for a batch of {batch}")
        key = (batch, str(device))
        if key not in self._key_cache:
            self._key_cache[key] = torch.from_numpy(sample_keys(seeds, stage).view(np.int64)).to(device)
        return self._key_cache[key]

    def philox_stream(self, n: int):
        """(seed, offset0, stride) of the in-kernel noise stream for a loop of steps over n elements; advances the
        scheduler's offset past `steps` later via advance_philox."""
        if self._philox_seed is None:
            self._philox_seed = mix_seed(torch.initial_seed())
        return self._philox_seed, self._philox_offset, (n + 3) // 4

    def advance_philox(self, n: int, steps: int):
        self._philox_offset += steps * ((n + 3) // 4)

    def _step_noise(self, x: torch.Tensor, draws: bool, noise: Optional[torch.Tensor] = None, generator=None):
        """(noise, seed, offset, keys) of a fused step on x.  A step that draws noise (DDPM: sigma != 0, DDIM: eta > 0,
        DPM-Solver++: its SDE form) takes `noise`, else a draw from `generator` (one, or a list with one per batch
        element), else the per-sample streams of set_sample_keys, else the batch stream, whose offset it moves past the
        step.  A step that draws none takes none of them."""
        if not draws:
            return None, 0, 0, None
        if noise is None and generator is not None:
            noise = _generator_noise(x, generator)
        if noise is not None:
            return noise.to(device=x.device, dtype=torch.float32).contiguous(), 0, 0, None
        if self._sample_seeds is not None:
            return None, 0, 0, self.sample_key_tensor(x.shape[0], x.device)
        seed, offset, _ = self.philox_stream(x.numel())
        self.advance_philox(x.numel(), 1)
        return None, seed, offset, None

    # ---------------------------------------------------------------- known-token replacement (B-rep completion)
    def _abar_prev(self, t: int) -> torch.Tensor:
        raise NotImplementedError

    def replace_coefficients(self, t: int, initial: bool = False):
        """(sqrt(abar), sqrt(1 - abar)) as Python floats (fp32 arithmetic): abar = abar_prev(t) of this scheduler's step
        convention, the noise level `step` leaves x at; initial=True: abar_t itself, the level of a stage's starting noise"""
        a = self.alphas_cumprod[int(t)] if initial else self._abar_prev(int(t))
        return float(a ** 0.5), float((1 - a) ** 0.5)

    def replace_table(self, timesteps) -> torch.Tensor:
        """[len(timesteps), 2] fp32 (CPU): replace_coefficients(t) for every t of a denoising loop -- the device table that
        bg_replace_known_tab indexes with the step counter of bg_step_advance"""
        rows = [self.replace_coefficients(_as_int(t)) for t in timesteps]
        return torch.tensor(rows, dtype=torch.float32).reshape(-1, 2)

    def replace_seed(self) -> int:
        """batch-mode key of the replacement noise: mix_seed(step stream key, 2).  Reads the step stream's key but never
        its offset, so replacing tokens leaves the step noise exactly as it is without replacement."""
        if self._philox_seed is None:
            self._philox_seed = mix_seed(torch.initial_seed())
        return mix_seed(self._philox_seed, 2)

    def replace_known(self, sample: torch.Tensor, known: torch.Tensor, known_mask: torch.Tensor, timestep,
                      noise: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, initial: bool = False):
        """The sample with its known tokens set to q(x_prev(t) | known) = sqrt(abar_prev) known + sqrt(1 - abar_prev) z
        (inpainting by replacement): call it after `step(..., t, ...)` with the same t.  A token is the last dimension:
        known_mask has sample.shape[:-1], True = known; other tokens are left bit for bit as they are.  z: `noise`, else
        the per-sample streams of set_sample_keys (domain 2, counter t), else the batch key replace_seed() (counter t),
        which does not move the step's noise stream.  initial=True: the replacement before the first step at t (noise
        level abar_t, counter t + 1).  out: destination, may be `sample` (in place); default a new tensor."""
        if tuple(known.shape) != tuple(sample.shape) or tuple(known_mask.shape) != tuple(sample.shape[:-1]):
            raise RuntimeError(f"replace_known: known {tuple(known.shape)} and known_mask {tuple(known_mask.shape)} must "
                               f"have the sample's shape {tuple(sample.shape)} and its shape without the last dimension")
        if noise is not None and tuple(noise.shape) != tuple(sample.shape):
            raise RuntimeError(f"replace_known: noise has shape {tuple(noise.shape)}, sample has {tuple(sample.shape)}")
        if out is not None and (out.dtype != torch.float32 or not out.is_contiguous() or out.device != sample.device or
                                tuple(out.shape) != tuple(sample.shape)):
            raise RuntimeError("replace_known: `out` must be a contiguous fp32 tensor of the sample's shape and device")
        _require_cuda(sample, "sample")
        t = _as_int(timestep)
        sa, sb = self.replace_coefficients(t, initial)
        t_ctr = t + 1 if initial else t
        if out is None:
            dst = sample.float().contiguous().clone()
        else:
            dst = out
            if dst.data_ptr() != sample.data_ptr():
                dst.copy_(sample)
        kn = known.to(device=dst.device, dtype=torch.float32).contiguous()
        m = known_mask.to(device=dst.device, dtype=torch.uint8).contiguous()
        if noise is not None:
            noise = noise.to(device=dst.device, dtype=torch.float32).contiguous()
        n = dst.numel()
        seed, keys = 0, None
        if noise is None:
            if self._sample_seeds is not None:
                keys = self.sample_key_tensor(dst.shape[0], dst.device)
            else:
                seed = self.replace_seed()
        if n == 0:
            return dst
        with torch.cuda.device(dst.device):
            _ffi.check(_ffi.lib().bg_replace_known(dst.data_ptr(), kn.data_ptr(), m.data_ptr(), n, dst.shape[-1],
                                                  _ffi.ptr(noise), seed, _ffi.ptr(keys), n // dst.shape[0], t_ctr, sa, sb,
                                                  _ffi.current_stream()), "bg_replace_known")
        return dst


class DDPMScheduler(_NoiseStreams):
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
        self._init_noise_streams()
        self.set_timesteps(num_train_timesteps)

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

    def _abar_prev(self, t: int) -> torch.Tensor:
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        return self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one

    def coefficient_table(self, timesteps) -> torch.Tensor:
        """[len(timesteps), 5] fp32 (CPU): step_coefficients(t) for every t of a denoising loop -- the device table that
        bg_ddpm_step_tab indexes with its step counter when the loop is captured in a CUDA graph."""
        rows = [self.step_coefficients(_as_int(t)) for t in timesteps]
        return torch.tensor(rows, dtype=torch.float32).reshape(-1, 5)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None, return_dict: bool = True,
             noise: Optional[torch.Tensor] = None, model_output_uncond: Optional[torch.Tensor] = None,
             guidance_w: float = 0.0, out: Optional[torch.Tensor] = None):
        """x_{t-1}.  Extras over diffusers (all optional): `noise` = explicit N(0,1) tensor (parity runs),
        `model_output_uncond` + `guidance_w` = classifier-free combine fused into the step (sample.py:134),
        `out` = destination (may be `sample` for an in-place update).  `generator` may be one generator or, as in
        diffusers, a list with one per batch element (sample i's noise from generator[i]; CPU generators sample on the
        host).  Without `noise` or `generator` the noise comes from the in-kernel stream: batch-wide (set_noise_seed) or
        per sample (set_sample_keys)."""
        x, eps, eps_u, dst = _step_tensors("DDPMScheduler.step", model_output, sample, model_output_uncond, noise, out)
        t = _as_int(timestep)
        sb, sa, c_x0, c_x, sigma = self.step_coefficients(t)
        noise, seed, offset, keys = self._step_noise(x, sigma != 0.0, noise, generator)
        n = x.numel()
        clip = float(self.config.clip_sample_range) if self.config.clip_sample else 0.0
        with torch.cuda.device(x.device):
            _ffi.check(_ffi.lib().bg_ddpm_step(eps.data_ptr(), _ffi.ptr(eps_u), float(guidance_w), x.data_ptr(),
                                              dst.data_ptr(), _ffi.ptr(noise), seed, offset, _ffi.ptr(keys),
                                              n // x.shape[0], t, n, sb, sa, clip, c_x0, c_x, sigma,
                                              _ffi.current_stream()), "bg_ddpm_step")
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


class DDIMScheduler(_NoiseStreams):
    """diffusers 0.27 DDIMScheduler for epsilon-prediction models: few-step deterministic (eta = 0) or stochastic sampling
    of a model trained as a DDPM.  One fused kernel per step (bg_ddim_step); the per-step scalars are computed here in fp32
    torch as diffusers computes them."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, clip_sample: bool = True, set_alpha_to_one: bool = True,
                 steps_offset: int = 0, prediction_type: str = "epsilon", thresholding: bool = False,
                 dynamic_thresholding_ratio: float = 0.995, clip_sample_range: float = 1.0, sample_max_value: float = 1.0,
                 timestep_spacing: str = "leading", rescale_betas_zero_snr: bool = False, **unused):
        if prediction_type != "epsilon" or thresholding or rescale_betas_zero_snr or timestep_spacing != "leading" or \
                trained_betas is not None:
            raise NotImplementedError("only prediction_type='epsilon', timestep_spacing='leading', no thresholding, no "
                                      "zero-SNR rescaling and no trained_betas")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, trained_betas=trained_betas, clip_sample=clip_sample,
                                      set_alpha_to_one=set_alpha_to_one, steps_offset=steps_offset,
                                      prediction_type=prediction_type, thresholding=thresholding,
                                      dynamic_thresholding_ratio=dynamic_thresholding_ratio,
                                      clip_sample_range=clip_sample_range, sample_max_value=sample_max_value,
                                      timestep_spacing=timestep_spacing, rescale_betas_zero_snr=rescale_betas_zero_snr)
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))
        self._init_noise_streams()

    def set_timesteps(self, num_inference_steps: int, device=None):
        n_train = self.config.num_train_timesteps
        if num_inference_steps > n_train:
            raise ValueError("num_inference_steps cannot exceed num_train_timesteps")
        self.num_inference_steps = num_inference_steps
        ratio = n_train // num_inference_steps                      # timestep_spacing = "leading"
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(ts + self.config.steps_offset)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step_coefficients(self, t: int, eta: float = 0.0):
        """(sqrt(1-abar_t), sqrt(abar_t), sqrt(abar_prev), c_dir, sigma) as Python floats (fp32 arithmetic like diffusers)"""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        b_t = 1 - a_t
        variance = ((1 - a_prev) / b_t) * (1 - a_t / a_prev)
        std_dev_t = eta * variance ** 0.5
        c_dir = (1 - a_prev - std_dev_t ** 2) ** 0.5
        return float(b_t ** 0.5), float(a_t ** 0.5), float(a_prev ** 0.5), float(c_dir), float(std_dev_t)

    def _abar_prev(self, t: int) -> torch.Tensor:
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        return self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod

    def coefficient_table(self, timesteps, eta: float = 0.0) -> torch.Tensor:
        """[len(timesteps), 5] fp32 (CPU): step_coefficients(t, eta) for every t of a denoising loop -- the device table
        that bg_ddim_step_tab indexes with its step counter when the loop is captured in a CUDA graph."""
        rows = [self.step_coefficients(_as_int(t), eta) for t in timesteps]
        return torch.tensor(rows, dtype=torch.float32).reshape(-1, 5)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, eta: float = 0.0,
             use_clipped_model_output: bool = False, generator=None, variance_noise: Optional[torch.Tensor] = None,
             return_dict: bool = True, model_output_uncond: Optional[torch.Tensor] = None, guidance_w: float = 0.0,
             out: Optional[torch.Tensor] = None):
        """x_{t-1} of diffusers' DDIM step.  When eta > 0 the noise comes from `variance_noise`, else `generator` (one, or
        a list with one per batch element), else the in-kernel stream (per sample after set_sample_keys, else batch-wide),
        and is drawn on every step, the last one included, as diffusers draws it.  Extras over diffusers, as in
        DDPMScheduler.step: `model_output_uncond` + `guidance_w` fuse the classifier-free combine, `out` is the
        destination (may be `sample`).  pred_original_sample is not returned (None)."""
        t = _as_int(timestep)
        sb, sa, sa_prev, c_dir, sigma = self.step_coefficients(t, eta)
        if eta > 0 and variance_noise is not None and generator is not None:
            raise ValueError("Cannot pass both generator and variance_noise. Please make sure that either "
                             "`generator` or `variance_noise` stays `None`.")
        x, eps, eps_u, dst = _step_tensors("DDIMScheduler.step", model_output, sample, model_output_uncond,
                                           variance_noise, out)
        noise, seed, offset, keys = self._step_noise(x, eta > 0, variance_noise, generator)
        n = x.numel()
        with torch.cuda.device(x.device):
            _ffi.check(_ffi.lib().bg_ddim_step(eps.data_ptr(), _ffi.ptr(eps_u), float(guidance_w), x.data_ptr(),
                                              dst.data_ptr(), _ffi.ptr(noise), seed, offset, _ffi.ptr(keys),
                                              n // x.shape[0], t, n, sb, sa, sa_prev, c_dir, sigma,
                                              float(self.config.clip_sample_range) if self.config.clip_sample else 0.0,
                                              int(bool(use_clipped_model_output)), _ffi.current_stream()), "bg_ddim_step")
        return SchedulerOutput(dst) if return_dict else (dst,)

    def add_noise(self, original_samples, noise, timesteps):
        return DDPMScheduler.add_noise(self, original_samples, noise, timesteps)

    def __len__(self):
        return self.config.num_train_timesteps


def strength_timesteps(timesteps, strength: float):
    """The tail of a denoising loop that a variation at `strength` runs (diffusers' img2img get_timesteps):
    timesteps[N - min(int(N * strength), N):], N = len(timesteps).  strength 1 is the whole loop, 0 none of it.  The sample
    starts at add_noise(source, z, list[0]).  ValueError, as diffusers raises it: strength outside [0, 1], or a strength
    > 0 that leaves no step (int(N * strength) == 0)."""
    n = len(timesteps)
    s = float(strength)
    if not 0.0 <= s <= 1.0:
        raise ValueError(f"The value of strength should be in [0.0, 1.0] but is {strength}")
    k = min(int(n * s), n)
    if s > 0 and k < 1:
        raise ValueError(f"strength {strength} of a {n}-step schedule leaves no step (int({n} * strength) = 0); use a "
                         f"strength of at least {1.0 / n:g}")
    return timesteps[n - k:]


def repaint_timesteps(num_inference_steps: int, jump_length: int, jump_n_sample: int,
                      num_train_timesteps: int = 1000) -> np.ndarray:
    """int64 timesteps of diffusers' RePaintScheduler.set_timesteps: N - 1 .. 0 in steps of one, with a jump back up by
    jump_length after every jump_length-th index, jump_n_sample - 1 times each, scaled by num_train_timesteps // N"""
    n = min(num_train_timesteps, int(num_inference_steps))
    jumps = {j: jump_n_sample - 1 for j in range(0, n - jump_length, jump_length)}
    t, ts = n, []
    while t >= 1:
        t -= 1
        ts.append(t)
        if jumps.get(t, 0) > 0:
            jumps[t] -= 1
            for _ in range(jump_length):
                t += 1
                ts.append(t)
    return np.array(ts, dtype=np.int64) * (num_train_timesteps // n)


def repaint_entries(timesteps):
    """[(is_step, t)] of the RePaint loop over `timesteps` (diffusers' pipeline): an entry below the previous one is a
    denoising step at t; any other is an undo_step from the previous entry t_last (the first entry is a step)"""
    ts = [_as_int(t) for t in timesteps]
    out, t_last = [], (ts[0] + 1 if ts else 0)
    for t in ts:
        out.append((True, t) if t < t_last else (False, t_last))
        t_last = t
    return out


class RePaintScheduler(_NoiseStreams):
    """diffusers 0.27 RePaintScheduler for epsilon-prediction models: DDIM-form steps that keep the known region at
    q(x_prev | known), and undo steps that noise the whole sample back up so the generated part is denoised again around
    the known part (Lugmayr et al. 2022).  One fused kernel per entry (bg_repaint_step / bg_repaint_undo); the per-step
    scalars are those of DDIMScheduler (set_alpha_to_one), computed in fp32 torch as diffusers computes them.

    mask: 1 / True = known, one value per token (sample.shape[:-1], or with a trailing 1), bool, uint8 or a float tensor
    holding only 0 and 1 -- the kernel selects, it does not blend.  Extras over diffusers: `clip_sample_range` (diffusers
    clips to +-1), `model_output_uncond` + `guidance_w`, `noise`, `out`, the noise streams of set_noise_seed /
    set_sample_keys, and the coefficient tables of the graph form.  Keyed and in-kernel noise are counted by the entry
    index of the current timestep list (reset by set_timesteps; step and undo_step each take one entry)."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", eta: float = 0.0, trained_betas=None, clip_sample: bool = True,
                 clip_sample_range: float = 1.0, prediction_type: str = "epsilon", **unused):
        if trained_betas is not None or prediction_type != "epsilon":
            raise NotImplementedError("only prediction_type='epsilon' and no trained_betas")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, eta=eta, trained_betas=trained_betas,
                                      clip_sample=clip_sample, clip_sample_range=clip_sample_range,
                                      prediction_type=prediction_type)
        self._ddim = DDIMScheduler(num_train_timesteps, beta_start, beta_end, beta_schedule, clip_sample=clip_sample,
                                   set_alpha_to_one=True, clip_sample_range=clip_sample_range)
        self.betas, self.alphas_cumprod = self._ddim.betas, self._ddim.alphas_cumprod
        self.eta = float(eta)
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))
        self._entry = 0
        self._undo_rows = {}
        self._init_noise_streams()

    def set_timesteps(self, num_inference_steps: int, jump_length: int = 10, jump_n_sample: int = 10, device=None):
        n_train = self.config.num_train_timesteps
        if num_inference_steps < 1 or jump_length < 1 or jump_n_sample < 1:
            raise ValueError("num_inference_steps, jump_length and jump_n_sample must be positive")
        ts = repaint_timesteps(num_inference_steps, jump_length, jump_n_sample, n_train)
        n = min(n_train, num_inference_steps)
        if len(ts) * (n_train // n) >= 2 ** 32:
            raise ValueError(f"a list of {len(ts)} entries with {n_train // n} transitions per undo overflows the 32-bit "
                             "noise counter")
        self.num_inference_steps = n
        self._ddim.set_timesteps(n)
        self.timesteps = torch.from_numpy(ts)
        self._entry = 0

    def scale_model_input(self, sample, timestep=None):
        return sample

    @property
    def undo_transitions(self) -> int:
        """n = num_train_timesteps // num_inference_steps: the forward-diffusion transitions of one undo_step"""
        self._need_timesteps()
        return self.config.num_train_timesteps // self.num_inference_steps

    def _need_timesteps(self):
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")

    def step_coefficients(self, t: int, eta: Optional[float] = None):
        """(sqrt(1-abar_t), sqrt(abar_t), sqrt(abar_prev), c_dir, sigma, sqrt(1-abar_prev)) as Python floats: DDIM's
        coefficients (abar_prev = 1 past the last step) and the noise level of the known part"""
        self._need_timesteps()
        sb, sa, sa_prev, c_dir, sigma = self._ddim.step_coefficients(int(t), self.eta if eta is None else eta)
        return sb, sa, sa_prev, c_dir, sigma, float((1 - self._ddim._abar_prev(int(t))) ** 0.5)

    def undo_coefficients(self, t_last: int) -> torch.Tensor:
        """[n, 2] fp32 (CPU): (sqrt(1 - beta), sqrt(beta)) of transitions t_last .. t_last + n - 1, as diffusers computes
        them"""
        n = self.undo_transitions
        if not 0 <= t_last <= self.config.num_train_timesteps - n:
            raise ValueError(f"undo_step: timestep {t_last} + {n} transitions leaves the training range")
        rows = [(float((1 - self.betas[t_last + i]) ** 0.5), float(self.betas[t_last + i] ** 0.5)) for i in range(n)]
        return torch.tensor(rows, dtype=torch.float32)

    def coefficient_table(self, timesteps=None, eta: Optional[float] = None) -> torch.Tensor:
        """[len(timesteps), 6] fp32 (CPU): step_coefficients of every step entry of a RePaint loop (default: the whole
        list), zero rows at undo entries -- the device table bg_repaint_step_tab indexes with the entry counter"""
        ents = repaint_entries(self.timesteps if timesteps is None else timesteps)
        rows = [self.step_coefficients(t, eta) if is_step else (0.0,) * 6 for is_step, t in ents]
        return torch.tensor(rows, dtype=torch.float32).reshape(-1, 6)

    def undo_table(self, timesteps=None) -> torch.Tensor:
        """[len(timesteps), n, 2] fp32 (CPU): undo_coefficients(t_last) of every undo entry, zero at step entries -- the
        device table bg_repaint_undo_tab indexes with the entry counter"""
        ents = repaint_entries(self.timesteps if timesteps is None else timesteps)
        n = self.undo_transitions
        rows = [torch.zeros(n, 2) if is_step else self.undo_coefficients(t) for is_step, t in ents]
        return torch.stack(rows, 0) if rows else torch.zeros(0, n, 2)

    def repaint_seed(self, domain: int) -> int:
        """batch-mode key of the step (domain 3) or undo (domain 4) noise: mix_seed(step stream key, domain).  It never
        reads or advances the (seed, offset) stream of the other steps."""
        if self._philox_seed is None:
            self._philox_seed = mix_seed(torch.initial_seed())
        return mix_seed(self._philox_seed, domain)

    def _noise_source(self, batch, device, domain):
        if self._sample_seeds is not None:
            return 0, self.sample_key_tensor(batch, device)
        return self.repaint_seed(domain), None

    def _next_entry(self) -> int:
        k = self._entry
        self._entry += 1
        return k

    @staticmethod
    def token_mask(mask: torch.Tensor, sample: torch.Tensor) -> torch.Tensor:
        """the uint8 token mask (sample.shape[:-1]) of a step's `mask`; ValueError on another shape or a float value
        other than 0 and 1"""
        shp = tuple(sample.shape[:-1])
        m = mask
        if tuple(m.shape) == shp + (1,):
            m = m[..., 0]
        if tuple(m.shape) != shp:
            raise ValueError(f"RePaintScheduler: mask must have shape {shp} (one value per token) or {shp + (1,)}, got "
                             f"{tuple(mask.shape)}")
        if m.dtype.is_floating_point:
            if not bool(((m == 0) | (m == 1)).all()):
                raise ValueError("RePaintScheduler: a float mask must hold only 0 and 1 (the step selects known or "
                                 "generated values per token; it does not blend)")
        elif m.dtype == torch.uint8:
            return m.to(device=sample.device).contiguous()
        elif m.dtype != torch.bool:
            raise ValueError(f"RePaintScheduler: mask must be bool, uint8 or a 0/1 float tensor, got {m.dtype}")
        return (m != 0).to(device=sample.device, dtype=torch.uint8).contiguous()

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, original_image: Optional[torch.Tensor],
             mask: Optional[torch.Tensor], generator=None, return_dict: bool = True,
             model_output_uncond: Optional[torch.Tensor] = None, guidance_w: float = 0.0,
             noise: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None):
        """x at the previous timestep of diffusers' RePaint step: known tokens (mask = 1) at
        sqrt(abar_prev) original_image + sqrt(1 - abar_prev) z, the others the DDIM update with eta = self.eta and the
        variance term sigma z with the same z.  original_image = mask = None: nothing known.  z: `noise`, else `generator`
        (one, or a list with one per batch element), else the per-sample streams of set_sample_keys (domain 3), else the
        batch key repaint_seed(3), counted by the entry index.  pred_original_sample is not returned (None)."""
        x, eps, eps_u, dst = _step_tensors("RePaintScheduler.step", model_output, sample, model_output_uncond, noise, out)
        if (original_image is None) != (mask is None):
            raise ValueError("RePaintScheduler.step: give original_image and mask together, or neither")
        kn = m = None
        if mask is not None:
            if tuple(original_image.shape) != tuple(sample.shape):
                raise RuntimeError(f"RePaintScheduler.step: original_image has shape {tuple(original_image.shape)}, "
                                   f"sample has {tuple(sample.shape)}")
            m = self.token_mask(mask, x)
            kn = original_image.to(device=x.device, dtype=torch.float32).contiguous()
        t = _as_int(timestep)
        coefs = self.step_coefficients(t)
        k = self._next_entry()
        if noise is None and generator is not None:
            noise = _generator_noise(x, generator)
        if noise is not None:
            noise = noise.to(device=x.device, dtype=torch.float32).contiguous()
        n = x.numel()
        seed, keys = self._noise_source(x.shape[0], x.device, 3)
        clip = float(self.config.clip_sample_range) if self.config.clip_sample else 0.0
        with torch.cuda.device(x.device):
            _ffi.check(_ffi.lib().bg_repaint_step(eps.data_ptr(), _ffi.ptr(eps_u), float(guidance_w), x.data_ptr(),
                                                 dst.data_ptr(), _ffi.ptr(kn), _ffi.ptr(m), x.shape[-1], _ffi.ptr(noise),
                                                 seed, _ffi.ptr(keys), n // x.shape[0], k, n, *coefs, clip,
                                                 _ffi.current_stream()), "bg_repaint_step")
        return SchedulerOutput(dst) if return_dict else (dst,)

    def undo_step(self, sample: torch.Tensor, timestep, generator=None, noise: Optional[torch.Tensor] = None,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """sample noised by the n = num_train_timesteps // num_inference_steps forward transitions timestep ..
        timestep + n - 1: x = sqrt(1 - beta) x + sqrt(beta) z, a fresh z per transition.  z: `noise` of shape
        (n, *sample.shape), else n draws from `generator` in order (as diffusers draws them), else the per-sample streams
        (domain 4), else the batch key repaint_seed(4), counted by the entry index.  out: destination, may be `sample`."""
        _require_cuda(sample, "sample")
        t_last = _as_int(timestep)
        cf = self.undo_coefficients(t_last)
        nt = cf.shape[0]
        if noise is not None and tuple(noise.shape) != (nt,) + tuple(sample.shape):
            raise RuntimeError(f"undo_step: noise has shape {tuple(noise.shape)}, want {(nt,) + tuple(sample.shape)}")
        if out is not None and (out.dtype != torch.float32 or not out.is_contiguous() or out.device != sample.device or
                                tuple(out.shape) != tuple(sample.shape)):
            raise RuntimeError("undo_step: `out` must be a contiguous fp32 tensor of the sample's shape and device")
        k = self._next_entry()
        if out is None:
            dst = sample.float().contiguous().clone()
        else:
            dst = out
            if dst.data_ptr() != sample.data_ptr():
                dst.copy_(sample)
        if noise is None and generator is not None:
            noise = torch.stack([_generator_noise(dst, generator).to(dst.device) for _ in range(nt)], 0)
        if noise is not None:
            noise = noise.to(device=dst.device, dtype=torch.float32).contiguous()
        key = (t_last, nt, str(dst.device))
        if key not in self._undo_rows:
            self._undo_rows[key] = cf.to(dst.device)
        n = dst.numel()
        seed, keys = self._noise_source(dst.shape[0], dst.device, 4)
        with torch.cuda.device(dst.device):
            _ffi.check(_ffi.lib().bg_repaint_undo(dst.data_ptr(), n, nt, self._undo_rows[key].data_ptr(), _ffi.ptr(noise),
                                                 seed, _ffi.ptr(keys), n // dst.shape[0], k, _ffi.current_stream()),
                       "bg_repaint_undo")
        return dst

    def add_noise(self, original_samples, noise, timesteps):
        return DDPMScheduler.add_noise(self, original_samples, noise, timesteps)

    def __len__(self):
        return self.config.num_train_timesteps


DPM_ALGORITHMS = ("dpmsolver++", "sde-dpmsolver++")


def dpm_timesteps(num_train_timesteps: int, num_inference_steps: int, spacing: str, steps_offset: int = 0) -> np.ndarray:
    """int64 timesteps of diffusers' DPMSolverMultistepScheduler.set_timesteps (lambda_min_clipped = -inf)"""
    n, last = num_inference_steps, num_train_timesteps
    if spacing == "linspace":
        return np.linspace(0, last - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
    if spacing == "leading":
        ratio = last // (n + 1)
        return (np.arange(0, n + 1) * ratio).round()[::-1][:-1].copy().astype(np.int64) + steps_offset
    if spacing == "trailing":
        return np.arange(last, 0, -num_train_timesteps / n).round().copy().astype(np.int64) - 1
    raise NotImplementedError(f"timestep_spacing={spacing!r}")


class DPMSolverMultistepScheduler(_NoiseStreams):
    """diffusers 0.27 DPMSolverMultistepScheduler for epsilon-prediction models: the DPM-Solver++ multistep ("2M") sampler,
    deterministic ("dpmsolver++") or stochastic ("sde-dpmsolver++"), of a model trained as a DDPM.  One fused kernel per
    step (bg_dpm_step); the per-step scalars are computed here in fp32 torch as diffusers computes them.  The history of
    data predictions (diffusers' model_outputs list) is one device tensor of the sample's shape, `hist`, that the kernel
    reads and overwrites in place.

    Extras over diffusers: `clip_sample` / `clip_sample_range` clamp the data prediction x0 before it is used and stored
    (static thresholding; off by default, as in diffusers, which has no such option).  A `step` on a sample whose shape
    differs from the history's restarts the solver: that step is first order and the history is reallocated."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "epsilon", thresholding: bool = False, dynamic_thresholding_ratio: float = 0.995,
                 sample_max_value: float = 1.0, algorithm_type: str = "dpmsolver++", solver_type: str = "midpoint",
                 lower_order_final: bool = True, euler_at_final: bool = False, use_karras_sigmas: bool = False,
                 use_lu_lambdas: bool = False, final_sigmas_type: str = "zero", lambda_min_clipped: float = -float("inf"),
                 variance_type=None, timestep_spacing: str = "linspace", steps_offset: int = 0,
                 clip_sample: bool = False, clip_sample_range: float = 1.0, **unused):
        if prediction_type != "epsilon" or thresholding or use_karras_sigmas or use_lu_lambdas or \
                solver_order not in (1, 2) or algorithm_type not in DPM_ALGORITHMS or solver_type != "midpoint" or \
                final_sigmas_type != "zero" or lambda_min_clipped != -float("inf") or trained_betas is not None or \
                variance_type is not None or timestep_spacing not in ("linspace", "leading", "trailing"):
            raise NotImplementedError("only prediction_type='epsilon', solver_order 1 or 2, algorithm_type 'dpmsolver++' or "
                                      "'sde-dpmsolver++', solver_type='midpoint', final_sigmas_type='zero', "
                                      "timestep_spacing 'linspace' / 'leading' / 'trailing'; no thresholding, Karras or Lu "
                                      "sigmas, lambda_min_clipped, variance_type or trained_betas")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                                      prediction_type=prediction_type, thresholding=thresholding,
                                      dynamic_thresholding_ratio=dynamic_thresholding_ratio,
                                      sample_max_value=sample_max_value, algorithm_type=algorithm_type,
                                      solver_type=solver_type, lower_order_final=lower_order_final,
                                      euler_at_final=euler_at_final, use_karras_sigmas=use_karras_sigmas,
                                      use_lu_lambdas=use_lu_lambdas, final_sigmas_type=final_sigmas_type,
                                      lambda_min_clipped=lambda_min_clipped, variance_type=variance_type,
                                      timestep_spacing=timestep_spacing, steps_offset=steps_offset,
                                      clip_sample=clip_sample, clip_sample_range=clip_sample_range)
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.sigmas = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps,
                                                      dtype=np.float32)[::-1].copy())
        self.lower_order_nums = 0
        self._step_index = None
        self.hist = None
        self._init_noise_streams()

    @property
    def model_outputs(self):
        """diffusers' history list: the last data prediction (the device tensor `hist`) at the end once a step has run"""
        last = [self.hist] if self.lower_order_nums >= 1 else [None]
        return [None] * (self.config.solver_order - 1) + last

    @property
    def step_index(self):
        return self._step_index

    def set_timesteps(self, num_inference_steps: int, device=None):
        n_train = self.config.num_train_timesteps
        if num_inference_steps > n_train:
            raise ValueError("num_inference_steps cannot exceed num_train_timesteps")
        ts = dpm_timesteps(n_train, num_inference_steps, self.config.timestep_spacing, self.config.steps_offset)
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts).to(dtype=torch.int64)
        self.num_inference_steps = len(ts)
        self.lower_order_nums = 0
        self._step_index = None

    def scale_model_input(self, sample, timestep=None):
        return sample

    def index_for_timestep(self, timestep) -> int:
        """diffusers' rule: the position of `timestep` in the table, its second occurrence if it repeats, the last step if
        it is absent"""
        cand = (self.timesteps == _as_int(timestep)).nonzero().flatten().tolist()
        if not cand:
            return len(self.timesteps) - 1
        return cand[1] if len(cand) > 1 else cand[0]

    def _alpha_sigma(self, k: int):
        """(alpha, sigma_t, lambda) of sigmas[k] as fp32 torch scalars (diffusers' _sigma_to_alpha_sigma_t)"""
        s = self.sigmas[k]
        alpha = 1 / ((s ** 2 + 1) ** 0.5)
        sigma = s * alpha
        return alpha, sigma, torch.log(alpha) - torch.log(sigma)

    def step_order(self, k: int, restart: Optional[int] = None) -> int:
        """the order of step k of a loop that (re)starts with an empty history at step `restart` (default: the first
        step): 1 at the restart, at the last step (final sigma = 0) and for solver_order = 1; else 2"""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        last = k == self.num_inference_steps - 1
        return 1 if (self.config.solver_order == 1 or k == 0 or k == restart or last) else 2

    def step_coefficients(self, k: int, order: int):
        """(alpha_s, sigma_s, c_x, c_0, c_1, inv_r0, c_z) of step index k as Python floats (fp32 arithmetic like diffusers'
        dpm_solver_first_order_update / multistep_dpm_solver_second_order_update)"""
        alpha_t, sigma_t, lambda_t = self._alpha_sigma(k + 1)
        alpha_s, sigma_s, lambda_s = self._alpha_sigma(k)
        h = lambda_t - lambda_s
        if self.config.algorithm_type == "dpmsolver++":
            c_x, c_0, c_z = sigma_t / sigma_s, -(alpha_t * (torch.exp(-h) - 1.0)), 0.0
            c_1 = -(0.5 * (alpha_t * (torch.exp(-h) - 1.0)))
        else:
            c_x, c_0 = sigma_t / sigma_s * torch.exp(-h), alpha_t * (1 - torch.exp(-2.0 * h))
            c_1 = 0.5 * (alpha_t * (1 - torch.exp(-2.0 * h)))
            c_z = sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h))
        inv_r0 = 0.0
        if order == 2:
            lambda_s1 = self._alpha_sigma(k - 1)[2]
            inv_r0 = float(1.0 / ((lambda_s - lambda_s1) / h))
        else:
            c_1 = 0.0
        return float(alpha_s), float(sigma_s), float(c_x), float(c_0), float(c_1), inv_r0, float(c_z)

    def coefficient_table(self, timesteps=None, restart: Optional[int] = None) -> torch.Tensor:
        """[len(timesteps), 7] fp32 (CPU): step_coefficients of every step of a denoising loop over `timesteps` (default
        the whole table; a consecutive run of it), the order from step_order(k, restart) with `restart` a row of this
        table -- the device table that bg_dpm_step_tab indexes with its step counter when the loop is captured in a CUDA
        graph.  The rows depend on the neighbouring sigmas and the global step index, so a loop split into graph segments
        slices the table of the whole loop."""
        k0 = 0 if timesteps is None or len(timesteps) == 0 else self.index_for_timestep(timesteps[0])
        T = self.num_inference_steps if timesteps is None else len(timesteps)
        rows = [self.step_coefficients(k0 + j, self.step_order(k0 + j, None if restart is None else k0 + restart))
                for j in range(T)]
        return torch.tensor(rows, dtype=torch.float32).reshape(-1, 7)

    def history(self, x: torch.Tensor) -> torch.Tensor:
        """the history buffer for samples shaped like x: `hist`, reallocated (zeroed) when x's shape or device differs"""
        if self.hist is None or tuple(self.hist.shape) != tuple(x.shape) or self.hist.device != x.device:
            self.hist = torch.zeros(x.shape, dtype=torch.float32, device=x.device)
        return self.hist

    def _abar_after(self, k: int) -> torch.Tensor:
        s = self.sigmas[k + 1]
        return 1.0 / (1.0 + s * s)

    def _abar_prev(self, t: int) -> torch.Tensor:
        """abar of the level step(t) leaves x at: 1 / (1 + sigma_next^2), exactly 1 after the last step (sigma = 0).  The
        step just taken when it was at t (timesteps may repeat), else diffusers' index rule."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        k = self._step_index - 1 if self._step_index and int(self.timesteps[self._step_index - 1]) == int(t) else \
            self.index_for_timestep(t)
        return self._abar_after(k)

    def replace_table(self, timesteps) -> torch.Tensor:
        """[len(timesteps), 2] fp32 (CPU): replace_coefficients of every step of a loop over a consecutive run of the
        timestep table, row by row (repeated timesteps keep their own rows)"""
        k0 = self.index_for_timestep(timesteps[0]) if len(timesteps) else 0
        rows = []
        for j in range(len(timesteps)):
            a = self._abar_after(k0 + j)
            rows.append((float(a ** 0.5), float((1 - a) ** 0.5)))
        return torch.tensor(rows, dtype=torch.float32).reshape(-1, 2)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None,
             variance_noise: Optional[torch.Tensor] = None, return_dict: bool = True,
             model_output_uncond: Optional[torch.Tensor] = None, guidance_w: float = 0.0,
             out: Optional[torch.Tensor] = None):
        """x at the next timestep of diffusers' DPM-Solver++ step.  In SDE mode the noise comes from `variance_noise`, else
        `generator` (one, or a list with one per batch element), else the in-kernel stream (per sample after
        set_sample_keys, else batch-wide), and is drawn on every step, the last one included, as diffusers draws it.
        Extras over diffusers, as in DDIMScheduler.step: `model_output_uncond` + `guidance_w` fuse the classifier-free
        combine, `out` is the destination (may be `sample`).  pred_original_sample is not returned (None)."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        sde = self.config.algorithm_type == "sde-dpmsolver++"
        x, eps, eps_u, dst = _step_tensors("DPMSolverMultistepScheduler.step", model_output, sample, model_output_uncond,
                                           variance_noise if sde else None, out)
        if self._step_index is None:
            self._step_index = self.index_for_timestep(timestep)
        k = self._step_index
        if self.hist is None or tuple(self.hist.shape) != tuple(x.shape) or self.hist.device != x.device:
            self.lower_order_nums = 0           # a new shape restarts the solver: its history is of another sample
        hist = self.history(x)
        last = k == len(self.timesteps) - 1
        order = 1 if (self.config.solver_order == 1 or self.lower_order_nums < 1 or last) else 2
        coefs = self.step_coefficients(k, order)
        t = _as_int(timestep)
        noise, seed, offset, keys = self._step_noise(x, sde, variance_noise, generator)
        n = x.numel()
        clip = float(self.config.clip_sample_range) if self.config.clip_sample else 0.0
        with torch.cuda.device(x.device):
            _ffi.check(_ffi.lib().bg_dpm_step(eps.data_ptr(), _ffi.ptr(eps_u), float(guidance_w), x.data_ptr(),
                                             dst.data_ptr(), hist.data_ptr(), _ffi.ptr(noise), seed, offset,
                                             _ffi.ptr(keys), n // x.shape[0], t, n, *coefs, clip, _ffi.current_stream()),
                       "bg_dpm_step")
        if self.lower_order_nums < self.config.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        return SchedulerOutput(dst) if return_dict else (dst,)

    def add_noise(self, original_samples, noise, timesteps):
        return DDPMScheduler.add_noise(self, original_samples, noise, timesteps)

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
