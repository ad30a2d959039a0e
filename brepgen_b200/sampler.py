"""The diffusion half of the reference's `sample()` (sample.py:120-299), device resident.

Same stage order, tensor shapes, late face-count increase (sample.py:140-142), classifier-free guidance
(sample.py:46-51,132-134), de-duplication semantics (sample.py:159-183, 242-261), final masking and latent -> grid
reshapes (sample.py:284-294).  Differences, all result-preserving:
  * no D2H/H2D round trips: dedup runs as device kernels (csrc/dedup.cu), timesteps are device-resident views;
  * CFG combine is fused into the DDPM update kernel (PNDM steps combine with one bg_axpby); per-sample guidance
    (Guidance: a class, w and negative label per sample) combines with bg_cfg_combine before the step;
  * three schedules: "reference" = the shipped PNDM(200)[:158] + DDPM(1000)[-250:] hybrid, "ddpm" = N DDPM steps for
    every stage, which is BASELINE.json's benchmark definition (N = 1000), "ddim" = N DDIM steps for every stage
    (few-step sampling of the same DDPM-trained denoisers), "dpm" = N DPM-Solver++ steps for every stage (the
    second-order multistep sampler of the same denoisers), "unipc" = N UniPC steps for every stage (predictor-corrector,
    up to third order) and "repaint" = diffusers' RePaint list of DDIM-form steps and undo steps per stage (resampling,
    for completion).
Beyond the reference: completion (known=Completion), variations (source=Variation: SDEdit, each stage re-noised, or
DDIM-inverted, to a chosen strength and denoised again, or kept as given) and interpolation (source=Interpolation: two
designs DDIM-inverted, slerped and denoised).
Everything past sample.py:299 (OpenCASCADE post-processing) is out of scope (SURVEY.md section 2).

Batch sharding across GPUs: samples are independent through every stage, so each rank runs its own shard and there is
no collective on the hot path; `gather_outputs` is the one optional all_gather at the end.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, replace
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from . import _ffi
from .schedulers import (DPM_ALGORITHMS, UNIPC_SOLVER_TYPES, DDIMInverseScheduler, DDIMScheduler, DDPMScheduler,
                         DPMSolverMultistepScheduler, PNDMScheduler, RePaintScheduler, UniPCMultistepScheduler,
                         dpm_timesteps, repaint_entries, sample_keys, sample_seed, strength_timesteps)

NOISE_MODES = ("batch", "per_sample")

TEXT2INT = {"uncond": 0, "bathtub": 1, "bed": 2, "bench": 3, "bookshelf": 4, "cabinet": 5, "chair": 6, "couch": 7,
            "lamp": 8, "sofa": 9, "table": 10}   # sample.py:21-32


@dataclass
class CascadeConfig:
    batch_size: int = 16                 # eval_config.yaml:9
    num_surfaces: int = 50               # eval_config.yaml:12 (doubled late for non-CFG runs, sample.py:140-142)
    num_edges: int = 40                  # eval_config.yaml:13
    use_cf: bool = False
    class_label: Union[int, str, Sequence[Union[int, str]]] = 0   # TEXT2INT value or name when use_cf; a sequence: one
                                                                   # per sample (per-sample guidance, see Guidance)
    bbox_threshold: float = 0.08         # eval_config.yaml:10
    guidance_w: Union[float, Sequence[float]] = 0.6               # sample.py:49; a sequence: one per sample
    negative_label: Union[int, str, Sequence[Union[int, str]]] = 0  # label of the guidance's second row ("uncond" in
                                                                     # the reference); a sequence: one per sample
    schedule: str = "reference"          # "reference" | "ddpm" | "ddim" | "dpm" | "unipc" | "repaint"
    ddpm_steps: int = 1000               # per stage, schedule == "ddpm"
    ddim_steps: int = 50                 # per stage, schedule == "ddim"
    ddim_eta: float = 0.0                # schedule == "ddim": 0 = deterministic DDIM, 1 = DDPM-like noise
    dpm_steps: int = 20                  # per stage, schedule == "dpm"
    dpm_order: int = 2                   # schedule == "dpm": 1 (DDIM-like) or 2 (DPM-Solver++ 2M)
    dpm_algorithm: str = "dpmsolver++"   # schedule == "dpm": "dpmsolver++" (ODE) or "sde-dpmsolver++" (SDE)
    unipc_steps: int = 10                # per stage, schedule == "unipc"
    unipc_order: int = 2                 # schedule == "unipc": predictor order 1, 2 or 3 (the corrector adds one)
    unipc_solver_type: str = "bh2"       # schedule == "unipc": "bh1" or "bh2" (UniPC's B(h))
    repaint_steps: int = 250             # schedule == "repaint": N of RePaintScheduler.set_timesteps (diffusers' default)
    repaint_eta: float = 0.0             # schedule == "repaint": DDIM eta of the steps
    repaint_jump_length: int = 10        # schedule == "repaint": entries noised back up per jump
    repaint_jump_n_sample: int = 10      # schedule == "repaint": passes over each jump (1 = no resampling: DDIM-N)
    dense_masks: bool = False            # True: skip dedup, every slot valid (the dense-FLOP benchmark mode)
    ragged_masks: bool = False           # benchmark only: synthetic masks shaped like a trained model's output (random-init
                                         # weights never produce duplicates): 1/8..1/2 of the faces valid, 3..E/3 edges each
    seed: int = 0
    decode: bool = True
    graph: str = "auto"                  # "on" | "off" | "auto": capture each DDPM loop (advance, forward, fused step) in a CUDA
                                         # graph and replay it; auto = on for launch-bound shapes (few tokens, many steps)
    noise: str = "batch"                 # "batch": initial noise from a CPU generator seeded with `seed` (the reference's
                                         # draws), step noise from one Philox stream per (seed, rank, stage).  "per_sample":
                                         # every sample has its own streams, keyed by its seed, so a B-rep is a function of
                                         # (seed, global sample index) whatever the batch size or GPU count
    sample_base: int = 0                 # per_sample: global index of this batch's first sample
    sample_seeds: Optional[Sequence[int]] = None   # per_sample: one seed per sample instead of sample_seed(seed, index)


def config_from_eval_args(eval_args: dict, **overrides) -> CascadeConfig:
    """One entry of the reference's eval_config.yaml (`config[mode]`, sample.py:379-381) -> CascadeConfig, as sample()
    reads it (sample.py:39-51): batch_size, bbox_threshold, num_surfaces, num_edges, use_cf and, for classifier-free runs, the
    class label looked up in text2int (sample.py:21-32; an unknown label raises KeyError like the reference).  z_threshold
    and save_folder belong to the post-processing half (sample.py:303-368) and are ignored here."""
    use_cf = bool(eval_args["use_cf"])
    cfg = CascadeConfig(batch_size=int(eval_args["batch_size"]), num_surfaces=int(eval_args["num_surfaces"]),
                        num_edges=int(eval_args["num_edges"]), use_cf=use_cf,
                        class_label=TEXT2INT[eval_args["class_label"]] if use_cf else 0,
                        bbox_threshold=float(eval_args["bbox_threshold"]))
    for k, v in overrides.items():
        if not hasattr(cfg, k):
            raise TypeError(f"CascadeConfig has no field {k!r}")
        setattr(cfg, k, v)
    return cfg


def load_cascade(eval_args: dict, device="cuda", load=torch.load) -> "Cascade":
    """The model-loading block of sample() (sample.py:56-99): the four denoisers from `*_weight` checkpoints of state dicts
    (strict), the two decoders from the full-autoencoder checkpoints (strict=False: `encoder.*` / `quant_conv.*` are ignored),
    constructed with the reference's keyword arguments, moved to `device`, eval()."""
    from .models import EdgePosNet, EdgeZNet, SurfPosNet, SurfZNet
    from .vae import AutoencoderKL1DFastDecode, AutoencoderKLFastDecode
    use_cf = bool(eval_args["use_cf"])
    models = {}
    for name, cls, key in (("surfpos", SurfPosNet, "surfpos_weight"), ("surfz", SurfZNet, "surfz_weight"),
                           ("edgepos", EdgePosNet, "edgepos_weight"), ("edgez", EdgeZNet, "edgez_weight")):
        m = cls(use_cf)
        m.load_state_dict(load(eval_args[key]))
        models[name] = m.to(device).eval()
    surf_vae = AutoencoderKLFastDecode(
        in_channels=3, out_channels=3,
        down_block_types=["DownEncoderBlock2D", "DownEncoderBlock2D", "DownEncoderBlock2D", "DownEncoderBlock2D"],
        up_block_types=["UpDecoderBlock2D", "UpDecoderBlock2D", "UpDecoderBlock2D", "UpDecoderBlock2D"],
        block_out_channels=[128, 256, 512, 512], layers_per_block=2, act_fn="silu", latent_channels=3, norm_num_groups=32,
        sample_size=512)
    surf_vae.load_state_dict(load(eval_args["surfvae_weight"]), strict=False)
    edge_vae = AutoencoderKL1DFastDecode(
        in_channels=3, out_channels=3, down_block_types=["DownBlock1D", "DownBlock1D", "DownBlock1D"],
        up_block_types=["UpBlock1D", "UpBlock1D", "UpBlock1D"], block_out_channels=[128, 256, 512], layers_per_block=2,
        act_fn="silu", latent_channels=3, norm_num_groups=32, sample_size=512)
    edge_vae.load_state_dict(load(eval_args["edgevae_weight"]), strict=False)
    return Cascade(models, surf_vae.to(device).eval(), edge_vae.to(device).eval(), device=device)


def shard_batch(global_batch: int, rank: int, world_size: int):
    """contiguous shard [lo, hi) of the batch owned by `rank` (sizes differ by at most one)"""
    base, rem = divmod(global_batch, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_config(cfg: CascadeConfig, global_batch: int, rank: int, world_size: int) -> CascadeConfig:
    """The per-sample-noise config of `rank`'s shard of a `global_batch`-sample run: batch_size and sample_base from
    shard_batch (and its slice of cfg.sample_seeds).  N ranks running their shards generate the same B-reps as one GPU
    running cfg with batch_size = global_batch."""
    lo, hi = shard_batch(global_batch, rank, world_size)
    seeds = None
    if cfg.sample_seeds is not None:
        if len(cfg.sample_seeds) != global_batch:
            raise ValueError(f"sample_seeds has {len(cfg.sample_seeds)} entries for a batch of {global_batch}")
        seeds = list(cfg.sample_seeds)[lo:hi]
    guided = {}
    for f in GUIDANCE_FIELDS:     # per-sample guidance fields have the global length, as sample_seeds
        v = getattr(cfg, f)
        if _is_seq(v):
            if len(v) != global_batch:
                raise ValueError(f"CascadeConfig.{f} has {len(v)} entries for a batch of {global_batch}")
            guided[f] = list(v)[lo:hi]
    return replace(cfg, noise="per_sample", batch_size=hi - lo, sample_base=cfg.sample_base + lo, sample_seeds=seeds,
                   **guided)


def per_sample_seeds(cfg: CascadeConfig) -> Optional[List[int]]:
    """cfg's per-sample seeds (None in batch mode); raises on an unknown noise mode or a sample_seeds of the wrong length"""
    if cfg.noise not in NOISE_MODES:
        raise ValueError(f"CascadeConfig.noise must be one of {NOISE_MODES}, got {cfg.noise!r}")
    if cfg.noise == "batch":
        return None
    if cfg.sample_seeds is not None:
        if len(cfg.sample_seeds) != cfg.batch_size:
            raise ValueError(f"sample_seeds has {len(cfg.sample_seeds)} entries for batch_size {cfg.batch_size}")
        return [int(s) for s in cfg.sample_seeds]
    return [sample_seed(int(cfg.seed), int(cfg.sample_base) + b) for b in range(cfg.batch_size)]


GUIDANCE_FIELDS = ("class_label", "guidance_w", "negative_label")


def _is_seq(v) -> bool:
    return not isinstance(v, (str, bytes)) and (isinstance(v, Sequence) or getattr(v, "ndim", 0) > 0)


def _label(v, field: str) -> int:
    if isinstance(v, str):
        return TEXT2INT[v]            # an unknown name raises KeyError, as config_from_eval_args does
    i = int(v)
    if i != v or not 0 <= i < len(TEXT2INT):
        raise ValueError(f"CascadeConfig.{field}: label {v!r} is not an integer in [0, {len(TEXT2INT)}) (the class "
                         "embedding's rows)")
    return i


def per_sample_guidance(cfg: CascadeConfig) -> bool:
    """True when any of class_label, guidance_w and negative_label is a sequence (one entry per sample)"""
    return any(_is_seq(getattr(cfg, f)) for f in GUIDANCE_FIELDS)


def check_guidance(cfg: CascadeConfig) -> Optional[Tuple[List[int], List[int], List[float]]]:
    """raises on classifier-free guidance fields cfg cannot run (host checks only: nothing is launched): a sequence whose
    length is not batch_size, per-sample fields or a non-zero negative_label without use_cf, a label outside [0, 11) (an
    unknown name raises KeyError), a non-finite guidance_w.  Returns (class labels, negative labels, weights) with one
    entry per sample (scalars broadcast), or None without use_cf."""
    if not cfg.use_cf:
        if per_sample_guidance(cfg):
            raise ValueError("per-sample class_label, guidance_w or negative_label need a classifier-free model "
                             "(use_cf=True)")
        if _label(cfg.negative_label, "negative_label") != 0:
            raise ValueError(f"negative_label {cfg.negative_label!r} needs a classifier-free model (use_cf=True)")
        return None
    B = cfg.batch_size
    vals = []
    for f in GUIDANCE_FIELDS:
        v = getattr(cfg, f)
        if _is_seq(v):
            if len(v) != B:
                raise ValueError(f"CascadeConfig.{f} has {len(v)} entries for batch_size {B}")
            vals.append(list(v))
        else:
            vals.append([v] * B)
    cls = [_label(v, "class_label") for v in vals[0]]
    neg = [_label(v, "negative_label") for v in vals[2]]
    w = [float(v) for v in vals[1]]
    if not all(math.isfinite(v) for v in w):
        raise ValueError(f"CascadeConfig.guidance_w must be finite, got {cfg.guidance_w!r}")
    return cls, neg, w


class Guidance:
    """The classifier-free layout of a denoising loop's forward batch over n samples (n = copies of cfg's batch, e.g. the
    two designs of an interpolation, each copy guided as its sample):
      * without CFG the batch is the samples themselves;
      * scalar fields: the reference's layout, [class]*n + [negative]*n (2n rows), and the step kernels' fused combine
        with the one w;
      * per-sample fields (per_sample_guidance): the n conditional rows, then the unconditional row of each guided sample
        (w_b != 0) in batch order (n + G rows).  bg_cfg_combine combines every guided sample with its row, in place in
        the conditional half, before the step, which then runs without an uncond input; an unguided sample's eps is its
        conditional prediction, exactly what e*(1 + 0) - e_u*0 gives, without paying for the forward.
    Device state (per-sample mode): g (G,) int64 guided samples, uncond_row (n,) int32 (-1 = unguided), w (n,) fp32."""

    def __init__(self, cfg: CascadeConfig, device, n: Optional[int] = None):
        fields = check_guidance(cfg)
        self.use_cf = bool(cfg.use_cf)
        self.per_sample = per_sample_guidance(cfg)
        self.n = cfg.batch_size if n is None else int(n)
        self.device = device
        self.w = cfg.guidance_w                    # the fused kernels' weight (scalar mode; ignored without an uncond)
        self._labels, self._label = None, None
        self.G = self.n if self.use_cf else 0
        if self.per_sample:
            B = cfg.batch_size
            if self.n % B:
                raise ValueError(f"a loop over {self.n} samples is not copies of a batch of {B}")
            cls, neg, w = (v * (self.n // B) for v in fields)
            guided = [b for b in range(self.n) if w[b] != 0.0]
            row = [-1] * self.n
            for i, b in enumerate(guided):
                row[b] = i
            self.G = len(guided)
            self._labels = cls + [neg[b] for b in guided]
            self.g = torch.tensor(guided, dtype=torch.int64, device=device)
            self.uncond_row = torch.tensor(row, dtype=torch.int32, device=device)
            self.w_dev = torch.tensor(w, dtype=torch.float32, device=device)
        elif self.use_cf:
            self._labels = [fields[0][0]] * self.n + [fields[1][0]] * self.n
        self.rows = self.n + self.G                # rows of the forward batch

    @property
    def label(self) -> Optional[torch.Tensor]:
        """(rows, 1) int64 class labels of the forward batch (None without CFG)"""
        if self._label is None and self._labels is not None:
            self._label = torch.tensor(self._labels, device=self.device).reshape(-1, 1)
        return self._label

    def double(self, t: torch.Tensor) -> torch.Tensor:
        """t (n, ...) -> its rows of the forward batch: t, cat([t, t]) or cat([t, t[g]])"""
        if not self.use_cf:
            return t
        if not self.per_sample:
            return torch.cat([t, t], 0)
        return torch.cat([t, t.index_select(0, self.g)], 0) if self.G else t

    def split(self, pred: torch.Tensor):
        """(eps, eps_uncond or None, w) of a forward batch's prediction for a step kernel.  Per-sample mode combines in
        place into the conditional half (bg_cfg_combine) and returns no uncond."""
        if not self.use_cf:
            return pred, None, self.w
        if not self.per_sample:
            n = pred.shape[0] // 2
            return pred[:n], pred[n:], self.w
        pc = pred[:self.n]
        if self.G:
            if pred.dtype != torch.float32 or not pred.is_contiguous():
                raise RuntimeError("Guidance.split: the prediction must be contiguous fp32")
            _ffi.check(_ffi.lib().bg_cfg_combine(pc.data_ptr(), pred[self.n:].data_ptr(), self.uncond_row.data_ptr(),
                                                self.w_dev.data_ptr(), self.n, self.G, pc[0].numel(), pc.data_ptr(),
                                                _ffi.current_stream()), "bg_cfg_combine")
        return pc, None, 0.0

    def eps(self, pred: torch.Tensor) -> torch.Tensor:
        """the guided eps of a forward batch's prediction, for a step without a fused combine (PNDM)"""
        pc, pu, w = self.split(pred)
        if pu is None:
            return pc
        eps = torch.empty_like(pc)
        _ffi.check(_ffi.lib().bg_axpby(pc.data_ptr(), 1.0 + w, pu.data_ptr(), -w, eps.data_ptr(), eps.numel(),
                                      _ffi.current_stream()), "bg_axpby")
        return eps


def check_schedule(cfg: CascadeConfig) -> None:
    """raises ValueError on out-of-range DDIM settings (ddim_steps outside [1, 1000], ddim_eta < 0), DPM settings
    (dpm_steps outside [1, 1000], dpm_order not 1 or 2, an unknown dpm_algorithm), UniPC settings (unipc_steps outside
    [1, 1000], unipc_order not 1, 2 or 3, an unknown unipc_solver_type) and RePaint settings (repaint_steps outside
    [1, 1000], repaint_eta < 0, repaint_jump_length or repaint_jump_n_sample < 1)"""
    if cfg.schedule == "ddim":
        if not 1 <= int(cfg.ddim_steps) <= 1000:
            raise ValueError(f"CascadeConfig.ddim_steps must be in [1, 1000], got {cfg.ddim_steps}")
        if not float(cfg.ddim_eta) >= 0.0:
            raise ValueError(f"CascadeConfig.ddim_eta must be >= 0, got {cfg.ddim_eta}")
    if cfg.schedule == "dpm":
        if not 1 <= int(cfg.dpm_steps) <= 1000:
            raise ValueError(f"CascadeConfig.dpm_steps must be in [1, 1000], got {cfg.dpm_steps}")
        if cfg.dpm_order not in (1, 2):
            raise ValueError(f"CascadeConfig.dpm_order must be 1 or 2, got {cfg.dpm_order}")
        if cfg.dpm_algorithm not in DPM_ALGORITHMS:
            raise ValueError(f"CascadeConfig.dpm_algorithm must be one of {DPM_ALGORITHMS}, got {cfg.dpm_algorithm!r}")
    if cfg.schedule == "unipc":
        if not 1 <= int(cfg.unipc_steps) <= 1000:
            raise ValueError(f"CascadeConfig.unipc_steps must be in [1, 1000], got {cfg.unipc_steps}")
        if cfg.unipc_order not in (1, 2, 3):
            raise ValueError(f"CascadeConfig.unipc_order must be 1, 2 or 3, got {cfg.unipc_order}")
        if cfg.unipc_solver_type not in UNIPC_SOLVER_TYPES:
            raise ValueError(f"CascadeConfig.unipc_solver_type must be one of {UNIPC_SOLVER_TYPES}, got "
                             f"{cfg.unipc_solver_type!r}")
    if cfg.schedule == "repaint":
        if not 1 <= int(cfg.repaint_steps) <= 1000:
            raise ValueError(f"CascadeConfig.repaint_steps must be in [1, 1000], got {cfg.repaint_steps}")
        if not float(cfg.repaint_eta) >= 0.0:
            raise ValueError(f"CascadeConfig.repaint_eta must be >= 0, got {cfg.repaint_eta}")
        for f in ("repaint_jump_length", "repaint_jump_n_sample"):
            if not int(getattr(cfg, f)) >= 1:
                raise ValueError(f"CascadeConfig.{f} must be >= 1, got {getattr(cfg, f)}")


@dataclass
class Completion:
    """Known parts of a B-rep for Cascade.run(known=...): sample b keeps faces 0..n_faces[b]-1 (and, when the edge fields
    are given, their edges) and the cascade generates the rest around them.  Units are those Cascade.run returns (boxes
    already divided by 3); rows past n_faces[b] are ignored.  K <= num_surfaces, E = num_edges.
      n_faces (B,) ints; surfPos (B, K, 6); surfZ (B, K, 48) or None (latents generated for the known boxes);
      edgePos (B, K, E, 6), edge_z (B, K, E, 12), edgeV (B, K, E, 6), edge_mask (B, K, E) bool (True = padded, as edgeM):
      all four or none, and only with surfZ."""
    n_faces: Sequence[int]
    surfPos: torch.Tensor
    surfZ: Optional[torch.Tensor] = None
    edgePos: Optional[torch.Tensor] = None
    edge_z: Optional[torch.Tensor] = None
    edgeV: Optional[torch.Tensor] = None
    edge_mask: Optional[torch.Tensor] = None

    @staticmethod
    def from_outputs(out: Dict[str, torch.Tensor], n_faces: Sequence[int], edges: bool = True) -> "Completion":
        """the first n_faces[b] faces of sample b of a previous Cascade.run output (with their latents and, if `edges`,
        their edges): regenerating everything else is run(cfg, known=Completion.from_outputs(out, n))"""
        n = torch.as_tensor(n_faces, dtype=torch.int64).cpu().reshape(-1)
        nv = (~out["surfMask"]).sum(1).cpu()
        if n.numel() != nv.numel() or bool((n < 0).any()) or bool((n > nv).any()):
            raise ValueError(f"n_faces {n.tolist()} must give 0..(valid faces) per sample; valid faces: {nv.tolist()}")
        K = int(n.max()) if n.numel() else 0
        cut = lambda k: out[k][:, :K].clone()
        e = dict(edgePos=cut("edgePos"), edge_z=cut("edge_z"), edgeV=cut("edgeV"), edge_mask=cut("edgeM")) if edges else {}
        return Completion(n_faces=n.tolist(), surfPos=cut("surfPos"), surfZ=cut("surfZ"), **e)


def check_completion(cfg: CascadeConfig, known: Completion) -> torch.Tensor:
    """raises on a Completion `cfg` cannot run (host checks only; Cascade.run adds the duplicate-face check on the
    device); returns n_faces as a CPU int64 tensor"""
    if cfg.schedule == "reference":
        raise NotImplementedError("completion needs schedule='ddpm', 'ddim', 'dpm', 'unipc' or 'repaint': PNDM's Runge-Kutta "
                                  "steps advance from a sample stored earlier (cur_sample), so known tokens cannot be "
                                  "replaced between them")
    if cfg.dense_masks or cfg.ragged_masks:
        raise ValueError("completion runs the de-duplication; dense_masks and ragged_masks are benchmark modes")
    B, E = cfg.batch_size, cfg.num_edges
    n = torch.as_tensor(known.n_faces, dtype=torch.int64).cpu().reshape(-1)
    if n.numel() != B:
        raise ValueError(f"Completion.n_faces has {n.numel()} entries for batch_size {B}")

    def shape(name, t, want):
        if t is None or tuple(t.shape) != tuple(want):
            raise ValueError(f"Completion.{name} must have shape {tuple(want)}, got "
                             f"{None if t is None else tuple(t.shape)}")
    if known.surfPos is None or known.surfPos.dim() != 3:
        raise ValueError("Completion.surfPos must be a (B, K, 6) tensor")
    K = known.surfPos.shape[1]
    shape("surfPos", known.surfPos, (B, K, 6))
    if K > cfg.num_surfaces:
        raise ValueError(f"Completion has K = {K} face slots, more than num_surfaces = {cfg.num_surfaces}")
    if bool((n < 0).any()) or bool((n > K).any()):
        raise ValueError(f"Completion.n_faces must lie in [0, {K}], got {n.tolist()}")
    if known.surfZ is not None:
        shape("surfZ", known.surfZ, (B, K, 48))
    edge = [known.edgePos, known.edge_z, known.edgeV, known.edge_mask]
    if any(e is not None for e in edge):
        if not all(e is not None for e in edge):
            raise ValueError("Completion: give edgePos, edge_z, edgeV and edge_mask together, or none of them")
        if known.surfZ is None:
            raise ValueError("Completion: known edges need known surface latents (surfZ)")
        shape("edgePos", known.edgePos, (B, K, E, 6))
        shape("edge_z", known.edge_z, (B, K, E, 12))
        shape("edgeV", known.edgeV, (B, K, E, 6))
        shape("edge_mask", known.edge_mask, (B, K, E))
        if known.edge_mask.dtype != torch.bool:
            raise ValueError("Completion.edge_mask must be a bool tensor (True = padded)")
        faces = torch.arange(K)[None, :] < n[:, None]
        if bool((known.edge_mask[..., 0].cpu() & faces).any()):
            raise ValueError("Completion.edge_mask[..., 0] is set on a known face: edge slot 0 of a face is always valid")
    return n


STAGES = ("surfPos", "surfZ", "edgePos", "edgeZV")


@dataclass
class Variation:
    """A B-rep to vary with Cascade.run(source=...) (SDEdit, diffusers' img2img `strength`): each varied stage starts from
    its source noised to an intermediate timestep and runs only the rest of the schedule.  Tensors in the units and shapes
    Cascade.run returns for the cfg (boxes divided by 3): surfPos (B, S, 6), surfMask (B, S) bool, surfZ (B, S, 48),
    edgePos (B, S, E, 6), edgeM (B, S, E) bool, edge_z (B, S, E, 12), edgeV (B, S, E, 6); S = 2 * num_surfaces without
    CFG, num_surfaces with it; E = num_edges.  strength: one value in [0, 1] for all stages, or four for (surfPos, surfZ,
    edgePos, edgeZV).  1 = a fresh sample, 0 = keep the stage as given (zero strengths must come first: a later stage is
    conditioned on the earlier ones).
    start: "noise" = the source noised to the tail's first timestep with fresh z (SDEdit); "invert" = the source
    DDIM-inverted to that timestep (schedule "ddim", ddim_eta 0), deterministic: at strength 1 on every stage the run
    reconstructs the source.  The inversion runs in the stage's slot layout with the conditioning gathered from the
    source through the same maps; slots without a source take the stage's z before the inversion.  A non-CFG surfPos
    stage is inverted at the slots it starts with all the way, while its denoising doubles them at t <= 249 as a plain
    run does, so there the inversion is not the exact reverse of the denoising."""
    surfPos: torch.Tensor
    surfMask: torch.Tensor
    surfZ: torch.Tensor
    edgePos: torch.Tensor
    edgeM: torch.Tensor
    edge_z: torch.Tensor
    edgeV: torch.Tensor
    strength: Union[float, Sequence[float]] = 1.0
    start: str = "noise"

    @staticmethod
    def from_outputs(out: Dict[str, torch.Tensor], strength: Union[float, Sequence[float]],
                     start: str = "noise") -> "Variation":
        """a variation of an earlier Cascade.run output: run(cfg, source=Variation.from_outputs(out, 0.5))"""
        return Variation(*(out[k] for k in ("surfPos", "surfMask", "surfZ", "edgePos", "edgeM", "edge_z", "edgeV")),
                         strength=strength, start=start)


VARIATION_STARTS = ("noise", "invert")


@dataclass
class Interpolation:
    """Two B-reps to interpolate with Cascade.run(source=...): every stage DDIM-inverts a and b (schedule "ddim",
    ddim_eta 0) to the first timestep of its tail as one batch, slerps the two noises per sample with weight alpha[b]
    (bg_slerp: 0 = a, 1 = b) and denoises the result.  a and b are Variations with equal strengths, all > 0 (their
    `start` is not read); alpha holds one value in [0, 1] per sample.  Each design is laid out by its own pad_repeat fill
    and carried across the face de-duplication by the same survivor slots, so slot k of a is paired with slot k of b:
    faces are paired by fill order, not matched geometrically.  Slots without a source (the same in a and b) keep a's."""
    a: Variation
    b: Variation
    alpha: Union[Sequence[float], torch.Tensor]


def stage_timesteps(cfg: CascadeConfig) -> torch.Tensor:
    """the timestep list every stage of cfg's "ddpm", "ddim", "dpm" or "unipc" schedule runs (as Cascade.run sets it)"""
    if cfg.schedule in ("dpm", "unipc"):
        steps = cfg.dpm_steps if cfg.schedule == "dpm" else cfg.unipc_steps
        return torch.from_numpy(dpm_timesteps(1000, int(steps), "linspace"))
    s = DDIMScheduler() if cfg.schedule == "ddim" else DDPMScheduler()
    s.set_timesteps(int(cfg.ddim_steps if cfg.schedule == "ddim" else cfg.ddpm_steps))
    return s.timesteps


def start_slots(cfg: CascadeConfig, t0: int) -> int:
    """face slots of a plain run at timestep t0: num_surfaces before the late increase of a non-CFG run (t > 249), else S"""
    S = cfg.num_surfaces if cfg.use_cf else 2 * cfg.num_surfaces
    return cfg.num_surfaces if (not cfg.use_cf and t0 > 249) else S


def check_variation(cfg: CascadeConfig, source: Variation) -> Tuple[float, float, float, float]:
    """raises on a Variation `cfg` cannot run (host checks only: nothing is launched); returns the four stage strengths"""
    if source.start not in VARIATION_STARTS:
        raise ValueError(f"Variation.start must be one of {VARIATION_STARTS}, got {source.start!r}")
    if source.start == "invert" and (cfg.schedule != "ddim" or float(cfg.ddim_eta) != 0.0):
        raise NotImplementedError(f"DDIM inversion needs schedule 'ddim' with ddim_eta = 0, got {cfg.schedule!r} with "
                                  f"ddim_eta = {cfg.ddim_eta}: it reverses the deterministic DDIM step")
    if cfg.schedule not in ("ddpm", "ddim", "dpm", "unipc"):
        raise NotImplementedError(f"variations need schedule 'ddpm', 'ddim', 'dpm' or 'unipc', got {cfg.schedule!r}: the "
                                  "'reference' hybrid starts with PNDM's Runge-Kutta warm-up, and 'repaint' is for completion")
    if cfg.dense_masks or cfg.ragged_masks:
        raise ValueError("variations run the de-duplication; dense_masks and ragged_masks are benchmark modes")
    B, E = cfg.batch_size, cfg.num_edges
    S = cfg.num_surfaces if cfg.use_cf else 2 * cfg.num_surfaces
    want = {"surfPos": (B, S, 6), "surfMask": (B, S), "surfZ": (B, S, 48), "edgePos": (B, S, E, 6), "edgeM": (B, S, E),
            "edge_z": (B, S, E, 12), "edgeV": (B, S, E, 6)}
    for name, shape in want.items():
        t = getattr(source, name)
        if not torch.is_tensor(t) or tuple(t.shape) != shape:
            raise ValueError(f"Variation.{name} must be a tensor of shape {shape}, got "
                             f"{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}")
        if name in ("surfMask", "edgeM"):
            if t.dtype != torch.bool:
                raise ValueError(f"Variation.{name} must be a bool tensor (True = padded)")
        elif not t.dtype.is_floating_point:
            raise ValueError(f"Variation.{name} must be a floating-point tensor, got {t.dtype}")
    st = source.strength
    st = [st] * 4 if isinstance(st, (int, float)) else list(st)
    if len(st) != 4:
        raise ValueError(f"Variation.strength must be one value or four (surfPos, surfZ, edgePos, edgeZV), got {len(st)}")
    st = [float(v) for v in st]
    ts = stage_timesteps(cfg)
    for name, v in zip(STAGES, st):
        try:
            strength_timesteps(ts, v)
        except ValueError as e:
            raise ValueError(f"Variation strength of {name}: {e}") from None
    first = next((i for i, v in enumerate(st) if v > 0), 4)
    if any(v == 0 for v in st[first:]):
        raise ValueError(f"Variation strengths {st}: zero strengths must come first (a stage is conditioned on the ones "
                         "before it, so it cannot be kept while they change)")
    mask = source.surfMask.cpu()
    if source.start == "invert" and bool(mask.all(1).any()):
        raise ValueError(f"Variation: samples {torch.nonzero(mask.all(1)).flatten().tolist()} have no valid face to invert")
    if bool((source.edgeM[..., 0].cpu() & ~mask).any()):
        raise ValueError("Variation.edgeM[..., 0] is set on a valid face: edge slot 0 of a face is always valid")
    if st[0] > 0:
        t0 = int(strength_timesteps(ts, st[0])[0])
        slots = start_slots(cfg, t0)
        nv = (~mask).sum(1)
        if bool((nv > slots).any()):
            lim = max((v for v in ts.tolist() if v <= 249), default=None)
            k = len(ts) - ts.tolist().index(lim) if lim is not None else None
            hint = f"; a surfPos strength below {(k + 1) / len(ts):g} starts at t <= 249 with {S} slots" if k else ""
            raise ValueError(f"Variation: samples {torch.nonzero(nv > slots).flatten().tolist()} have more valid faces "
                             f"({nv.max().item()}) than the {slots} face slots a run has at t = {t0}, where a surfPos "
                             f"strength of {st[0]} starts{hint}")
    return tuple(st)


def check_interpolation(cfg: CascadeConfig, source: Interpolation) -> Tuple[Tuple[float, ...], torch.Tensor]:
    """raises on an Interpolation `cfg` cannot run (host checks only: nothing is launched); returns the four stage
    strengths and alpha as a CPU fp32 tensor"""
    st = []
    for name in ("a", "b"):
        v = getattr(source, name)
        if not isinstance(v, Variation):
            raise ValueError(f"Interpolation.{name} must be a Variation, got {type(v).__name__}")
        try:
            st.append(check_variation(cfg, replace(v, start="invert")))
        except ValueError as e:
            raise ValueError(f"Interpolation.{name}: {e}") from None
    if st[0] != st[1]:
        raise ValueError(f"Interpolation: a and b must have equal strengths, got {list(st[0])} and {list(st[1])}")
    if any(v == 0 for v in st[0]):
        raise ValueError(f"Interpolation strengths {list(st[0])} must all be > 0: both designs are inverted at every stage")
    alpha = torch.as_tensor(source.alpha, dtype=torch.float64).cpu().reshape(-1)
    if alpha.numel() != cfg.batch_size:
        raise ValueError(f"Interpolation.alpha has {alpha.numel()} values for batch_size {cfg.batch_size}")
    if not bool(((alpha >= 0) & (alpha <= 1)).all()):
        raise ValueError(f"Interpolation.alpha must lie in [0, 1], got {alpha.tolist()}")
    return st[0], alpha.float()


def randn_keyed(seeds: Sequence[int], stage: int, shape, device, domain: int = 1, t: int = 0) -> torch.Tensor:
    """(len(seeds), *shape[1:]) fp32 normals from the per-sample streams (bg_randn_keyed); default domain 1 = initial noise"""
    B = len(seeds)
    keys = torch.from_numpy(sample_keys(seeds, stage).view("int64")).to(device)
    out = torch.empty((B,) + tuple(shape[1:]), dtype=torch.float32, device=device)
    per = out[0].numel()
    with torch.cuda.device(out.device):
        _ffi.check(_ffi.lib().bg_randn_keyed(keys.data_ptr(), B, per, int(domain), int(t), out.data_ptr(),
                                            _ffi.current_stream()), "bg_randn_keyed")
    return out


def dedup_surfaces(surfPos: torch.Tensor, threshold: float):
    B, S, _ = surfPos.shape
    x = surfPos.float().contiguous()
    out = torch.empty_like(x)
    mask = torch.empty(B, S, dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        _ffi.check(_ffi.lib().bg_dedup_surfaces(x.data_ptr(), B, S, float(threshold), out.data_ptr(), mask.data_ptr(),
                                               _ffi.current_stream()), "bg_dedup_surfaces")
    return out, mask


def dedup_surfaces_index(surfPos: torch.Tensor, threshold: float):
    """dedup_surfaces plus the input slot of every survivor (B, S) int32, -1 past them"""
    B, S, _ = surfPos.shape
    x = surfPos.float().contiguous()
    out = torch.empty_like(x)
    mask = torch.empty(B, S, dtype=torch.bool, device=x.device)
    idx = torch.empty(B, S, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        _ffi.check(_ffi.lib().bg_dedup_surfaces_index(x.data_ptr(), B, S, float(threshold), out.data_ptr(),
                                                     mask.data_ptr(), idx.data_ptr(), _ffi.current_stream()),
                   "bg_dedup_surfaces_index")
    return out, mask, idx


def fill_index(src_mask: torch.Tensor, out_slots: int, row_map: Optional[torch.Tensor] = None) -> torch.Tensor:
    """pad_repeat gather map (bg_fill_index): src_mask (..., in_slots) bool, True = padded; row_map (rows,) int32 source
    row of each output row (-1 = none), default the identity.  Returns (rows, out_slots) int32 flat source-token indices."""
    m = src_mask.to(torch.uint8).contiguous()
    in_slots = m.shape[-1]
    n_src = m.numel() // in_slots
    rows = n_src if row_map is None else row_map.numel()
    rm = None if row_map is None else row_map.to(torch.int32).contiguous()
    out = torch.empty(rows, out_slots, dtype=torch.int32, device=m.device)
    with torch.cuda.device(m.device):
        _ffi.check(_ffi.lib().bg_fill_index(m.data_ptr(), _ffi.ptr(rm), rows, n_src, in_slots, out_slots, out.data_ptr(),
                                           _ffi.current_stream()), "bg_fill_index")
    return out


def slerp(a: torch.Tensor, b: torch.Tensor, alpha: torch.Tensor, token_mask: Optional[torch.Tensor] = None,
          out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """per-sample spherical interpolation (bg_slerp) of contiguous fp32 a, b (B, ..., D) with weights alpha (B,); tokens
    are the last dimension; token_mask (B, ...) bool or uint8, True = copied from a; out may be a"""
    B, D = a.shape[0], a.shape[-1]
    al = alpha.to(device=a.device, dtype=torch.float32).contiguous()
    m = None if token_mask is None else token_mask.to(torch.uint8).contiguous()
    out = torch.empty_like(a) if out is None else out
    with torch.cuda.device(a.device):
        _ffi.check(_ffi.lib().bg_slerp(a.data_ptr(), b.data_ptr(), al.data_ptr(), _ffi.ptr(m), B, a.numel() // B, D,
                                      out.data_ptr(), _ffi.current_stream()), "bg_slerp")
    return out


def dedup_edges(edgePos: torch.Tensor, surfMask: torch.Tensor, threshold: float):
    B, S, E, _ = edgePos.shape
    x = edgePos.float().contiguous()
    sm = surfMask.to(torch.bool).contiguous()
    mask = torch.empty(B, S, E, dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        _ffi.check(_ffi.lib().bg_dedup_edges(x.data_ptr(), sm.data_ptr(), B, S, E, float(threshold), mask.data_ptr(),
                                            _ffi.current_stream()), "bg_dedup_edges")
    return mask


class Cascade:
    """models: dict with 'surfpos', 'surfz', 'edgepos', 'edgez' drop-in denoisers (already on the device);
    surf_vae / edge_vae: drop-in decoders or None (decode skipped)."""

    def __init__(self, models: Dict[str, torch.nn.Module], surf_vae=None, edge_vae=None, device=None):
        self.m = models
        self.surf_vae, self.edge_vae = surf_vae, edge_vae
        self.device = torch.device(device if device is not None else "cuda")
        self.pndm = PNDMScheduler(num_train_timesteps=1000, beta_schedule="linear", prediction_type="epsilon",
                                  beta_start=0.0001, beta_end=0.02)
        self.ddpm = DDPMScheduler(num_train_timesteps=1000, beta_schedule="linear", prediction_type="epsilon",
                                  beta_start=0.0001, beta_end=0.02, clip_sample=True, clip_sample_range=3)
        self.ddim = DDIMScheduler(num_train_timesteps=1000, beta_schedule="linear", prediction_type="epsilon",
                                  beta_start=0.0001, beta_end=0.02, clip_sample=True, clip_sample_range=3,
                                  set_alpha_to_one=True)
        self.ddim_inv = DDIMInverseScheduler(num_train_timesteps=1000, beta_schedule="linear", prediction_type="epsilon",
                                             beta_start=0.0001, beta_end=0.02, clip_sample=True, clip_sample_range=3,
                                             set_alpha_to_one=True)
        self.dpm = self._dpm_scheduler(2, "dpmsolver++")
        self.unipc = self._unipc_scheduler(2, "bh2")
        self.repaint = RePaintScheduler(num_train_timesteps=1000, beta_schedule="linear", beta_start=0.0001,
                                        beta_end=0.02, clip_sample=True, clip_sample_range=3)

    @staticmethod
    def _dpm_scheduler(order: int, algorithm: str) -> DPMSolverMultistepScheduler:
        return DPMSolverMultistepScheduler(num_train_timesteps=1000, beta_schedule="linear", prediction_type="epsilon",
                                           beta_start=0.0001, beta_end=0.02, solver_order=order,
                                           algorithm_type=algorithm, clip_sample=True, clip_sample_range=3)

    @staticmethod
    def _unipc_scheduler(order: int, solver_type: str) -> UniPCMultistepScheduler:
        # final sigma 0: every stage ends on its data prediction, as the DDIM and DPM stages do
        return UniPCMultistepScheduler(num_train_timesteps=1000, beta_schedule="linear", prediction_type="epsilon",
                                       beta_start=0.0001, beta_end=0.02, solver_order=order, solver_type=solver_type,
                                       final_sigmas_type="zero", clip_sample=True, clip_sample_range=3)

    # ------------------------------------------------------------------ one DDPM loop as a replayed CUDA graph
    def _use_graph(self, cfg: CascadeConfig, n_steps: int, tokens: int) -> bool:
        if cfg.graph == "on":
            return True
        if cfg.graph == "off":
            return False
        # a forward is ~105 launches from Python (~1 ms of host time); below ~100 k tokens the GPU finishes sooner than that
        return n_steps >= 32 and tokens <= 100_000

    def _loop_graph(self, cfg: CascadeConfig, sched, timesteps, x, fwd, known=None, tables=None):
        """sched: self.ddpm, self.ddim, self.ddim_inv (a DDIMScheduler whose table rows are the inverse step's, sigma = 0)
        or self.dpm; timesteps: 1-D int64 CPU tensor; x: (B, ...) fp32 on the device; fwd(x_in, t_dev)
        -> eps of a (possibly CFG-doubled) batch.  The loop body of sample.py:145-153 -- [step counter / timestep advance] ->
        forward -> fused scheduler step (CFG combine, x0, clip, DDPM posterior mean or DDIM update, Philox noise) -- is
        captured ONCE and replayed len(timesteps) times: no per-step host work.  Nothing step-specific is a kernel argument:
        the timestep comes from a device scalar, the coefficients from a device table indexed by a device counter
        (bg_step_advance / bg_ddpm_step_tab / bg_ddim_step_tab / bg_dpm_step_tab), and per-sample noise from the keys at
        the device timestep.  known: {slots: (values, token mask)} of a completion; bg_replace_known_tab then follows the
        step inside the captured body.  tables: (step coefficients, replacement coefficients) of this segment, required for
        self.dpm and self.unipc, whose rows depend on the whole loop; their history buffer `hist` (and UniPC's corrected
        sample `last`) lives in the scheduler, so it carries over from one segment to the next."""
        dev = self.device
        lib = _ffi.lib()
        T = len(timesteps)
        B = x.shape[0]
        guid = Guidance(cfg, dev, B)
        xb = x.detach().float().contiguous().clone()
        n = xb.numel()
        ddim = isinstance(sched, DDIMScheduler)
        dpm = isinstance(sched, DPMSolverMultistepScheduler)
        unipc = isinstance(sched, UniPCMultistepScheduler)
        if dpm:
            coef = tables[0].to(dev)
            hist = sched.history(xb)
        elif unipc:
            coef = tables[0].to(dev)
            hist, last = sched.buffers(xb)
        else:
            coef = (sched.coefficient_table(timesteps, cfg.ddim_eta) if ddim else sched.coefficient_table(timesteps)).to(dev)
        ts = timesteps.to(device=dev, dtype=torch.int64).contiguous()
        step = torch.full((1,), -1, dtype=torch.int32, device=dev)
        t_cur = torch.zeros(1, dtype=torch.int64, device=dev)
        keyed = sched.per_sample_noise
        seed, off0, stride, keys = 0, 0, 0, None
        if keyed:     # per-sample streams counted by the device timestep t_cur: no offset to carry between graphs
            keys = sched.sample_key_tensor(B, dev)
        else:
            seed, off0, stride = sched.philox_stream(n)
        clip = float(sched.config.clip_sample_range) if sched.config.clip_sample else 0.0
        if known is not None:
            kn, km = known[xb.shape[1]]
            rtab = (tables[1] if (dpm or unipc) else sched.replace_table(timesteps)).to(dev)
            rseed = 0 if keyed else sched.replace_seed()

        def replace(st):
            if known is not None:
                _ffi.check(lib.bg_replace_known_tab(xb.data_ptr(), kn.data_ptr(), km.data_ptr(), n, xb.shape[-1], rseed,
                                                    _ffi.ptr(keys), n // B, t_cur.data_ptr(), rtab.data_ptr(),
                                                    step.data_ptr(), st), "bg_replace_known_tab")

        def body():
            st = _ffi.current_stream()
            _ffi.check(lib.bg_step_advance(ts.data_ptr(), T, step.data_ptr(), t_cur.data_ptr(), st), "bg_step_advance")
            pc, pu, w = guid.split(fwd(guid.double(xb), t_cur))
            if dpm:
                _ffi.check(lib.bg_dpm_step_tab(pc.data_ptr(), _ffi.ptr(pu), float(w), xb.data_ptr(),
                                               xb.data_ptr(), hist.data_ptr(), seed, off0, stride, _ffi.ptr(keys), n // B,
                                               t_cur.data_ptr(), n, coef.data_ptr(), step.data_ptr(), clip, st),
                           "bg_dpm_step_tab")
            elif unipc:
                _ffi.check(lib.bg_unipc_step_tab(pc.data_ptr(), _ffi.ptr(pu), float(w), xb.data_ptr(),
                                                 xb.data_ptr(), last.data_ptr(), hist.data_ptr(), n // B, n,
                                                 coef.data_ptr(), step.data_ptr(), clip, st), "bg_unipc_step_tab")
            elif ddim:
                _ffi.check(lib.bg_ddim_step_tab(pc.data_ptr(), _ffi.ptr(pu), float(w), xb.data_ptr(),
                                                xb.data_ptr(), seed, off0, stride, _ffi.ptr(keys), n // B, t_cur.data_ptr(),
                                                n, coef.data_ptr(), step.data_ptr(), clip, 0, st), "bg_ddim_step_tab")
            else:
                _ffi.check(lib.bg_ddpm_step_tab(pc.data_ptr(), _ffi.ptr(pu), float(w), xb.data_ptr(),
                                                xb.data_ptr(), seed, off0, stride, _ffi.ptr(keys), n // B, t_cur.data_ptr(),
                                                n, coef.data_ptr(), step.data_ptr(), clip, st), "bg_ddpm_step_tab")
            replace(st)

        # warm-up outside the capture (packs the weights, allocates the workspace), then rewind the state it touched
        x0 = xb.clone()
        h0 = hist.clone() if (dpm or unipc) else None
        last0 = last.clone() if unipc else None
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            body()
        torch.cuda.current_stream(dev).wait_stream(side)
        xb.copy_(x0)
        if dpm or unipc:
            hist.copy_(h0)
        if unipc:
            last.copy_(last0)
        step.fill_(-1)
        g = torch.cuda.CUDAGraph()
        l0 = lib.bg_launch_count()
        with torch.cuda.graph(g):
            body()
        per_replay = lib.bg_launch_count() - l0
        for _ in range(T):
            g.replay()
        _ffi.note_replay(per_replay, T)
        # DDIM draws (and advances the stream) only when eta > 0, DPM-Solver++ only in its SDE form, UniPC never
        draws = cfg.ddim_eta > 0 if ddim else (sched.config.algorithm_type == "sde-dpmsolver++" if dpm else not unipc)
        if not keyed and draws:
            sched.advance_philox(n, T)
        self.last_graph_steps = getattr(self, "last_graph_steps", 0) + T
        return xb

    # ------------------------------------------------------------------ one denoising loop
    def _loop(self, cfg: CascadeConfig, sched, timesteps, x, fwd, label2, gen, on_step=None, noise_fn=None, known=None,
              rnoise_fn=None):
        """fwd(x_in, t_dev) -> eps for the forward batch of x (Guidance: CFG-doubled, or with the guided samples'
        unconditional rows; label2 is not read, the forward carries its labels); noise_fn(k, shape) -> explicit DDPM / DDIM
        step noise.
        known: {slots: (values, token mask)} of a completion: the known tokens are replaced before the first step and after
        every step (sched.replace_known); rnoise_fn(k, shape) -> explicit replacement noise (k = -1 before the first step).
        sched may be self.ddim_inv with its ascending timesteps: a DDIM inversion, run as a DDIM loop that draws nothing."""
        guid = Guidance(cfg, self.device, x.shape[0])
        k = 0
        fused = isinstance(sched, (DDPMScheduler, DDIMScheduler, DPMSolverMultistepScheduler,   # CFG, noise in the kernel
                                   UniPCMultistepScheduler))
        if known is not None and len(timesteps) > 0:
            x = self._replace(sched, known, x, timesteps[0], -1, rnoise_fn, initial=True)
        if fused and noise_fn is None and rnoise_fn is None and gen is None and len(timesteps) > 0 and \
                self._use_graph(cfg, len(timesteps), x[0].numel() // x.shape[-1] * guid.rows):
            # on_step (the late face-count increase, sample.py:140-142) changes the shape once: one graph per segment
            lo = 0
            ts_list = [int(t) for t in timesteps]
            while lo < len(ts_list):
                if on_step is not None:
                    x = on_step(ts_list[lo], x)
                hi = lo + 1
                if on_step is not None:
                    while hi < len(ts_list) and on_step(ts_list[hi], x).shape == x.shape:
                        hi += 1
                else:
                    hi = len(ts_list)
                tabs = None
                if isinstance(sched, (DPMSolverMultistepScheduler, UniPCMultistepScheduler)):
                    # each segment starts the solver (first order, no UniPC corrector): the loop's first step, a
                    # variation's truncated list starting mid-table, and a segment after the late increase; rows depend
                    # on the whole loop
                    tabs = (sched.coefficient_table(timesteps, restart=lo)[lo:hi],
                            sched.replace_table(timesteps)[lo:hi])
                x = self._loop_graph(cfg, sched, timesteps[lo:hi], x, fwd, known, tabs)
                lo = hi
            return x
        ts_dev = timesteps.to(self.device)
        for i in range(len(timesteps)):
            t = timesteps[i]
            t_dev = ts_dev[i:i + 1]
            if on_step is not None:
                x = on_step(int(t), x)
            pred = fwd(guid.double(x), t_dev)
            if fused:
                pc, pu, w = guid.split(pred)
                cf = {} if pu is None else dict(model_output_uncond=pu, guidance_w=w)
                x = self._fused_step(cfg, sched, k, t, x, pc, gen, noise_fn, **cf)
            else:
                x = sched.step(guid.eps(pred), t, x).prev_sample
            if known is not None:
                x = self._replace(sched, known, x, t, k, rnoise_fn)
            k += 1
        return x

    def _replace(self, sched, known, x, t, k, rnoise_fn, initial=False):
        """known tokens of x noised to the level step k at t left it at (initial: the stage's starting level); in place on
        a step's output, on a copy of the stage's initial noise (which may be the caller's init_noise tensor)"""
        kn, km = known[x.shape[1]]
        nz = rnoise_fn(k, x.shape).to(self.device) if rnoise_fn is not None else None
        return sched.replace_known(x, kn, km, t, noise=nz, out=None if initial else x, initial=initial)

    def _fused_step(self, cfg, sched, k, t, x, pred, gen, noise_fn, **cf):
        """one DDPM, DDIM, DPM-Solver++ or UniPC step; explicit noise from noise_fn on the steps where diffusers draws it:
        DDPM at t > 0, DDIM on every step when eta > 0, DPM-Solver++ on every step of its SDE form, UniPC never"""
        if isinstance(sched, UniPCMultistepScheduler):
            return sched.step(pred, t, x, **cf).prev_sample
        if isinstance(sched, DPMSolverMultistepScheduler):
            sde = sched.config.algorithm_type == "sde-dpmsolver++"
            nz = noise_fn(k, x.shape).to(self.device) if (noise_fn is not None and sde) else None
            return sched.step(pred, t, x, generator=gen, variance_noise=nz, **cf).prev_sample
        if isinstance(sched, DDIMInverseScheduler):
            return sched.step(pred, t, x, **cf).prev_sample
        if isinstance(sched, DDIMScheduler):
            nz = noise_fn(k, x.shape).to(self.device) if (noise_fn is not None and cfg.ddim_eta > 0) else None
            return sched.step(pred, t, x, eta=cfg.ddim_eta, generator=gen, variance_noise=nz, **cf).prev_sample
        nz = noise_fn(k, x.shape).to(self.device) if (noise_fn is not None and int(t) > 0) else None
        return sched.step(pred, t, x, generator=gen, noise=nz, **cf).prev_sample

    # ------------------------------------------------------------------ RePaint: steps and undo steps in list order
    def _loop_repaint(self, cfg: CascadeConfig, sched: RePaintScheduler, x, fwd, on_step=None, noise_fn=None, known=None,
                      unoise_fn=None):
        """The loop of diffusers' RePaint pipeline over sched.timesteps: a step entry runs fwd and the fused RePaint step
        against the known tokens of x's current shape (known: {slots: (values, token mask)}, or None); an undo entry
        noises x back up from the previous entry.  on_step(t, x) is probed at every entry, so the late face-count increase
        happens once, at the first t <= 249; later jumps back above 249 keep the doubled shape.  noise_fn(k, shape) /
        unoise_fn(k, (n, *shape)) -> explicit noise of entry k (parity runs); without them a launch-bound stage runs as
        two replayed CUDA graphs per segment."""
        ts = sched.timesteps
        ents = repaint_entries(ts)
        dev = self.device
        guid = Guidance(cfg, dev, x.shape[0])
        tokens = x[0].numel() // x.shape[-1] * guid.rows
        if noise_fn is None and unoise_fn is None and len(ents) > 0 and self._use_graph(cfg, len(ents), tokens):
            tables = (sched.coefficient_table().to(dev), sched.undo_table().to(dev),
                      ts.to(device=dev, dtype=torch.int64).contiguous())
            lo = 0
            while lo < len(ents):
                if on_step is not None:
                    x = on_step(int(ts[lo]), x)
                hi = lo + 1
                while hi < len(ents) and (on_step is None or on_step(int(ts[hi]), x).shape == x.shape):
                    hi += 1
                x = self._loop_graph_repaint(cfg, sched, ents, lo, hi, x, fwd, known, tables)
                lo = hi
            return x
        ts_dev = ts.to(dev)
        for k, (is_step, t) in enumerate(ents):
            if on_step is not None:
                x = on_step(int(ts[k]), x)
            if is_step:
                kn, km = known[x.shape[1]] if known is not None else (None, None)
                nz = noise_fn(k, x.shape).to(dev) if noise_fn is not None else None
                pc, pu, w = guid.split(fwd(guid.double(x), ts_dev[k:k + 1]))
                cf = {} if pu is None else dict(model_output_uncond=pu, guidance_w=w)
                x = sched.step(pc, t, x, kn, km, noise=nz, **cf).prev_sample
            else:
                nz = unoise_fn(k, (sched.undo_transitions,) + tuple(x.shape)).to(dev) if unoise_fn is not None else None
                x = sched.undo_step(x, t, noise=nz, out=x)
        return x

    def _loop_graph_repaint(self, cfg, sched, ents, lo, hi, x, fwd, known, tables):
        """entries lo..hi-1 of a stage's RePaint list (one shape) as two captured bodies sharing the entry counter `step`
        and t_cur: advance -> forward -> bg_repaint_step_tab, and advance -> bg_repaint_undo_tab, replayed in list order.
        The counter runs over the whole list (it starts at lo - 1), so the tables (step coefficients, undo coefficients,
        timesteps) are those of the whole stage and the noise counters are the eager loop's."""
        dev = self.device
        lib = _ffi.lib()
        coef, utab, ts = tables
        T = len(ents)
        B = x.shape[0]
        guid = Guidance(cfg, dev, B)
        xb = x.detach().float().contiguous().clone()
        n = xb.numel()
        step = torch.full((1,), lo - 1, dtype=torch.int32, device=dev)
        t_cur = torch.zeros(1, dtype=torch.int64, device=dev)
        keys = sched.sample_key_tensor(B, dev) if sched.per_sample_noise else None
        s3, s4 = (0, 0) if keys is not None else (sched.repaint_seed(3), sched.repaint_seed(4))
        clip = float(sched.config.clip_sample_range) if sched.config.clip_sample else 0.0
        kn, km = known[xb.shape[1]] if known is not None else (None, None)
        nt = sched.undo_transitions

        def advance(st):
            _ffi.check(lib.bg_step_advance(ts.data_ptr(), T, step.data_ptr(), t_cur.data_ptr(), st), "bg_step_advance")

        def step_body():
            st = _ffi.current_stream()
            advance(st)
            pc, pu, w = guid.split(fwd(guid.double(xb), t_cur))
            _ffi.check(lib.bg_repaint_step_tab(pc.data_ptr(), _ffi.ptr(pu), float(w), xb.data_ptr(),
                                               xb.data_ptr(), _ffi.ptr(kn), _ffi.ptr(km), xb.shape[-1], s3,
                                               _ffi.ptr(keys), n // B, n, coef.data_ptr(), step.data_ptr(), clip, st),
                       "bg_repaint_step_tab")

        def undo_body():
            st = _ffi.current_stream()
            advance(st)
            _ffi.check(lib.bg_repaint_undo_tab(xb.data_ptr(), n, nt, s4, _ffi.ptr(keys), n // B, utab.data_ptr(),
                                               step.data_ptr(), st), "bg_repaint_undo_tab")

        # warm-up outside the capture (packs the weights, allocates the workspace), then rewind the state it touched
        x0 = xb.clone()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            step_body()
        torch.cuda.current_stream(dev).wait_stream(side)
        xb.copy_(x0)
        step.fill_(lo - 1)
        kinds = [ents[k][0] for k in range(lo, hi)]
        graphs, per_replay = {}, {}
        for is_step, body in ((True, step_body), (False, undo_body)):
            if is_step in kinds:
                g = torch.cuda.CUDAGraph()
                l0 = lib.bg_launch_count()
                with torch.cuda.graph(g):
                    body()
                graphs[is_step], per_replay[is_step] = g, lib.bg_launch_count() - l0
        for is_step in kinds:
            graphs[is_step].replay()
        for is_step in graphs:
            _ffi.note_replay(per_replay[is_step], kinds.count(is_step))
        self.last_graph_steps = getattr(self, "last_graph_steps", 0) + (hi - lo)
        return xb

    _STAGE_ID = {"surfPos": 0, "surfZ": 1, "edgePos": 2, "edgeZV": 3}

    def _stage(self, cfg, x, fwd, label2, gen, hybrid_ddpm_tail: bool, on_step=None, noise_fn=None, name="surfPos",
               known=None, rnoise_fn=None, unoise_fn=None, timesteps=None):
        """one stage's denoising loop from x; timesteps: a tail of the schedule's list to run instead of all of it (a
        variation; schedules "ddpm", "ddim", "dpm" and "unipc")"""
        seeds = getattr(self, "_sample_seeds", None)
        if cfg.schedule == "dpm" and (self.dpm.config.solver_order, self.dpm.config.algorithm_type) != \
                (cfg.dpm_order, cfg.dpm_algorithm):
            self.dpm = self._dpm_scheduler(cfg.dpm_order, cfg.dpm_algorithm)
        if cfg.schedule == "unipc" and (self.unipc.config.solver_order, self.unipc.config.solver_type) != \
                (cfg.unipc_order, cfg.unipc_solver_type):
            self.unipc = self._unipc_scheduler(cfg.unipc_order, cfg.unipc_solver_type)
        noisy = {"ddim": self.ddim, "dpm": self.dpm, "unipc": self.unipc, "repaint": self.repaint}.get(cfg.schedule,
                                                                                                      self.ddpm)
        if seeds is not None:
            noisy.set_sample_keys(sample_seeds=seeds, stage=self._STAGE_ID[name])
        else:
            noisy.set_noise_seed(*getattr(self, "_noise_key", (int(cfg.seed), 0)), self._STAGE_ID[name])
        if cfg.schedule == "ddim":
            self.ddim.set_timesteps(cfg.ddim_steps)
            ts = self.ddim.timesteps if timesteps is None else timesteps
            return self._loop(cfg, self.ddim, ts, x, fwd, label2, gen, on_step, noise_fn, known, rnoise_fn)
        if cfg.schedule == "dpm":
            self.dpm.set_timesteps(cfg.dpm_steps)
            ts = self.dpm.timesteps if timesteps is None else timesteps
            return self._loop(cfg, self.dpm, ts, x, fwd, label2, gen, on_step, noise_fn, known, rnoise_fn)
        if cfg.schedule == "unipc":
            self.unipc.set_timesteps(cfg.unipc_steps)
            ts = self.unipc.timesteps if timesteps is None else timesteps
            return self._loop(cfg, self.unipc, ts, x, fwd, label2, gen, on_step, noise_fn, known, rnoise_fn)
        if cfg.schedule == "repaint":
            self.repaint.eta = float(cfg.repaint_eta)
            self.repaint.set_timesteps(cfg.repaint_steps, cfg.repaint_jump_length, cfg.repaint_jump_n_sample)
            return self._loop_repaint(cfg, self.repaint, x, fwd, on_step, noise_fn, known, unoise_fn)
        if cfg.schedule == "ddpm":
            self.ddpm.set_timesteps(cfg.ddpm_steps)
            ts = self.ddpm.timesteps if timesteps is None else timesteps
            return self._loop(cfg, self.ddpm, ts, x, fwd, label2, gen, on_step, noise_fn, known, rnoise_fn)
        # the shipped hybrid: PNDM(200) then, for the position stages, DDPM(1000)[-250:]
        self.pndm.set_timesteps(200)
        ts = self.pndm.timesteps[:158] if hybrid_ddpm_tail else self.pndm.timesteps
        x = self._loop(cfg, self.pndm, ts, x, fwd, label2, gen)
        if hybrid_ddpm_tail:
            if on_step is not None:
                x = on_step(-1, x)
            self.ddpm.set_timesteps(1000)
            x = self._loop(cfg, self.ddpm, self.ddpm.timesteps[-250:], x, fwd, label2, gen, None, noise_fn)
        return x

    # ------------------------------------------------------------------ completion
    def _known_tensors(self, cfg: CascadeConfig, known: Completion, n: torch.Tensor) -> dict:
        """device tensors of a checked Completion: per stage {slots: (model-unit values, uint8 token mask)}, plus the face
        mask 'face' (B, S), the given edge masks 'edgeM' and the given outputs 'out' to write through.  Raises ValueError
        when known faces of a sample duplicate each other under the de-duplication rule (bg_dedup_surfaces on the
        model-unit boxes): the de-duplication would then drop a known face."""
        dev = self.device
        B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
        S = S0 if cfg.use_cf else 2 * S0
        K = known.surfPos.shape[1]
        nd = n.to(dev)
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()

        def pad(t, slots):            # (B, K, ...) -> (B, slots, ...), zero past K
            p = torch.zeros((B, slots) + tuple(t.shape[2:]), dtype=t.dtype, device=dev)
            p[:, :K] = t.to(dev)
            return p
        face = lambda slots: torch.arange(slots, device=dev)[None, :] < nd[:, None]
        pos = f32(known.surfPos) * 3.0
        if K > 0 and bool((n > 1).any()):
            rows = torch.where(face(K)[..., None], pos, pos[:, :1])    # past n_faces: copies of face 0, always dropped
            _, m = dedup_surfaces(rows, cfg.bbox_threshold)
            bad = (m & face(K)).any(1).cpu()
            if bool(bad.any()):
                raise ValueError(f"Completion: known faces of samples {torch.nonzero(bad).flatten().tolist()} duplicate "
                                 f"each other under the de-duplication rule (bbox_threshold {cfg.bbox_threshold})")
        u8 = lambda m: m.to(torch.uint8).contiguous()
        kn = {"face": face(S), "out": {"surfPos": pad(f32(known.surfPos), S)}}
        kn["surfPos"] = {S0: (pad(pos, S0), u8(face(S0)))}
        if not cfg.use_cf:            # the late increase doubles the slots: both copies stay known
            kn["surfPos"][2 * S0] = (pad(pos, S0).repeat(1, 2, 1), u8(face(S0).repeat(1, 2)))
        if known.surfZ is not None:
            kn["surfZ"] = {S: (pad(f32(known.surfZ), S), u8(face(S)))}
            kn["out"]["surfZ"] = kn["surfZ"][S][0]
        if known.edgePos is not None:
            em = u8(face(S)[..., None].expand(B, S, E))
            kn["edgePos"] = {S: (pad(f32(known.edgePos) * 3.0, S), em)}
            zv = torch.cat([f32(known.edge_z), f32(known.edgeV)], -1)
            kn["edgeZV"] = {S: (pad(zv, S), em)}
            kn["edgeM"] = pad(known.edge_mask.to(torch.bool), S)
            kn["out"].update(edgePos=pad(f32(known.edgePos), S), edgeM=kn["edgeM"], edge_z=pad(f32(known.edge_z), S),
                             edgeV=pad(f32(known.edgeV), S))
        return kn

    # ------------------------------------------------------------------ variations
    def _vary_start(self, name, shape, src, index, scale, t0, init_noise, seeds, cpu_gen, copies=1):
        """the start of a varied stage (bg_add_noise_gather): sa*(scale*src[index]) + sb*z with (sa, sb) of add_noise at
        t0, or (1, 0) when t0 is None (the gathered source itself, which an inversion starts from); index (int32, one per
        token of `shape`) into the tokens of src, -1 = pure noise.  z: init_noise[name], else the per-sample keys of the
        stage drawn in the kernel (bg_randn_keyed's initial noise), else the CPU generator.  copies: index holds that many
        maps of `shape` one after the other, and each copy of the output takes the same z."""
        dev = self.device
        dim = shape[-1]
        out = torch.empty((copies * shape[0],) + tuple(shape[1:]), dtype=torch.float32, device=dev)
        n_tok = out.numel() // dim
        z = keys = None
        if init_noise is not None and name in init_noise:
            z = init_noise[name].to(device=dev, dtype=torch.float32).contiguous()
            if tuple(z.shape) != tuple(shape):
                raise ValueError(f"init_noise[{name!r}] has shape {tuple(z.shape)}; this variation starts at {tuple(shape)}")
        elif seeds is not None:
            keys = torch.from_numpy(sample_keys(seeds, self._STAGE_ID[name]).view("int64")).to(dev)
        else:
            z = torch.randn(shape, generator=cpu_gen).to(dev)
        if copies > 1:
            z, keys = (None if v is None else torch.cat([v] * copies) for v in (z, keys))
        sa, sb = (1.0, 0.0) if t0 is None else self.ddpm.replace_coefficients(t0, initial=True)
        src = src.reshape(-1, dim)
        idx = index.to(torch.int32).contiguous()
        with torch.cuda.device(dev):
            _ffi.check(_ffi.lib().bg_add_noise_gather(src.data_ptr(), src.shape[0], idx.data_ptr(), n_tok, dim,
                                                     float(scale), sa, sb, _ffi.ptr(z), _ffi.ptr(keys), n_tok // out.shape[0],
                                                     1, 0, out.data_ptr(), _ffi.current_stream()), "bg_add_noise_gather")
        return out

    def _invert_start(self, cfg, name, shape, srcs, maps, scale, tail, fwd, alpha, init_noise, seeds, cpu_gen):
        """the start of a stage of an inverted variation (one source) or an interpolation (two): every source gathered
        through its own map (maps: one (B, ...) int32 map per source; -1 slots take the stage's z), DDIM-inverted as one
        batch along the reversed tail, so that it lands at the tail's first timestep, by fwd(x, t) with the conditioning
        of that batch; two sources are then slerped with weights alpha, tokens without a source copied from the first."""
        B = shape[0]
        off = [0]
        for s in srcs[:-1]:
            off.append(off[-1] + s[name].numel() // shape[-1])
        src = torch.cat([s[name].reshape(-1, shape[-1]) for s in srcs])
        index = torch.cat([torch.where(i >= 0, i + o, i) for i, o in zip(maps, off)])
        x = self._vary_start(name, shape, src, index, scale, None, init_noise, seeds, cpu_gen, copies=len(srcs))
        self.ddim_inv.set_timesteps(cfg.ddim_steps)
        x = self._loop(cfg, self.ddim_inv, tail.flip(0), x, fwd, None, None)
        if len(srcs) == 2:
            x = slerp(x[:B], x[B:], alpha, maps[0] < 0, out=x[:B])
        return x

    # ------------------------------------------------------------------ the cascade
    @torch.no_grad()
    def run(self, cfg: CascadeConfig, init_noise: Optional[Dict[str, torch.Tensor]] = None, step_noise=None,
            known: Optional[Completion] = None, replace_noise=None, undo_noise=None,
            source: Optional[Union[Variation, Interpolation]] = None):
        """step_noise(stage_name, k, shape) -> tensor: explicit DDPM / DDIM / DPM step noise of step k (parity runs; DDPM
        draws it at t > 0, DDIM on every step when ddim_eta > 0, DPM on every step of "sde-dpmsolver++"); default = in-kernel
        Philox
        keyed by (cfg.seed, rank, stage): reproducible from cfg.seed, independent across ranks and stages.
        cfg.noise == "per_sample": initial and step noise come from each sample's own streams (bg_randn_keyed and the fused
        steps' sample keys), so sample b's outputs depend on its seed alone; init_noise / step_noise still take precedence.
        known: a Completion (schedules "ddpm", "ddim", "dpm" and "unipc"): every stage that has known tokens replaces them before its
        first step and after every step with the known values noised to the step's level, so the rest is generated
        around them; the known parts come out as given, bit for bit.  replace_noise(stage_name, k, shape) -> tensor:
        explicit noise of that replacement (k = -1 before the first step; parity runs), mirroring step_noise.
        source: a Variation (schedules "ddpm", "ddim", "dpm" and "unipc"; not with known): each stage with strength s > 0 starts
        from its source noised to the first timestep of strength_timesteps(list, s) and runs that tail of the list; a
        stage with strength 0 is not run and returns the source as given, bit for bit.  A varied stage's slots take
        their source tokens in the trainers' pad_repeat layout (bg_fill_index), across the face de-duplication
        (bg_dedup_surfaces_index); slots without a source start from pure noise.  init_noise[name] is the start noise z
        of a varied stage (shape: the stage's starting shape).  Variation(start="invert") and source=Interpolation
        (schedule "ddim", ddim_eta 0): a varied stage starts from its source (both sources) DDIM-inverted along the
        reversed tail instead (self.ddim_inv through the same loops), then slerped (bg_slerp) for an interpolation; z only
        fills the slots without a source, so neither draws any other noise.
        schedule "repaint": step_noise(stage_name, k, shape) is the one z of the step at list entry k (drawn at every
        step); undo_noise(stage_name, k, (n, *shape)) the normals of the undo step at entry k.  Known tokens are kept by
        the RePaint step itself (no separate replacement: replace_noise is not used), and known=None is DDIM with
        resampling."""
        check_schedule(cfg)
        check_guidance(cfg)
        if source is not None and known is not None:
            raise ValueError("Cascade.run: a variation (source=) cannot be combined with a completion (known=)")
        n_known = check_completion(cfg, known) if known is not None else None
        interp = isinstance(source, Interpolation)
        alpha = None
        if interp:
            strength, alpha = check_interpolation(cfg, source)
        else:
            strength = check_variation(cfg, source) if source is not None else None
        seeds = per_sample_seeds(cfg)
        self._sample_seeds = seeds
        dev = self.device
        rank = 0
        try:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                rank = dist.get_rank()
        except Exception:
            pass
        self._noise_key = (int(cfg.seed), rank)
        nf = (lambda name: (lambda k, shape: step_noise(name, k, shape))) if step_noise is not None else (lambda name: None)
        rnf = (lambda name: (lambda k, shape: replace_noise(name, k, shape))) if replace_noise is not None else \
            (lambda name: None)
        unf = (lambda name: (lambda k, shape: undo_noise(name, k, shape))) if undo_noise is not None else \
            (lambda name: None)
        gen = None
        B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
        S = S0 if cfg.use_cf else 2 * S0
        kn = self._known_tensors(cfg, known, n_known) if known is not None else {}
        cpu_gen = torch.Generator().manual_seed(cfg.seed)             # initial noise: CPU generator (utils.py:62-97)
        guid = Guidance(cfg, dev)     # the forward batch of every stage: its labels, and rep2 of the conditioning
        label2 = guid.label

        def noise(name, shape):
            if init_noise is not None and name in init_noise:
                return init_noise[name].to(dev).float()
            if seeds is not None:
                return randn_keyed(seeds, self._STAGE_ID[name], shape, dev)
            return torch.randn(shape, generator=cpu_gen).to(dev)

        rep2 = guid.double

        # STEP 1-1 surface positions (sample.py:126-153)
        def late_increase(t, x):
            # non-CFG runs double the face slots once the DDPM tail (t < 250) starts (sample.py:140-142).  Pure function of
            # (t, shape): the graph path probes it to find the segment boundaries.
            if not cfg.use_cf and x.shape[1] == S0 and (t < 0 or t <= 249):
                return x.repeat(1, 2, 1)
            return x

        # a variation: the source on the device, the tail of the list each varied stage runs (None: kept), and where the
        # start of each varied stage takes its tokens from (flat source-token indices, -1 = none)
        # an interpolation: both designs, each with its own maps, inverted as one batch of 2B and slerped
        var = source is not None
        sources = [source.a, source.b] if interp else [source]
        invert = interp or (var and source.start == "invert")
        tails, srcs = {}, []
        if var:
            full = stage_timesteps(cfg)
            tails = {name: strength_timesteps(full, v) if v > 0 else None for name, v in zip(STAGES, strength)}
            for v in sources:
                s = {}
                for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV", "surfMask", "edgeM"):
                    t = getattr(v, k)
                    s[k] = t.to(device=dev, dtype=t.dtype if t.dtype == torch.bool else torch.float32,
                                copy=True).contiguous()
                s["edgeZV"] = torch.cat([s["edge_z"], s["edgeV"]], -1)
                srcs.append(s)
        src = srcs[0] if var else {}
        kept = lambda name: var and tails[name] is None
        # the inversion's batch: every source's copy of sample b is inverted under sample b's guidance
        inv = Guidance(cfg, dev, len(srcs) * B) if invert else None
        label_inv = inv.label if invert else None

        def take(field, maps, scale=1.0):
            # the inversion's conditioning: each source's field gathered through its map (0 where -1), one batch
            return inv.double(torch.cat([torch.where((i >= 0)[..., None], s[field].reshape(-1, s[field].shape[-1])[
                i.long().clamp(min=0)] * scale, 0.0) for s, i in zip(srcs, maps)]))

        def holes(maps):
            return inv.double(torch.cat([i < 0 for i in maps]))

        def vary(name, shape, maps, scale, model, cond=tuple):
            """maps: one index map per source; model, cond(): the denoiser and its conditioning for an inversion"""
            if not invert:
                return self._vary_start(name, shape, src[name], maps[0], scale, int(tails[name][0]), init_noise, seeds,
                                        cpu_gen)
            c = cond()
            return self._invert_start(cfg, name, shape, srcs, maps, scale, tails[name],
                                      lambda x, t: self.m[model](x, t, *c, label_inv), alpha, init_noise, seeds,
                                      cpu_gen)

        mask_gen = torch.Generator().manual_seed(cfg.seed + 12345)
        if kept("surfPos"):
            surfPos, surfMask = src["surfPos"] * 3.0, src["surfMask"]
            rows = [torch.where(surfMask, -1, torch.arange(B * S, dtype=torch.int32, device=dev).view(B, S))]
        else:
            if var:       # the source's valid faces repeated to the slots a plain run has at the first timestep
                S1 = start_slots(cfg, int(tails["surfPos"][0]))
                fill = [fill_index(s["surfMask"], S1) for s in srcs]
            surfPos = vary("surfPos", (B, S1, 6), fill, 3.0, "surfpos") if var else noise("surfPos", (B, S0, 6))
            surfPos = self._stage(cfg, surfPos, lambda x, t: self.m["surfpos"](x, t, label2), label2, gen, True,
                                  on_step=late_increase, noise_fn=nf("surfPos"), name="surfPos", known=kn.get("surfPos"),
                                  rnoise_fn=rnf("surfPos"), unoise_fn=unf("surfPos"), timesteps=tails.get("surfPos"))
            if not cfg.use_cf and surfPos.shape[1] == S0:
                surfPos = surfPos.repeat(1, 2, 1)

            # STEP 1-2 duplicate faces (sample.py:159-183)
            if cfg.ragged_masks:
                nv = torch.randint(max(1, S // 8), max(2, S // 2) + 1, (B,), generator=mask_gen)
                surfMask = (torch.arange(S)[None, :] >= nv[:, None]).to(dev)
            elif cfg.dense_masks:
                surfMask = torch.zeros(B, S, dtype=torch.bool, device=dev)
            elif var:     # survivor k came from slot idx[k], which the late increase's repeat took from fill slot idx % S1
                surfPos, surfMask, idx = dedup_surfaces_index(surfPos, cfg.bbox_threshold)
                i = idx.long()
                rows = [torch.where(i >= 0, f.gather(1, i.clamp(min=0) % S1), -1) for f in fill]
            else:
                surfPos, surfMask = dedup_surfaces(surfPos, cfg.bbox_threshold)
        sP, sM = rep2(surfPos), rep2(surfMask)

        # STEP 1-3 surface latents (sample.py:189-202)
        if kept("surfZ"):
            surfZ = src["surfZ"]
        else:
            surfZ = vary("surfZ", (B, S, 48), rows, 1.0, "surfz", lambda: (take("surfPos", rows, 3.0), holes(rows))) \
                if var else noise("surfZ", (B, S, 48))
            surfZ = self._stage(cfg, surfZ, lambda x, t: self.m["surfz"](x, t, sP, sM, label2), label2, gen, False,
                                noise_fn=nf("surfZ"), name="surfZ", known=kn.get("surfZ"), rnoise_fn=rnf("surfZ"),
                                unoise_fn=unf("surfZ"), timesteps=tails.get("surfZ"))
        sZ = rep2(surfZ)

        # STEP 2-1 edge positions (sample.py:208-236)
        if kept("edgePos"):
            edgePos, edgeM = src["edgePos"] * 3.0, src["edgeM"]
            edges = [torch.arange(B * S * E, dtype=torch.int32, device=dev).view(B, S, E)]
        else:
            if var:       # the valid edges of each face's source face, repeated to E slots
                edges = [fill_index(s["edgeM"], E, r.flatten()).view(B, S, E) for s, r in zip(srcs, rows)]
            edgePos = vary("edgePos", (B, S, E, 6), edges, 3.0, "edgepos",
                           lambda: (take("surfPos", rows, 3.0), take("surfZ", rows), holes(rows))) \
                if var else noise("edgePos", (B, S, E, 6))
            edgePos = self._stage(cfg, edgePos, lambda x, t: self.m["edgepos"](x, t, sP, sZ, sM, label2), label2, gen,
                                  True, noise_fn=nf("edgePos"), name="edgePos", known=kn.get("edgePos"),
                                  rnoise_fn=rnf("edgePos"), unoise_fn=unf("edgePos"), timesteps=tails.get("edgePos"))

            # STEP 2-2 duplicate edges per face (sample.py:242-261)
            if cfg.ragged_masks:
                ne = torch.randint(min(3, E), max(min(3, E), E // 3) + 1, (B, S), generator=mask_gen)
                edgeM = (torch.arange(E)[None, None, :] >= ne[..., None]).to(dev) | surfMask[..., None]
            elif cfg.dense_masks:
                edgeM = torch.zeros(B, S, E, dtype=torch.bool, device=dev)
            else:
                edgeM = dedup_edges(edgePos, surfMask, cfg.bbox_threshold)
        if "edgeM" in kn:             # the known faces keep their given edge masks
            edgeM = torch.where(kn["face"][..., None], kn["edgeM"], edgeM)
        eP, eM = rep2(edgePos), rep2(edgeM)

        # STEP 2-3 edge latents + vertices (sample.py:267-286)
        if kept("edgeZV"):
            edgeZV = src["edgeZV"]
        else:
            edgeZV = vary("edgeZV", (B, S, E, 18), edges, 1.0, "edgez",
                          lambda: (take("edgePos", edges, 3.0), take("surfPos", rows, 3.0), take("surfZ", rows),
                                   holes(edges))) if var else noise("edgeZV", (B, S, E, 18))
            edgeZV = self._stage(cfg, edgeZV, lambda x, t: self.m["edgez"](x, t, eP, sP, sZ, eM, label2), label2, gen,
                                 False, noise_fn=nf("edgeZV"), name="edgeZV", known=kn.get("edgeZV"),
                                 rnoise_fn=rnf("edgeZV"), unoise_fn=unf("edgeZV"), timesteps=tails.get("edgeZV"))
            edgeZV = edgeZV.masked_fill(edgeM.unsqueeze(-1), 0.0)
        edge_z, edgeV = edgeZV[..., :12], edgeZV[..., 12:]

        out = {"surfPos": surfPos / 3.0, "surfMask": surfMask, "surfZ": surfZ, "edgePos": edgePos / 3.0, "edgeM": edgeM,
               "edge_z": edge_z.contiguous(), "edgeV": edgeV.contiguous()}
        if kn:                        # the given values of the known faces, written through (the decoders see them too)
            for k, v in kn["out"].items():
                f = kn["face"].reshape(kn["face"].shape + (1,) * (v.dim() - 2))
                out[k] = torch.where(f, v, out[k]).contiguous()
            surfZ, edge_z = out["surfZ"], out["edge_z"]
        if var:                       # kept stages return the source as given (the decoders see it too)
            fields = {"surfPos": ("surfPos", "surfMask"), "surfZ": ("surfZ",), "edgePos": ("edgePos", "edgeM"),
                      "edgeZV": ("edge_z", "edgeV")}
            for name in STAGES:
                if kept(name):
                    out.update({k: src[k] for k in fields[name]})
            surfZ, edge_z = out["surfZ"], out["edge_z"]
        # decoders (sample.py:289-294)
        if cfg.decode and self.surf_vae is not None:
            z = surfZ.unflatten(-1, (16, 3)).flatten(0, 1).permute(0, 2, 1).unflatten(-1, (4, 4))
            out["surf_ncs"] = self.surf_vae(z).permute(0, 2, 3, 1).unflatten(0, (B, S))
        if cfg.decode and self.edge_vae is not None:
            z = edge_z.unflatten(-1, (4, 3)).reshape(-1, 4, 3).permute(0, 2, 1)
            out["edge_ncs"] = self.edge_vae(z).permute(0, 2, 1).reshape(B, S, E, 32, 3)
        return out


def gather_outputs(out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """optional final all_gather of every output tensor along the batch dimension (equal shard sizes)"""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return out
    ws = dist.get_world_size()
    res = {}
    for k, v in out.items():
        v = v.contiguous()
        as_u8 = v.dtype == torch.bool
        if as_u8:
            v = v.to(torch.uint8)
        bufs = [torch.empty_like(v) for _ in range(ws)]
        dist.all_gather(bufs, v)
        g = torch.cat(bufs, 0)
        res[k] = g.to(torch.bool) if as_u8 else g
    return res
