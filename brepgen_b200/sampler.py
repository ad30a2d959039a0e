"""The diffusion half of the reference's `sample()` (sample.py:120-299), device resident.

Same stage order, tensor shapes, late face-count increase (sample.py:140-142), classifier-free guidance
(sample.py:46-51,132-134), de-duplication semantics (sample.py:159-183, 242-261), final masking and latent -> grid
reshapes (sample.py:284-294).  Differences, all result-preserving:
  * no D2H/H2D round trips: dedup runs as device kernels (csrc/dedup.cu), timesteps are device-resident views;
  * CFG combine is fused into the DDPM update kernel (PNDM steps combine with one bg_axpby);
  * two schedules: "reference" = the shipped PNDM(200)[:158] + DDPM(1000)[-250:] hybrid, and "ddpm" = N DDPM steps for
    every stage, which is BASELINE.json's benchmark definition (N = 1000).
Everything past sample.py:299 (OpenCASCADE post-processing) is out of scope (SURVEY.md section 2).

Batch sharding across GPUs: samples are independent through every stage, so each rank runs its own shard and there is
no collective on the hot path; `gather_outputs` is the one optional all_gather at the end.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import torch

from . import _ffi
from .schedulers import DDPMScheduler, PNDMScheduler

TEXT2INT = {"uncond": 0, "bathtub": 1, "bed": 2, "bench": 3, "bookshelf": 4, "cabinet": 5, "chair": 6, "couch": 7,
            "lamp": 8, "sofa": 9, "table": 10}   # sample.py:21-32


@dataclass
class CascadeConfig:
    batch_size: int = 16                 # eval_config.yaml:9
    num_surfaces: int = 50               # eval_config.yaml:12 (doubled late for non-CFG runs, sample.py:140-142)
    num_edges: int = 40                  # eval_config.yaml:13
    use_cf: bool = False
    class_label: int = 0                 # TEXT2INT[...] when use_cf
    bbox_threshold: float = 0.08         # eval_config.yaml:10
    guidance_w: float = 0.6              # sample.py:49
    schedule: str = "reference"          # "reference" | "ddpm"
    ddpm_steps: int = 1000               # per stage, schedule == "ddpm"
    dense_masks: bool = False            # True: skip dedup, every slot valid (the dense-FLOP benchmark mode)
    ragged_masks: bool = False           # benchmark only: synthetic masks shaped like a trained model's output (random-init
                                         # weights never produce duplicates): 1/8..1/2 of the faces valid, 3..E/3 edges each
    seed: int = 0
    decode: bool = True
    graph: str = "auto"                  # "on" | "off" | "auto": capture each DDPM loop (advance, forward, fused step) in a CUDA
                                         # graph and replay it; auto = on for launch-bound shapes (few tokens, many steps)


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


def dedup_surfaces(surfPos: torch.Tensor, threshold: float):
    B, S, _ = surfPos.shape
    x = surfPos.float().contiguous()
    out = torch.empty_like(x)
    mask = torch.empty(B, S, dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        _ffi.check(_ffi.lib().bg_dedup_surfaces(x.data_ptr(), B, S, float(threshold), out.data_ptr(), mask.data_ptr(),
                                               _ffi.current_stream()), "bg_dedup_surfaces")
    return out, mask


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

    # ------------------------------------------------------------------ one DDPM loop as a replayed CUDA graph
    def _use_graph(self, cfg: CascadeConfig, n_steps: int, tokens: int) -> bool:
        if cfg.graph == "on":
            return True
        if cfg.graph == "off":
            return False
        # a forward is ~105 launches from Python (~1 ms of host time); below ~100 k tokens the GPU finishes sooner than that
        return n_steps >= 32 and tokens <= 100_000

    def _loop_graph(self, cfg: CascadeConfig, timesteps, x, fwd):
        """timesteps: 1-D int64 CPU tensor; x: (B, ...) fp32 on the device; fwd(x_in, t_dev) -> eps of a (possibly CFG-doubled)
        batch.  The loop body of sample.py:145-153 -- [step counter / timestep advance] -> forward -> fused scheduler step
        (CFG combine, x0, clip, posterior mean, Philox noise) -- is captured ONCE and replayed len(timesteps) times: no
        per-step host work.  Nothing step-specific is a kernel argument: the timestep comes from a device scalar, the
        coefficients from a device table indexed by a device counter (bg_step_advance / bg_ddpm_step_tab)."""
        dev = self.device
        lib = _ffi.lib()
        T = len(timesteps)
        B = x.shape[0]
        xb = x.detach().float().contiguous().clone()
        n = xb.numel()
        coef = self.ddpm.coefficient_table(timesteps).to(dev)
        ts = timesteps.to(device=dev, dtype=torch.int64).contiguous()
        step = torch.full((1,), -1, dtype=torch.int32, device=dev)
        t_cur = torch.zeros(1, dtype=torch.int64, device=dev)
        seed, off0, stride = self.ddpm.philox_stream(n)
        clip = float(self.ddpm.config.clip_sample_range) if self.ddpm.config.clip_sample else 0.0

        def body():
            st = _ffi.current_stream()
            _ffi.check(lib.bg_step_advance(ts.data_ptr(), T, step.data_ptr(), t_cur.data_ptr(), st), "bg_step_advance")
            pred = fwd(torch.cat([xb, xb], 0) if cfg.use_cf else xb, t_cur)
            pc = pred[:B] if cfg.use_cf else pred
            pu = pred[B:] if cfg.use_cf else None
            _ffi.check(lib.bg_ddpm_step_tab(pc.data_ptr(), _ffi.ptr(pu), float(cfg.guidance_w), xb.data_ptr(), xb.data_ptr(),
                                            seed, off0, stride, n, coef.data_ptr(), step.data_ptr(), clip, st),
                       "bg_ddpm_step_tab")

        # warm-up outside the capture (packs the weights, allocates the workspace), then rewind the state it touched
        x0 = xb.clone()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            body()
        torch.cuda.current_stream(dev).wait_stream(side)
        xb.copy_(x0)
        step.fill_(-1)
        g = torch.cuda.CUDAGraph()
        l0 = lib.bg_launch_count()
        with torch.cuda.graph(g):
            body()
        per_replay = lib.bg_launch_count() - l0
        for _ in range(T):
            g.replay()
        _ffi.note_replay(per_replay, T)
        self.ddpm.advance_philox(n, T)
        self.last_graph_steps = getattr(self, "last_graph_steps", 0) + T
        return xb

    # ------------------------------------------------------------------ one denoising loop
    def _loop(self, cfg: CascadeConfig, sched, timesteps, x, fwd, label2, gen, on_step=None, noise_fn=None):
        """fwd(x_in, t_dev) -> eps for a (possibly CFG-doubled) batch; noise_fn(k, shape) -> explicit DDPM step noise"""
        B = x.shape[0]
        k = 0
        is_ddpm = isinstance(sched, DDPMScheduler)
        if is_ddpm and noise_fn is None and gen is None and len(timesteps) > 0 and \
                self._use_graph(cfg, len(timesteps), x[0].numel() // x.shape[-1] * B * (2 if cfg.use_cf else 1)):
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
                x = self._loop_graph(cfg, timesteps[lo:hi], x, fwd)
                lo = hi
            return x
        ts_dev = timesteps.to(self.device)
        for i in range(len(timesteps)):
            t = timesteps[i]
            t_dev = ts_dev[i:i + 1]
            if on_step is not None:
                x = on_step(int(t), x)
                B = x.shape[0]
            if cfg.use_cf:
                pred = fwd(torch.cat([x, x], 0), t_dev)
                if is_ddpm:
                    nz = noise_fn(k, x.shape).to(self.device) if (noise_fn is not None and int(t) > 0) else None
                    x = sched.step(pred[:B], t, x, generator=gen, noise=nz, model_output_uncond=pred[B:],
                                   guidance_w=cfg.guidance_w).prev_sample
                else:
                    eps = torch.empty_like(x)
                    w = cfg.guidance_w
                    _ffi.check(_ffi.lib().bg_axpby(pred[:B].data_ptr(), 1.0 + w, pred[B:].data_ptr(), -w, eps.data_ptr(),
                                                  eps.numel(), _ffi.current_stream()), "bg_axpby")
                    x = sched.step(eps, t, x).prev_sample
            else:
                pred = fwd(x, t_dev)
                if is_ddpm:
                    nz = noise_fn(k, x.shape).to(self.device) if (noise_fn is not None and int(t) > 0) else None
                    x = sched.step(pred, t, x, generator=gen, noise=nz).prev_sample
                else:
                    x = sched.step(pred, t, x).prev_sample
            k += 1
        return x

    _STAGE_ID = {"surfPos": 0, "surfZ": 1, "edgePos": 2, "edgeZV": 3}

    def _stage(self, cfg, x, fwd, label2, gen, hybrid_ddpm_tail: bool, on_step=None, noise_fn=None, name="surfPos"):
        self.ddpm.set_noise_seed(*getattr(self, "_noise_key", (int(cfg.seed), 0)), self._STAGE_ID[name])
        if cfg.schedule == "ddpm":
            self.ddpm.set_timesteps(cfg.ddpm_steps)
            return self._loop(cfg, self.ddpm, self.ddpm.timesteps, x, fwd, label2, gen, on_step, noise_fn)
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

    # ------------------------------------------------------------------ the cascade
    @torch.no_grad()
    def run(self, cfg: CascadeConfig, init_noise: Optional[Dict[str, torch.Tensor]] = None, step_noise=None):
        """step_noise(stage_name, k, shape) -> tensor: explicit DDPM step noise (parity runs); default = in-kernel Philox
        keyed by (cfg.seed, rank, stage): reproducible from cfg.seed, independent across ranks and stages."""
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
        gen = None
        B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
        S = S0 if cfg.use_cf else 2 * S0
        cpu_gen = torch.Generator().manual_seed(cfg.seed)             # initial noise: CPU generator (utils.py:62-97)
        label2 = None
        if cfg.use_cf:
            label2 = torch.tensor([cfg.class_label] * B + [TEXT2INT["uncond"]] * B, device=dev).reshape(-1, 1)

        def noise(name, shape):
            if init_noise is not None and name in init_noise:
                return init_noise[name].to(dev).float()
            return torch.randn(shape, generator=cpu_gen).to(dev)

        rep2 = (lambda t: torch.cat([t, t], 0)) if cfg.use_cf else (lambda t: t)

        # STEP 1-1 surface positions (sample.py:126-153)
        def late_increase(t, x):
            # non-CFG runs double the face slots once the DDPM tail (t < 250) starts (sample.py:140-142).  Pure function of
            # (t, shape): the graph path probes it to find the segment boundaries.
            if not cfg.use_cf and x.shape[1] == S0 and (t < 0 or t <= 249):
                return x.repeat(1, 2, 1)
            return x

        surfPos = noise("surfPos", (B, S0, 6))
        surfPos = self._stage(cfg, surfPos, lambda x, t: self.m["surfpos"](x, t, label2), label2, gen, True,
                              on_step=late_increase, noise_fn=nf("surfPos"), name="surfPos")
        if not cfg.use_cf and surfPos.shape[1] == S0:
            surfPos = surfPos.repeat(1, 2, 1)

        # STEP 1-2 duplicate faces (sample.py:159-183)
        mask_gen = torch.Generator().manual_seed(cfg.seed + 12345)
        if cfg.ragged_masks:
            nv = torch.randint(max(1, S // 8), max(2, S // 2) + 1, (B,), generator=mask_gen)
            surfMask = (torch.arange(S)[None, :] >= nv[:, None]).to(dev)
        elif cfg.dense_masks:
            surfMask = torch.zeros(B, S, dtype=torch.bool, device=dev)
        else:
            surfPos, surfMask = dedup_surfaces(surfPos, cfg.bbox_threshold)
        sP, sM = rep2(surfPos), rep2(surfMask)

        # STEP 1-3 surface latents (sample.py:189-202)
        surfZ = noise("surfZ", (B, S, 48))
        surfZ = self._stage(cfg, surfZ, lambda x, t: self.m["surfz"](x, t, sP, sM, label2), label2, gen, False,
                            noise_fn=nf("surfZ"), name="surfZ")
        sZ = rep2(surfZ)

        # STEP 2-1 edge positions (sample.py:208-236)
        edgePos = noise("edgePos", (B, S, E, 6))
        edgePos = self._stage(cfg, edgePos, lambda x, t: self.m["edgepos"](x, t, sP, sZ, sM, label2), label2, gen, True,
                              noise_fn=nf("edgePos"), name="edgePos")

        # STEP 2-2 duplicate edges per face (sample.py:242-261)
        if cfg.ragged_masks:
            ne = torch.randint(min(3, E), max(min(3, E), E // 3) + 1, (B, S), generator=mask_gen)
            edgeM = (torch.arange(E)[None, None, :] >= ne[..., None]).to(dev) | surfMask[..., None]
        elif cfg.dense_masks:
            edgeM = torch.zeros(B, S, E, dtype=torch.bool, device=dev)
        else:
            edgeM = dedup_edges(edgePos, surfMask, cfg.bbox_threshold)
        eP, eM = rep2(edgePos), rep2(edgeM)

        # STEP 2-3 edge latents + vertices (sample.py:267-286)
        edgeZV = noise("edgeZV", (B, S, E, 18))
        edgeZV = self._stage(cfg, edgeZV, lambda x, t: self.m["edgez"](x, t, eP, sP, sZ, eM, label2), label2, gen, False,
                             noise_fn=nf("edgeZV"), name="edgeZV")
        edgeZV = edgeZV.masked_fill(edgeM.unsqueeze(-1), 0.0)
        edge_z, edgeV = edgeZV[..., :12], edgeZV[..., 12:]

        out = {"surfPos": surfPos / 3.0, "surfMask": surfMask, "surfZ": surfZ, "edgePos": edgePos / 3.0, "edgeM": edgeM,
               "edge_z": edge_z.contiguous(), "edgeV": edgeV.contiguous()}
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
