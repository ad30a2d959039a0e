"""ORACLE (test infrastructure): DDIM inversion, per-sample slerp and the cascade driver of inverted variations and
interpolations.

DDIMInverseOracle restates diffusers 0.27 DDIMInverseScheduler (epsilon prediction, "leading" spacing) in fp32 torch:
step(eps, t, x) moves x from level t - ratio up to level t,
    x0 = clamp((x - sqrt(1 - abar_cur) eps) / sqrt(abar_cur), +-clip),   x_next = sqrt(abar_t) x0 + sqrt(1 - abar_t) eps,
cur = min(t - ratio, 999), abar below the first timestep 1 (set_alpha_to_one) or alphas_cumprod[0].  diffusers is not
installed here, so it is pinned by equivalence to the already-pinned DDIMOracle (tests/test_inversion.py): the forward
step at t undoes the inverse step at t.

run_cascade_inverted_variation / run_cascade_interpolation restate oracle/variation.py's DDIM driver with a different
start for every varied stage: the source gathered through the variation's layout (fill_rows, the survivors of
dedup_surfaces_survivors; -1 slots take z), inverted along the reversed tail with the conditioning gathered from the
source through the same maps (0 where a map is -1; mask = map < 0), and, for an interpolation, the two inverted starts
slerped in fp64 with the stage's token mask.  Each source is inverted as a batch of its own.
"""
from __future__ import annotations

import numpy as np
import torch

from . import denoisers as O
from .cascade import dedup_edges_np
from .ddim import DDIMOracle
from .schedulers import linear_alphas_cumprod
from .variation import STAGES, dedup_surfaces_survivors, fill_rows, strengths


class DDIMInverseOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, clip_sample=True, clip_sample_range=1.0,
                 set_alpha_to_one=True, steps_offset=0):
        self.n_train = num_train_timesteps
        self.acp = linear_alphas_cumprod(num_train_timesteps, beta_start, beta_end)
        self.initial_acp = torch.tensor(1.0) if set_alpha_to_one else self.acp[0]
        self.clip_sample, self.clip_range = clip_sample, float(clip_sample_range)
        self.steps_offset = steps_offset
        self.set_timesteps(num_train_timesteps)

    def set_timesteps(self, n: int):
        self.n_inf = n
        ratio = self.n_train // n
        self.timesteps = torch.from_numpy((np.arange(0, n) * ratio).round().astype(np.int64) + self.steps_offset)

    def coeffs(self, t: int):
        """(sqrt(1-abar_cur), sqrt(abar_cur), sqrt(abar_t), sqrt(1-abar_t)) as fp32 torch scalars"""
        cur = min(t - self.n_train // self.n_inf, self.n_train - 1)
        a_cur = self.acp[cur] if cur >= 0 else self.initial_acp
        a_t = self.acp[t]
        return (1 - a_cur) ** 0.5, a_cur ** 0.5, a_t ** 0.5, (1 - a_t) ** 0.5

    def step(self, eps, t, x):
        sb, sa, sa_next, c_dir = self.coeffs(int(t))
        x0 = (x - sb * eps) / sa
        if self.clip_sample:
            x0 = x0.clamp(-self.clip_range, self.clip_range)
        return sa_next * x0 + c_dir * eps


def slerp(a, b, alpha, token_mask=None, dot_threshold=0.9995):
    """fp64 per-sample slerp of a, b (B, ..., D): a.b and the norms over the tokens (last dimension) whose token_mask
    (B, ...) entry is False; the lerp when |cos| > dot_threshold or a norm is zero; alpha 0 -> a, 1 -> b; masked tokens
    copied from a.  Returns fp64."""
    a, b = a.double(), b.double()
    out = a.clone()
    B = a.shape[0]
    keep = torch.ones(a.shape[:-1], dtype=torch.bool) if token_mask is None else ~token_mask.bool().cpu()
    for i in range(B):
        al = float(alpha[i])
        va, vb = a[i][keep[i]], b[i][keep[i]]
        if al == 0.0:
            continue
        if al == 1.0:
            out[i][keep[i]] = vb
            continue
        nn = float((va * va).sum() * (vb * vb).sum()) ** 0.5
        c = min(max(float((va * vb).sum()) / nn, -1.0), 1.0) if nn > 0 else 1.0
        if abs(c) > dot_threshold:
            v = (1 - al) * va + al * vb
        else:
            th = np.arccos(c)
            v = np.sin((1 - al) * th) / np.sin(th) * va + np.sin(al * th) / np.sin(th) * vb
        out[i][keep[i]] = v
    return out


def _run(sds, cfg, sources, alpha, init_noise, forwards=None):
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    S = S0 if cfg.use_cf else 2 * S0
    w = cfg.guidance_w
    st = strengths(sources[0])
    label2 = None
    if cfg.use_cf:
        label2 = torch.tensor([cfg.class_label] * B + [0] * B).reshape(-1, 1)
    rep2 = (lambda t: torch.cat([t, t], 0)) if cfg.use_cf else (lambda t: t)
    sched = DDIMOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True)
    sched.set_timesteps(cfg.ddim_steps)
    inv = DDIMInverseOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True)
    inv.set_timesteps(cfg.ddim_steps)
    full = sched.timesteps
    N = len(full)
    tails = {name: full[N - min(int(N * s), N):] for name, s in zip(STAGES, st)}

    def predict(fwd, x, t):
        tt = torch.tensor([int(t)])
        if cfg.use_cf:
            p = fwd(torch.cat([x, x], 0), tt)
            return p[:B] * (1 + w) - p[B:] * w
        return fwd(x, tt)

    def stage(name, x, fwd, late=None):
        for t in tails[name]:
            if late is not None:
                x = late(int(t), x)
            x = sched.step(predict(fwd, x, t), int(t), x)
        return x

    if forwards is None:
        forwards = {"surfpos": lambda *a: O.surfpos_forward(sds["surfpos"], *a),
                    "surfz": lambda *a: O.surfz_forward(sds["surfz"], *a),
                    "edgepos": lambda *a: O.edgepos_forward(sds["edgepos"], *a),
                    "edgez": lambda *a: O.edgez_forward(sds["edgez"], *a)}
    F = forwards
    srcs = []
    for v in sources:
        s = {k: getattr(v, k).detach().cpu() for k in ("surfPos", "surfMask", "surfZ", "edgePos", "edgeM", "edge_z",
                                                        "edgeV")}
        s = {k: t if t.dtype == torch.bool else t.float() for k, t in s.items()}
        s["edgeZV"] = torch.cat([s["edge_z"], s["edgeV"]], -1)
        srcs.append(s)
    thr = np.float32(cfg.bbox_threshold)

    def take(s, field, index, scale, shape):
        """scale * s[field] gathered through the flat token indices `index`, 0 where -1"""
        tok = s[field].reshape(-1, s[field].shape[-1])
        return torch.stack([scale * tok[i] if i >= 0 else torch.zeros(tok.shape[-1]) for i in index]).reshape(shape)

    def holes(index, shape):
        return torch.tensor([i < 0 for i in index]).reshape(shape)

    def start(name, field, maps, scale, shape, model, cond):
        """maps: per source, flat source-token indices; cond(k): the conditioning of source k"""
        z = init_noise[name]
        assert tuple(z.shape) == tuple(shape), (name, tuple(z.shape), shape)
        xs = []
        for k, s in enumerate(srcs):
            has = ~holes(maps[k], shape[:-1])[..., None]
            x = torch.where(has, take(s, field, maps[k], scale, shape), z)
            c = cond(k)
            for t in reversed(tails[name]):
                x = inv.step(predict(lambda x, t: F[model](x, t, *[rep2(v) for v in c], label2), x, t), int(t), x)
            xs.append(x)
        if len(xs) == 1:
            return xs[0]
        return slerp(xs[0], xs[1], alpha, holes(maps[0], shape[:-1])).float()

    with torch.no_grad():
        if st[0] == 0:
            surfPos, surfMask = srcs[0]["surfPos"] * 3.0, srcs[0]["surfMask"]
            rows = [[b * S + f if not bool(surfMask[b, f]) else -1 for b in range(B) for f in range(S)]]
        else:
            S1 = S0 if (not cfg.use_cf and int(tails["surfPos"][0]) > 249) else S
            fill = [fill_rows(s["surfMask"].numpy(), S1) for s in srcs]
            x = start("surfPos", "surfPos", [[i for r in f for i in r] for f in fill], 3.0, (B, S1, 6), "surfpos",
                      lambda k: ())
            state = {"late": S1 == S}

            def late_increase(t, x):          # sample.py:140-142: double the face slots at the first t <= 249
                if not state["late"] and t <= 249:
                    state["late"] = True
                    return x.repeat(1, 2, 1)
                return x
            surfPos = stage("surfPos", x, lambda x, t: F["surfpos"](x, t, label2), late_increase)
            if not state["late"]:
                surfPos = surfPos.repeat(1, 2, 1)
            p, m, kept = dedup_surfaces_survivors(surfPos.numpy(), thr)
            surfPos, surfMask = torch.from_numpy(p), torch.from_numpy(m)
            rows = [[f[b][kept[b][k] % S1] if k < len(kept[b]) else -1 for b in range(B) for k in range(S)]
                    for f in fill]
        sP, sM = rep2(surfPos), rep2(surfMask)
        cP = lambda k: take(srcs[k], "surfPos", rows[k], 3.0, (B, S, 6))
        cZ = lambda k: take(srcs[k], "surfZ", rows[k], 1.0, (B, S, 48))
        cM = lambda k: holes(rows[k], (B, S))

        if st[1] == 0:
            surfZ = srcs[0]["surfZ"]
        else:
            x = start("surfZ", "surfZ", rows, 1.0, (B, S, 48), "surfz", lambda k: (cP(k), cM(k)))
            surfZ = stage("surfZ", x, lambda x, t: F["surfz"](x, t, sP, sM, label2))
        sZ = rep2(surfZ)

        if st[2] == 0:
            edgePos, edgeM = srcs[0]["edgePos"] * 3.0, srcs[0]["edgeM"]
            edges = [list(range(B * S * E))]
        else:
            edges = [[i for r in fill_rows(s["edgeM"].reshape(-1, E).numpy(), E, rows[k]) for i in r]
                     for k, s in enumerate(srcs)]
            x = start("edgePos", "edgePos", edges, 3.0, (B, S, E, 6), "edgepos", lambda k: (cP(k), cZ(k), cM(k)))
            edgePos = stage("edgePos", x, lambda x, t: F["edgepos"](x, t, sP, sZ, sM, label2))
            edgeM = torch.from_numpy(dedup_edges_np(edgePos.numpy(), surfMask.numpy(), thr))
        eP, eM = rep2(edgePos), rep2(edgeM)

        if st[3] == 0:
            edge_z, edgeV = srcs[0]["edge_z"], srcs[0]["edgeV"]
        else:
            x = start("edgeZV", "edgeZV", edges, 1.0, (B, S, E, 18), "edgez",
                      lambda k: (take(srcs[k], "edgePos", edges[k], 3.0, (B, S, E, 6)), cP(k), cZ(k),
                                 holes(edges[k], (B, S, E))))
            edgeZV = stage("edgeZV", x, lambda x, t: F["edgez"](x, t, eP, sP, sZ, eM, label2))
            edgeZV = edgeZV.masked_fill(edgeM.unsqueeze(-1), 0.0)
            edge_z, edgeV = edgeZV[..., :12], edgeZV[..., 12:]
    out = {"surfPos": surfPos / 3.0, "surfMask": surfMask, "surfZ": surfZ, "edgePos": edgePos / 3.0, "edgeM": edgeM,
           "edge_z": edge_z, "edgeV": edgeV}
    if st[0] == 0:
        out["surfPos"] = srcs[0]["surfPos"]
    if st[2] == 0:
        out["edgePos"] = srcs[0]["edgePos"]
    return out


def run_cascade_inverted_variation(sds, cfg, source, init_noise, forwards=None):
    """Variation(start="invert") of `source` (brepgen_b200.sampler.Variation-like) under schedule "ddim", ddim_eta 0.
    init_noise: name -> z of each varied stage in its starting shape (it fills the slots without a source).  Returns the
    tensors oracle.cascade.run_cascade returns (no decode)."""
    return _run(sds, cfg, [source], None, init_noise, forwards)


def run_cascade_interpolation(sds, cfg, a, b, alpha, init_noise, forwards=None):
    """Interpolation(a, b, alpha) under schedule "ddim", ddim_eta 0 (a, b: Variation-like with equal strengths, all > 0);
    both sources' -1 slots take the same z.  Returns the tensors oracle.cascade.run_cascade returns (no decode)."""
    return _run(sds, cfg, [a, b], alpha, init_noise, forwards)
