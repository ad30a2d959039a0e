"""CPU tests of B-rep completion (Cascade.run(known=...)): the Completion checks, the replacement coefficients against the
oracle schedulers, the counter / key / stream plumbing of replace_known (with a recording stand-in for the library) and the
completion oracle (oracle/completion.py) against the unmodified cascade oracles."""
import contextlib

import numpy as np
import pytest
import torch

from brepgen_b200.sampler import Cascade, CascadeConfig, Completion
from brepgen_b200.schedulers import DDIMScheduler, DDPMScheduler, mix_seed
from oracle.completion import run_cascade_completion
from oracle.ddim import DDIMOracle
from oracle.schedulers import DDPMOracle


class _RecordingLib:
    """records every library call instead of launching (host-logic tests run without a device)"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("bg_"):
            raise AttributeError(name)

        def call(*a):
            self.calls.append((name, a))
            return 0
        return call

    def named(self, name):
        return [a for n, a in self.calls if n == name]


@pytest.fixture
def fake_lib(monkeypatch):
    from brepgen_b200 import _ffi, schedulers
    fake = _RecordingLib()
    monkeypatch.setattr(_ffi, "lib", lambda: fake)
    monkeypatch.setattr(_ffi, "current_stream", lambda: 0)
    monkeypatch.setattr(schedulers, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "device", contextlib.nullcontext)
    return fake


def _known(B=2, K=3, E=4, n=(2, 3), z=True, edges=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    kw = dict(n_faces=list(n), surfPos=torch.rand(B, K, 6, generator=g) * 2 - 1)
    if z:
        kw["surfZ"] = torch.randn(B, K, 48, generator=g)
    if edges:
        kw.update(edgePos=torch.rand(B, K, E, 6, generator=g), edge_z=torch.randn(B, K, E, 12, generator=g),
                  edgeV=torch.randn(B, K, E, 6, generator=g),
                  edge_mask=torch.arange(E)[None, None, :].expand(B, K, E) >= 2)
    return Completion(**kw)


def _cfg(**kw):
    base = dict(batch_size=2, num_surfaces=5, num_edges=4, schedule="ddim", ddim_steps=4, decode=False, graph="off")
    base.update(kw)
    return CascadeConfig(**base)


# -------------------------------------------------------------------------------------------------------- validation
def _bad_cases():
    k = _known()
    return [
        ("schedule reference", dict(schedule="reference"), k, NotImplementedError),
        ("dense masks", dict(dense_masks=True), k, ValueError),
        ("ragged masks", dict(ragged_masks=True), k, ValueError),
        ("n_faces length", {}, _known(n=(1,)), ValueError),
        ("n_faces > K", {}, _known(n=(2, 4)), ValueError),
        ("n_faces < 0", {}, _known(n=(-1, 2)), ValueError),
        ("K > num_surfaces", dict(num_surfaces=2), k, ValueError),
        ("batch size", dict(batch_size=3), k, ValueError),
        ("surfPos last dim", {}, Completion(n_faces=[1, 1], surfPos=torch.zeros(2, 3, 5)), ValueError),
        ("surfPos rank", {}, Completion(n_faces=[1, 1], surfPos=torch.zeros(2, 6)), ValueError),
        ("surfZ shape", {}, Completion(n_faces=[1, 1], surfPos=torch.zeros(2, 3, 6), surfZ=torch.zeros(2, 2, 48)),
         ValueError),
        ("num_edges", dict(num_edges=5), k, ValueError),
        ("edge_z shape", {}, Completion(**dict(vars(k), edge_z=torch.zeros(2, 3, 4, 11))), ValueError),
        ("edge_mask dtype", {}, Completion(**dict(vars(k), edge_mask=k.edge_mask.float())), ValueError),
        ("edges without surfZ", {}, Completion(**dict(vars(k), surfZ=None)), ValueError),
        ("edge fields partial", {}, Completion(**dict(vars(k), edgeV=None)), ValueError),
        ("edge slot 0 padded on a known face", {},
         Completion(**dict(vars(k), edge_mask=k.edge_mask.clone().index_put_((torch.tensor([1]), torch.tensor([2]),
                                                                             torch.tensor([0])), torch.tensor(True)))),
         ValueError),
    ]


@pytest.mark.parametrize("name,cfg_kw,known,exc", _bad_cases(), ids=[c[0] for c in _bad_cases()])
def test_bad_completions_raise_before_any_launch(fake_lib, name, cfg_kw, known, exc):
    with pytest.raises(exc):
        Cascade({}, device="cpu").run(_cfg(**cfg_kw), known=known)
    assert fake_lib.calls == []


def test_edge_slot_0_padded_past_n_faces_is_allowed():
    from brepgen_b200.sampler import check_completion
    k = _known(n=(1, 3))
    k.edge_mask[0, 2, 0] = True          # face 2 of sample 0 is not known
    assert check_completion(_cfg(), k).tolist() == [1, 3]


def test_duplicate_known_faces_raise_through_the_dedup_kernel(fake_lib, monkeypatch):
    """the duplicate check is bg_dedup_surfaces on the model-unit boxes (here a stand-in running the oracle's rule), the
    only library call made before the error; face rows past n_faces never count"""
    from brepgen_b200 import sampler
    from oracle.cascade import dedup_surfaces_np
    seen = []

    def dedup(x, thr):
        seen.append(x.clone())
        p, m = dedup_surfaces_np(x.numpy(), np.float32(thr))
        return torch.from_numpy(p), torch.from_numpy(m)
    monkeypatch.setattr(sampler, "dedup_surfaces", dedup)
    k = _known(n=(2, 3), edges=False)
    k.surfPos[1, 2] = k.surfPos[1, 0] + 0.001                          # within bbox_threshold / 3 of face 0
    with pytest.raises(ValueError, match=r"samples \[1\]"):
        Cascade({}, device="cpu").run(_cfg(), known=k)
    assert fake_lib.calls == [] and len(seen) == 1
    assert torch.equal(seen[0][1], k.surfPos[1] * 3.0)
    assert torch.equal(seen[0][0, 2], seen[0][0, 0])                  # sample 0, row past n_faces = 2: copy of face 0
    # the same duplicate past n_faces is no error: the check passes and the run goes on to the denoisers
    k.n_faces = [2, 2]
    with pytest.raises(KeyError):
        Cascade({}, device="cpu").run(_cfg(), known=k)


def test_from_outputs_cuts_the_first_faces():
    B, S, E = 3, 6, 4
    g = torch.Generator().manual_seed(1)
    out = {"surfPos": torch.randn(B, S, 6, generator=g), "surfMask": torch.arange(S)[None, :] >= torch.tensor([[4], [6], [2]]),
           "surfZ": torch.randn(B, S, 48, generator=g), "edgePos": torch.randn(B, S, E, 6, generator=g),
           "edgeM": torch.rand(B, S, E, generator=g) > 0.5, "edge_z": torch.randn(B, S, E, 12, generator=g),
           "edgeV": torch.randn(B, S, E, 6, generator=g)}
    c = Completion.from_outputs(out, [1, 3, 0])
    assert c.n_faces == [1, 3, 0] and c.surfPos.shape == (B, 3, 6) and c.edge_mask.shape == (B, 3, E)
    for f, k in (("surfPos", "surfPos"), ("surfZ", "surfZ"), ("edgePos", "edgePos"), ("edge_z", "edge_z"),
                 ("edgeV", "edgeV"), ("edge_mask", "edgeM")):
        assert torch.equal(getattr(c, f), out[k][:, :3])
    c = Completion.from_outputs(out, [1, 3, 0], edges=False)
    assert c.edgePos is None and c.edge_mask is None and c.surfZ is not None
    with pytest.raises(ValueError):
        Completion.from_outputs(out, [5, 1, 1])      # sample 0 has 4 valid faces
    with pytest.raises(ValueError):
        Completion.from_outputs(out, [1, 1])


# ---------------------------------------------------------------------------------------------- replacement tables
@pytest.mark.parametrize("kind", ["ddpm", "ddim"])
@pytest.mark.parametrize("n_steps", [1, 4, 10, 50, 1000])
def test_replace_table_matches_oracle(kind, n_steps):
    if kind == "ddpm":
        s, o = DDPMScheduler(clip_sample_range=3), DDPMOracle()
        final = torch.tensor(1.0)
    else:
        s, o = DDIMScheduler(clip_sample_range=3, set_alpha_to_one=True), DDIMOracle(set_alpha_to_one=True)
        final = o.final_acp
    s.set_timesteps(n_steps), o.set_timesteps(n_steps)
    tab = s.replace_table(s.timesteps)
    assert tab.shape == (n_steps, 2) and tab.dtype == torch.float32
    for i, t in enumerate(o.timesteps.tolist()):
        prev_t = t - o.n_train // o.n_inf
        a = o.acp[prev_t] if prev_t >= 0 else final
        assert tab[i].tolist() == [float(a ** 0.5), float((1 - a) ** 0.5)], (i, t)
        a_t = o.acp[t]
        assert list(s.replace_coefficients(t, initial=True)) == [float(a_t ** 0.5), float((1 - a_t) ** 0.5)]
    assert tab[-1].tolist() == [1.0, 0.0]
    assert s.replace_coefficients(int(s.timesteps[-1])) == (1.0, 0.0)


# -------------------------------------------------------------------------------------------- counters and streams
# positions in the bg_replace_known argument list
R_X, R_KNOWN, R_MASK, R_N, R_PER_TOKEN, R_NOISE, R_SEED, R_KEYS, R_PER_SAMPLE, R_T, R_SA, R_SB = range(12)


def test_replace_known_arguments(fake_lib):
    s = DDPMScheduler(clip_sample_range=3)
    s.set_timesteps(4)
    x, kn = torch.zeros(3, 5, 6), torch.ones(3, 5, 6)
    m = torch.zeros(3, 5, dtype=torch.bool)
    s.set_noise_seed(7, 0, 2)
    y = s.replace_known(x, kn, m, 500)
    a = fake_lib.named("bg_replace_known")[0]
    assert y is not x and y.data_ptr() == a[R_X]
    assert (a[R_N], a[R_PER_TOKEN], a[R_PER_SAMPLE], a[R_T]) == (90, 6, 30, 500)
    assert a[R_SEED] == mix_seed(mix_seed(7, 0, 2), 2) and a[R_KEYS] is None and a[R_NOISE] is None
    assert (a[R_SA], a[R_SB]) == s.replace_coefficients(500) == tuple(float(v) for v in (
        s.alphas_cumprod[250] ** 0.5, (1 - s.alphas_cumprod[250]) ** 0.5))
    s.replace_known(x, kn, m, 750, initial=True, out=x)
    a = fake_lib.named("bg_replace_known")[1]
    assert a[R_X] == x.data_ptr() and a[R_T] == 751
    assert (a[R_SA], a[R_SB]) == tuple(float(v) for v in (s.alphas_cumprod[750] ** 0.5, (1 - s.alphas_cumprod[750]) ** 0.5))
    s.replace_known(x, kn, m, 500, noise=torch.zeros(3, 5, 6))
    assert fake_lib.named("bg_replace_known")[2][R_NOISE] is not None
    s.set_sample_keys(seed=3, first=4, stage=1)
    s.replace_known(x, kn, m, 250)
    a = fake_lib.named("bg_replace_known")[3]
    assert a[R_KEYS] == s.sample_key_tensor(3, x.device).data_ptr() and a[R_SEED] == 0
    for bad in (dict(known=torch.ones(3, 5, 7)), dict(known_mask=torch.zeros(3, 6, dtype=torch.bool)),
                dict(noise=torch.zeros(3, 5))):
        args = dict(sample=x, known=kn, known_mask=m, timestep=500)
        args.update(bad)
        with pytest.raises(RuntimeError):
            s.replace_known(**args)
    assert len(fake_lib.named("bg_replace_known")) == 4


def _stage_calls(fake_lib, kind, noise, known, use_cf=False, S0=3):
    """runs Cascade._stage('surfPos') with stand-in networks; returns (step calls, replace calls, scheduler)"""
    fake_lib.calls.clear()
    cfg = _cfg(schedule=kind, ddpm_steps=5, ddim_steps=5, ddim_eta=0.7, noise=noise, num_surfaces=S0, use_cf=use_cf)
    c = Cascade({}, device="cpu")
    c._sample_seeds = [11, 12] if noise == "per_sample" else None
    c._noise_key = (4, 0)
    B = 2
    kn = None
    if known:
        face = torch.zeros(B, S0, dtype=torch.uint8)
        face[0, 0] = 1
        kn = {S0: (torch.ones(B, S0, 6), face), 2 * S0: (torch.ones(B, 2 * S0, 6), face.repeat(1, 2))}

    def late(t, x):
        return x.repeat(1, 2, 1) if (not use_cf and x.shape[1] == S0 and t <= 249) else x
    c._stage(cfg, torch.zeros(B, S0, 6), lambda x, t: torch.zeros_like(x), None, None, True, on_step=late, known=kn)
    step = "bg_ddim_step" if kind == "ddim" else "bg_ddpm_step"
    sched = c.ddim if kind == "ddim" else c.ddpm
    return fake_lib.named(step), fake_lib.named("bg_replace_known"), sched


@pytest.mark.parametrize("kind", ["ddpm", "ddim"])
@pytest.mark.parametrize("noise", ["batch", "per_sample"])
def test_stage_counters_keys_and_untouched_step_stream(fake_lib, kind, noise):
    steps0, rep0, s0 = _stage_calls(fake_lib, kind, noise, known=False)
    off0 = s0._philox_offset
    steps1, rep1, s1 = _stage_calls(fake_lib, kind, noise, known=True)
    assert rep0 == []
    # the step calls, their noise offsets and the scheduler's stream position are those of the run without completion
    ptrs = (0, 1, 3, 4, 8)      # eps, eps_uncond, x, out and sample_keys (per-run tensors)
    strip = lambda calls: [tuple(v for i, v in enumerate(a) if i not in ptrs) for a in calls]
    assert strip(steps1) == strip(steps0) and s1._philox_offset == off0
    ts = s1.timesteps.tolist()
    assert [a[R_T] for a in rep1] == [ts[0] + 1] + ts              # t_first + 1 before the loop, then t of each step
    assert [a[R_N] for a in rep1] == [2 * 3 * 6] + [2 * (3 if t > 249 else 6) * 6 for t in ts]   # late increase
    assert [(a[R_SA], a[R_SB]) for a in rep1[1:]] == [tuple(r) for r in s1.replace_table(ts).tolist()]
    assert (rep1[-1][R_SA], rep1[-1][R_SB]) == (1.0, 0.0)
    if noise == "per_sample":
        keys = s1.sample_key_tensor(2, "cpu").data_ptr()
        assert all(a[R_KEYS] == keys and a[R_SEED] == 0 and a[R_PER_SAMPLE] == a[R_N] // 2 for a in rep1)
        if kind == "ddim":
            assert all(a[8] == keys for a in steps1)                  # bg_ddim_step's sample_keys
        else:
            # bg_ddpm_step's sample_keys on every step that draws (sigma != 0), none on the last step (t = 0, sigma = 0)
            assert [a[8] for a in steps1] == [keys] * (len(steps1) - 1) + [None]
            assert [a[17] != 0.0 for a in steps1] == [True] * (len(steps1) - 1) + [False]
    else:
        assert all(a[R_KEYS] is None and a[R_SEED] == mix_seed(mix_seed(4, 0, 0), 2) for a in rep1)


# ------------------------------------------------------------------------------------------------------------- oracle
def _stand_ins():
    def fwd(kind):
        def f(x, t, *rest):
            return torch.tanh(x * 0.7 + 0.01 * int(t) / 1000) * 0.5
        return f
    return {k: fwd(k) for k in ("surfpos", "surfz", "edgepos", "edgez")}


def _init(cfg, seed=1):
    g = torch.Generator().manual_seed(seed)
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    S = S0 if cfg.use_cf else 2 * S0
    return {"surfPos": torch.randn(B, S0, 6, generator=g), "surfZ": torch.randn(B, S, 48, generator=g),
            "edgePos": torch.randn(B, S, E, 6, generator=g), "edgeZV": torch.randn(B, S, E, 18, generator=g)}


def _bank(seed):
    g = torch.Generator().manual_seed(seed)
    bank = {}

    def noise(name, k, shape):
        if (name, k, tuple(shape)) not in bank:
            bank[(name, k, tuple(shape))] = torch.randn(tuple(shape), generator=g)
        return bank[(name, k, tuple(shape))]
    return noise, bank


@pytest.mark.parametrize("schedule,use_cf", [("ddpm", False), ("ddpm", True), ("ddim", False), ("ddim", True)])
def test_completion_oracle_without_known_is_the_cascade_oracle(schedule, use_cf):
    from oracle.cascade import run_cascade
    from oracle.ddim import run_cascade_ddim
    cfg = _cfg(schedule=schedule, ddpm_steps=6, ddim_steps=6, ddim_eta=0.5, use_cf=use_cf, class_label=3, batch_size=3)
    init = _init(cfg)
    n1, _ = _bank(5)
    n2, _ = _bank(5)
    ref = (run_cascade if schedule == "ddpm" else run_cascade_ddim)(None, cfg, init, n1, _stand_ins())
    got = run_cascade_completion(None, cfg, init, n2, known=None, forwards=_stand_ins())
    assert set(got) == set(ref)
    for k in ref:
        assert torch.equal(got[k], ref[k]), k


@pytest.mark.parametrize("schedule,use_cf", [("ddpm", False), ("ddim", True)])
@pytest.mark.parametrize("edges", [True, False])
def test_completion_oracle_returns_known_parts(schedule, use_cf, edges):
    cfg = _cfg(schedule=schedule, ddpm_steps=6, ddim_steps=6, ddim_eta=0.5, use_cf=use_cf, class_label=3, batch_size=3)
    sn, _ = _bank(5)
    a = run_cascade_completion(None, cfg, _init(cfg), sn, forwards=_stand_ins())
    nv = (~a["surfMask"]).sum(1)
    n = [0, min(2, int(nv[1])), int(nv[2])]
    known = Completion.from_outputs(a, n, edges=edges)
    rn, bank = _bank(8)
    b = run_cascade_completion(None, cfg, _init(cfg, seed=2), sn, known=known, replace_noise=rn, forwards=_stand_ins())
    assert {k for k, _, _ in bank} == ({"surfPos", "surfZ", "edgePos", "edgeZV"} if edges else {"surfPos", "surfZ"})
    assert min(k for _, k, _ in bank) == -1
    for i in range(3):
        f = slice(0, n[i])
        assert not b["surfMask"][i, f].any()
        fields = [("surfPos", "surfPos"), ("surfZ", "surfZ")]
        if edges:
            fields += [("edgePos", "edgePos"), ("edge_z", "edge_z"), ("edgeV", "edgeV"), ("edge_mask", "edgeM")]
        for fk, ok in fields:
            assert torch.equal(b[ok][i, f], getattr(known, fk)[i, f]), (i, fk)
    assert not torch.equal(b["surfPos"][0], a["surfPos"][0])          # the rest is generated anew
