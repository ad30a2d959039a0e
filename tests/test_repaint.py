"""RePaint resampling without a GPU: the timestep lists of the drop-in and the oracle, the oracle's step and undo against
pinned parts (DDIMOracle, the noising moments), the oracle cascade against run_cascade_ddim, the drop-in's host logic
(entry counters, noise keys, masks) with the library replaced by a recorder, and config validation."""
import contextlib

import numpy as np
import pytest
import torch

# N = 10, jump_length 2, jump_n_sample 3, written out from diffusers' set_timesteps statements (x 100)
LIST_10_2_3 = [9, 8, 7, 6, 7, 8, 7, 6, 7, 8, 7, 6, 5, 4, 5, 6, 5, 4, 5, 6, 5, 4, 3, 2, 3, 4, 3, 2, 3, 4, 3, 2, 1, 0, 1, 2,
               1, 0, 1, 2, 1, 0]


def test_timestep_lists():
    from brepgen_b200.schedulers import DDIMScheduler, RePaintScheduler, repaint_entries
    from oracle.repaint import RePaintOracle
    s, o = RePaintScheduler(), RePaintOracle()
    s.set_timesteps(10, 2, 3)
    o.set_timesteps(10, 2, 3)
    assert s.timesteps.tolist() == o.timesteps.tolist() == [100 * t for t in LIST_10_2_3]
    assert s.timesteps.dtype == torch.int64 and s.undo_transitions == 100
    ents = repaint_entries(s.timesteps)
    assert ents[:6] == [(True, 900), (True, 800), (True, 700), (True, 600), (False, 600), (False, 700)]
    assert ents[6] == (True, 700)
    # sizes of the table in the docs (computed)
    for (N, jl, jn), (entries, steps) in {(50, 5, 5): (410, 230), (250, 10, 10): (4570, 2410)}.items():
        s.set_timesteps(N, jl, jn)
        o.set_timesteps(N, jl, jn)
        assert torch.equal(s.timesteps, o.timesteps)
        kinds = [k for k, _ in repaint_entries(s.timesteps)]
        assert (len(kinds), kinds.count(True), kinds.count(False)) == (entries, steps, entries - steps)
    # jump_n_sample = 1: no resampling, DDIM's "leading" list
    d = DDIMScheduler()
    for N in (1, 4, 10, 50, 250, 1000):
        s.set_timesteps(N, 10, 1)
        d.set_timesteps(N)
        assert torch.equal(s.timesteps, d.timesteps), N
        assert all(k for k, _ in repaint_entries(s.timesteps))
    # jump_length >= N: nothing to jump over
    s.set_timesteps(5, 5, 4)
    assert s.timesteps.tolist() == [800, 600, 400, 200, 0]


@pytest.mark.parametrize("eta", [0.0, 0.7])
def test_oracle_step_with_nothing_known_is_ddim(eta):
    from oracle.ddim import DDIMOracle
    from oracle.repaint import RePaintOracle
    r = RePaintOracle(eta=eta, clip_sample_range=3.0)
    d = DDIMOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True)
    r.set_timesteps(20, 3, 4)
    d.set_timesteps(20)
    g = torch.Generator().manual_seed(2)
    x, eps, known, z = (torch.randn(4, 9, 6, generator=g) * 2 for _ in range(4))
    zero = torch.zeros(4, 9, 1)
    for t in (950, 500, 50, 0):
        want = d.step(eps, t, x, eta, noise=z if eta > 0 else None)
        assert torch.equal(r.step(eps, t, x, known, zero, z), want), t
        assert torch.equal(r.step(eps, t, x, None, None, z), want), t


def test_oracle_step_with_everything_known():
    from oracle.repaint import RePaintOracle
    r = RePaintOracle(eta=1.0, clip_sample_range=3.0)
    r.set_timesteps(20, 3, 4)
    g = torch.Generator().manual_seed(3)
    x, eps, known, z = (torch.randn(4, 9, 6, generator=g) for _ in range(4))
    one = torch.ones(4, 9, 1)
    for t in (950, 500, 50):
        a_prev = r.acp[t - 50]
        assert torch.equal(r.step(eps, t, x, known, one, z), a_prev ** 0.5 * known + (1 - a_prev) ** 0.5 * z), t
    assert torch.equal(r.step(eps, 0, x, known, one, z), known)
    # a token mask selects per token
    m = (torch.rand(4, 9, 1, generator=g) < 0.5).float()
    out = r.step(eps, 500, x, known, m, z)
    sel = m.bool().expand_as(x)
    assert torch.equal(out[sel], r.step(eps, 500, x, known, one, z)[sel])
    assert torch.equal(out[~sel], r.step(eps, 500, x, None, None, z)[~sel])


@pytest.mark.parametrize("t_last", [0, 300, 960])
def test_undo_moments(t_last):
    """n composed transitions of x: mean sqrt(P) x and variance 1 - P with P = prod(1 - beta_{t_last+i}) =
    abar_{t_last+n-1} / abar_{t_last-1}, over 2^20 seeded elements, within 5 sigma"""
    from oracle.repaint import RePaintOracle
    r = RePaintOracle()
    r.set_timesteps(50)                                  # n = 20 transitions per undo
    n = 20
    N = 1 << 20
    g = torch.Generator().manual_seed(t_last)
    x = torch.randn(N, generator=g) * 1.5
    out = r.undo_step(x, t_last, torch.randn(n, N, generator=g))
    P = float(torch.prod((1 - r.betas[t_last:t_last + n]).double()))
    a_hi = float(r.acp[t_last + n - 1])
    a_lo = float(r.acp[t_last - 1]) if t_last > 0 else 1.0
    assert P == pytest.approx(a_hi / a_lo, rel=1e-5)
    res = out.double() - P ** 0.5 * x.double()
    var = 1 - P
    assert abs(float(res.mean())) <= 5 * (var / N) ** 0.5
    assert abs(float(res.var()) - var) <= 5 * var * (2 / N) ** 0.5


def _standins(seen):
    def fwd(kind):
        def f(x, t, *rest):
            seen.setdefault(kind, []).append((int(t), tuple(x.shape)))
            return torch.tanh(x) * 0.5
        return f
    return {k: fwd(k) for k in ("surfpos", "surfz", "edgepos", "edgez")}


@pytest.mark.parametrize("use_cf", [False, True])
def test_oracle_cascade_without_resampling_is_ddim(use_cf):
    from brepgen_b200.sampler import CascadeConfig
    from oracle.ddim import run_cascade_ddim
    from oracle.repaint import run_cascade_repaint
    cfg = CascadeConfig(batch_size=2, num_surfaces=3, num_edges=2, use_cf=use_cf, class_label=6, schedule="repaint",
                        repaint_steps=10, repaint_jump_n_sample=1, repaint_eta=0.0, ddim_steps=10, ddim_eta=0.0)
    S = 3 if use_cf else 6
    g = torch.Generator().manual_seed(1)
    init = {"surfPos": torch.randn(2, 3, 6, generator=g), "surfZ": torch.randn(2, S, 48, generator=g),
            "edgePos": torch.randn(2, S, 2, 6, generator=g), "edgeZV": torch.randn(2, S, 2, 18, generator=g)}
    noise = lambda name, k, shape: torch.randn(tuple(shape), generator=g)
    a = run_cascade_repaint(None, cfg, init, noise, noise, forwards=_standins({}))
    b = run_cascade_ddim(None, cfg, init, noise, forwards=_standins({}))
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_oracle_cascade_driver_counts():
    """one forward per step entry and stage, undo noise of shape (n, *x) at undo entries, the face slots doubled once at
    the first t <= 249 and kept doubled across later jumps above 249"""
    from brepgen_b200.sampler import CascadeConfig
    from brepgen_b200.schedulers import repaint_entries, repaint_timesteps
    from oracle.repaint import run_cascade_repaint
    cfg = CascadeConfig(batch_size=2, num_surfaces=3, num_edges=2, schedule="repaint", repaint_steps=10,
                        repaint_jump_length=2, repaint_jump_n_sample=3, repaint_eta=0.5, dense_masks=True)
    g = torch.Generator().manual_seed(5)
    init = {"surfPos": torch.randn(2, 3, 6, generator=g), "surfZ": torch.randn(2, 6, 48, generator=g),
            "edgePos": torch.randn(2, 6, 2, 6, generator=g), "edgeZV": torch.randn(2, 6, 2, 18, generator=g)}
    seen, steps, undos = {}, [], []

    def step_noise(name, k, shape):
        steps.append((name, k))
        return torch.randn(tuple(shape), generator=g)

    def undo_noise(name, k, shape):
        undos.append((name, k, tuple(shape)))
        return torch.randn(tuple(shape), generator=g)
    out = run_cascade_repaint(None, cfg, init, step_noise, undo_noise, forwards=_standins(seen))
    ts = repaint_timesteps(10, 2, 3).tolist()
    ents = repaint_entries(ts)
    step_ts = [t for s, t in ents if s]
    assert all([t for t, _ in v] == step_ts for v in seen.values())
    first = step_ts.index(next(t for t in step_ts if t <= 249))
    assert [s[1] for _, s in seen["surfpos"]] == [3] * first + [6] * (len(step_ts) - first)
    assert max(step_ts[first:]) > 249                   # a jump back above 249 after the increase
    assert [k for n, k in steps if n == "surfZ"] == [k for k, (s, _) in enumerate(ents) if s]
    assert [(k, sh[0]) for n, k, sh in undos if n == "edgeZV"] == [(k, 100) for k, (s, _) in enumerate(ents) if not s]
    assert out["surfPos"].shape == (2, 6, 6) and all(torch.isfinite(v.float()).all() for v in out.values())


# -------------------------------------------------------------------------------------------- drop-in host logic
class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("bg_"):
            raise AttributeError(name)

        def f(*a):
            self.calls.append((name, a))
            return 0
        return f


@pytest.fixture
def rec(monkeypatch):
    from brepgen_b200 import _ffi, schedulers
    r = _Recorder()
    monkeypatch.setattr(_ffi, "lib", lambda: r)
    monkeypatch.setattr(_ffi, "current_stream", lambda: 0)
    monkeypatch.setattr(schedulers, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "device", contextlib.nullcontext)
    return r


# positions in the bg_repaint_step / bg_repaint_undo argument lists
S_KNOWN, S_MASK, S_PT, S_NOISE, S_SEED, S_KEYS, S_PER, S_K, S_N, S_COEF, S_CLIP = 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 20
U_N, U_NT, U_COEF, U_NOISE, U_SEED, U_KEYS, U_PER, U_K = 1, 2, 3, 4, 5, 6, 7, 8


def test_dropin_entry_counters_and_noise_keys(rec):
    """the pipeline loop: step and undo_step each take one entry of the list, so keyed and batch noise are counted by the
    entry index; the batch keys are mix_seed(stream key, 3 | 4) and never move the (seed, offset) stream"""
    from brepgen_b200.schedulers import DDIMScheduler, RePaintScheduler, mix_seed
    s = RePaintScheduler(eta=0.5, clip_sample_range=3.0)
    s.set_timesteps(10, 2, 3)
    s.set_noise_seed(7, 0, 2)
    x = torch.zeros(2, 5, 6)
    known = torch.ones(2, 5, 6)
    mask = torch.zeros(2, 5, dtype=torch.bool)
    mask[:, :2] = True
    t_last = int(s.timesteps[0]) + 1
    for t in s.timesteps.tolist():
        if t < t_last:
            s.step(x, t, x, known, mask)
        else:
            s.undo_step(x, t_last)
        t_last = t
    assert len(rec.calls) == len(LIST_10_2_3) and s._philox_offset == 0
    d = DDIMScheduler(clip_sample_range=3.0)
    d.set_timesteps(10)
    for k, (name, a) in enumerate(rec.calls):
        if name == "bg_repaint_step":
            assert a[S_K] == k and a[S_SEED] == mix_seed(mix_seed(7, 0, 2), 3) and a[S_KEYS] is None
            t = 100 * LIST_10_2_3[k]
            assert a[S_COEF:S_COEF + 5] == d.step_coefficients(t, 0.5) and a[S_CLIP] == 3.0
            assert a[S_COEF + 5] == float((1 - d._abar_prev(t)) ** 0.5) and a[S_PT] == 6 and a[S_N] == 60
        else:
            assert name == "bg_repaint_undo" and a[U_K] == k and a[U_NT] == 100 and a[U_N] == 60
            assert a[U_SEED] == mix_seed(mix_seed(7, 0, 2), 4) and a[U_KEYS] is None and a[U_NOISE] is None
    # per-sample keys: per_sample is one sample's element count; set_timesteps restarts the count
    s.set_sample_keys(seed=3, first=4, stage=1)
    s.set_timesteps(10, 2, 3)
    rec.calls.clear()
    s.step(x, 900, x, None, None)
    s.undo_step(x, 800)
    (_, a), (_, u) = rec.calls
    assert a[S_KEYS] is not None and a[S_PER] == 30 and a[S_K] == 0 and a[S_KNOWN] is None and a[S_MASK] is None
    assert u[U_KEYS] is not None and u[U_PER] == 30 and u[U_K] == 1


def test_dropin_undo_coefficients_and_generator(rec):
    from brepgen_b200.schedulers import RePaintScheduler
    s = RePaintScheduler()
    s.set_timesteps(50, 5, 5)
    cf = s.undo_coefficients(300)
    assert cf.shape == (20, 2) and cf.dtype == torch.float32
    for i in range(20):
        beta = s.betas[300 + i]
        assert float(cf[i, 0]) == float((1 - beta) ** 0.5) and float(cf[i, 1]) == float(beta ** 0.5)
    tab = s.undo_table()
    ct = s.coefficient_table()
    for k, t in enumerate(s.timesteps.tolist()):
        if k and t > int(s.timesteps[k - 1]):
            assert torch.equal(tab[k], s.undo_coefficients(int(s.timesteps[k - 1]))) and not ct[k].any()
        else:
            assert not tab[k].any() and ct[k].tolist() == list(torch.tensor(s.step_coefficients(t)).tolist())
    with pytest.raises(ValueError):
        s.undo_coefficients(990)
    # a generator is drawn n times, in order, as diffusers' undo_step draws it
    x = torch.zeros(2, 3, 6)
    g = torch.Generator().manual_seed(4)
    s.undo_step(x, 300, generator=g)
    ref = torch.Generator().manual_seed(4)
    for _ in range(20):
        torch.randn(x.shape, generator=ref)
    assert torch.equal(g.get_state(), ref.get_state()) and rec.calls[-1][1][U_NOISE] is not None
    with pytest.raises(RuntimeError, match="noise"):
        s.undo_step(x, 300, noise=torch.zeros(19, 2, 3, 6))


def test_dropin_masks(rec):
    from brepgen_b200.schedulers import RePaintScheduler
    s = RePaintScheduler()
    s.set_timesteps(10)
    x = torch.zeros(2, 5, 6)
    known = torch.ones(2, 5, 6)
    for ok in (torch.ones(2, 5, dtype=torch.bool), torch.ones(2, 5, 1, dtype=torch.uint8),
               torch.tensor([[1.0, 0, 1, 0, 0], [0, 0, 0, 0, 1]]), torch.zeros(2, 5, 1)):
        s.step(x, 900, x, known, ok)
        m = rec.calls[-1][1][S_MASK]
        assert m is not None
    bad_vals = torch.full((2, 5), 0.5)
    for bad in (bad_vals, torch.ones(2, 5, 6), torch.ones(5), torch.ones(2, 5, dtype=torch.int32)):
        with pytest.raises(ValueError):
            s.step(x, 900, x, known, bad)
    with pytest.raises(ValueError):
        s.step(x, 900, x, known, None)
    with pytest.raises(RuntimeError):
        s.step(x, 900, x, torch.ones(2, 5, 7), torch.ones(2, 5, dtype=torch.bool))
    for bad in (dict(trained_betas=[0.1] * 1000), dict(prediction_type="v_prediction")):
        with pytest.raises(NotImplementedError):
            RePaintScheduler(**bad)
    with pytest.raises(NotImplementedError):
        RePaintScheduler(beta_schedule="squaredcos_cap_v2")
    with pytest.raises(ValueError):
        RePaintScheduler().step(x, 900, x, None, None)            # set_timesteps not called


def test_token_mask_values():
    from brepgen_b200.schedulers import RePaintScheduler
    x = torch.zeros(2, 3, 4)
    m = RePaintScheduler.token_mask(torch.tensor([[1.0, 0.0, 1.0], [0.0, 0.0, 1.0]]), x)
    assert m.dtype == torch.uint8 and m.tolist() == [[1, 0, 1], [0, 0, 1]]
    assert RePaintScheduler.token_mask(torch.tensor([[True], [False], [True]]).reshape(1, 3, 1), x[:1]).tolist() == \
        [[1, 0, 1]]


# --------------------------------------------------------------------------------------------------- validation
def test_cascade_config_validation():
    from brepgen_b200.sampler import Cascade, CascadeConfig, Completion, check_completion, check_schedule
    cfg = CascadeConfig()
    assert (cfg.repaint_steps, cfg.repaint_eta, cfg.repaint_jump_length, cfg.repaint_jump_n_sample) == (250, 0.0, 10, 10)
    for ok in (dict(), dict(repaint_steps=1), dict(repaint_steps=1000, repaint_jump_length=1, repaint_jump_n_sample=1),
               dict(repaint_eta=1.0)):
        check_schedule(CascadeConfig(schedule="repaint", **ok))
    check_schedule(CascadeConfig(schedule="ddim", repaint_steps=0, repaint_eta=-1.0))   # unused by other schedules
    for bad in (dict(repaint_steps=0), dict(repaint_steps=1001), dict(repaint_eta=-0.1), dict(repaint_eta=float("nan")),
                dict(repaint_jump_length=0), dict(repaint_jump_n_sample=0)):
        with pytest.raises(ValueError):
            check_schedule(CascadeConfig(schedule="repaint", **bad))
        with pytest.raises(ValueError):      # run() rejects the config before it touches a device
            Cascade({}, device="cpu").run(CascadeConfig(schedule="repaint", **bad))
    known = Completion(n_faces=[1, 0], surfPos=torch.zeros(2, 1, 6))
    assert check_completion(CascadeConfig(batch_size=2, schedule="repaint"), known).tolist() == [1, 0]
    with pytest.raises(ValueError):
        check_completion(CascadeConfig(batch_size=3, schedule="repaint"), known)
    with pytest.raises(NotImplementedError, match="repaint"):
        check_completion(CascadeConfig(batch_size=2, schedule="reference"), known)
    c = Cascade({}, device="cpu")
    assert (c.repaint.config.clip_sample, c.repaint.config.clip_sample_range) == (True, 3)
    assert torch.equal(c.repaint.alphas_cumprod, c.ddim.alphas_cumprod)
    assert np.array_equal(c.repaint.betas.numpy(), c.ddpm.betas.numpy())
