"""CPU tests of the DPM-Solver++ scheduler: the oracle against diffusers' known answer, its timestep / sigma tables, first
order = DDIM, second-order convergence on a Gaussian problem with a closed-form solution, and the host logic of the
DPMSolverMultistepScheduler drop-in and CascadeConfig(schedule="dpm")."""
import contextlib

import numpy as np
import pytest
import torch

from oracle.ddim import DDIMOracle
from oracle.dpm import DPMOracle
from test_oracle_sched_kat import dummy_model, dummy_sample_deter

# diffusers' tests/schedulers/test_scheduler_dpm_multi.py::test_full_loop_no_noise: 10 steps of its default test config,
# which sets lower_order_final=False and final_sigmas_type="sigma_min" (so the last step is second order and ends at the
# smallest training sigma), |x| mean 0.3301.  The product supports final_sigmas_type="zero" only; under it the same loop
# ends at 0.2409 (DPM_ZERO_MEAN, this oracle's value, reproduced by the product kernel in test_gpu_dpm.py).
DPM_KAT_CONFIG = dict(lower_order_final=False, final_sigmas_type="sigma_min")
DPM_KAT_MEAN = 0.3301
DPM_ZERO_MEAN = 0.2409


def _full_loop(sch):
    sch.set_timesteps(10)
    x = dummy_sample_deter()
    for t in sch.timesteps:
        x = sch.step(dummy_model(x, int(t)), int(t), x)
    return x


def test_dpm_oracle_full_loop_matches_diffusers_known_answer():
    x = _full_loop(DPMOracle(**DPM_KAT_CONFIG))
    assert abs(float(x.abs().mean()) - DPM_KAT_MEAN) < 1e-3
    z = _full_loop(DPMOracle())
    assert abs(float(z.abs().mean()) - DPM_ZERO_MEAN) < 1e-4


def _diffusers_timesteps(spacing, n, steps_offset=0):
    """diffusers 0.27 DPMSolverMultistepScheduler.set_timesteps, lambda_min_clipped = -inf (last_timestep = 1000)"""
    if spacing == "linspace":
        return np.linspace(0, 999, n + 1).round()[::-1][:-1].astype(np.int64).tolist()
    if spacing == "leading":
        ratio = 1000 // (n + 1)
        return [int(v) + steps_offset for v in (np.arange(0, n + 1) * ratio).round()[::-1][:-1]]
    return [int(v) - 1 for v in np.arange(1000, 0, -1000 / n).round()]


@pytest.mark.parametrize("n", [10, 20, 25])
@pytest.mark.parametrize("spacing", ["linspace", "leading", "trailing"])
def test_timestep_and_sigma_tables(spacing, n):
    from brepgen_b200.schedulers import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler(timestep_spacing=spacing, steps_offset=1 if spacing == "leading" else 0)
    s.set_timesteps(n)
    want = _diffusers_timesteps(spacing, n, 1 if spacing == "leading" else 0)
    assert s.timesteps.tolist() == want and s.timesteps.dtype == torch.int64 and s.num_inference_steps == n
    acp = s.alphas_cumprod.double()
    sig = ((1 - acp) / acp).sqrt()
    assert s.sigmas.dtype == torch.float32 and s.sigmas.shape == (n + 1,) and float(s.sigmas[-1]) == 0.0
    assert torch.allclose(s.sigmas[:-1].double(), sig[torch.tensor(want)], rtol=1e-6)
    o = DPMOracle(timestep_spacing=spacing, steps_offset=1 if spacing == "leading" else 0)
    o.set_timesteps(n)
    assert torch.equal(s.timesteps, o.timesteps) and torch.equal(s.sigmas, o.sigmas)
    if spacing == "linspace" and n == 10:
        assert want == [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]


def test_which_steps_are_first_order():
    from brepgen_b200.schedulers import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(20)
    assert [s.step_order(k) for k in range(20)] == [1] + [2] * 18 + [1]
    assert [s.step_order(k, restart=12) for k in range(20)] == [1] + [2] * 11 + [1] + [2] * 6 + [1]
    tab = s.coefficient_table(s.timesteps, restart=12)
    assert tab.shape == (20, 7) and tab.dtype == torch.float32
    assert [k for k in range(20) if float(tab[k, 4]) == 0.0] == [0, 12, 19]
    assert [k for k in range(20) if float(tab[k, 5]) == 0.0] == [0, 12, 19]      # inv_r0 only on second-order rows
    assert torch.equal(s.coefficient_table(s.timesteps[12:], restart=0), tab[12:])  # a segment's rows: a slice
    assert float(tab[19, 2]) == 0.0 and float(tab[19, 3]) == 1.0              # last step: x = x0 (sigma_next = 0)
    assert (tab[:, 6] == 0).all()                                             # ODE: no noise
    one = DPMSolverMultistepScheduler(solver_order=1)
    one.set_timesteps(20)
    assert (one.coefficient_table()[:, 4] == 0).all()
    sde = DPMSolverMultistepScheduler(algorithm_type="sde-dpmsolver++")
    sde.set_timesteps(20)
    st = sde.coefficient_table()
    assert (st[:-1, 6] > 0).all() and float(st[-1, 6]) == 0.0


@pytest.mark.parametrize("clip", [False, True])
def test_first_order_step_is_the_ddim_step(clip):
    """a first-order DPM-Solver++ step from t to t' is the eta = 0 DDIM step from t to abar_t' (algebraically; with the
    clamp, DDIM's epsilon recomputed from the clipped x0).  'leading' with N = 9 steps lands on DDIM's N = 10 table."""
    g = torch.Generator().manual_seed(0)
    x, eps = torch.randn(4, 500, generator=g) * 2, torch.randn(4, 500, generator=g) * 2
    dpm = DPMOracle(solver_order=1, timestep_spacing="leading", clip_sample=clip, clip_sample_range=1.0)
    dpm.set_timesteps(9)
    assert dpm.timesteps.tolist() == list(range(900, 0, -100))
    worst = 0.0
    for k, t in enumerate(dpm.timesteps.tolist()):
        ddim = DDIMOracle(clip_sample=clip, clip_sample_range=1.0, set_alpha_to_one=True)
        ddim.set_timesteps(10 if k < 8 else 9)          # prev_t = t - 100, or < 0 (abar = 1) for the last step
        dpm.step_index = k
        a = dpm.step(eps, t, x)
        b = ddim.step(eps, t, x, eta=0.0, use_clipped_model_output=clip)
        err = float((a - b).abs().max() / max(1.0, float(b.abs().max())))
        worst = max(worst, err)
        assert err < 1e-6, (t, err)
    print(f"first-order DPM vs DDIM (clip={clip}): worst {worst:.2e}")


# ---------------------------------------------------------------------------------------- Gaussian convergence
MU, SD = 0.7, 0.4


def gaussian_problem(n=100_000, seed=0):
    """x0 ~ N(MU, SD^2) per element: the exact eps-predictor and the exact probability-flow endpoint of a start x_T"""
    acp = DPMOracle().acp.double()

    def eps_star(x, t):
        a = acp[int(t)]
        return ((1 - a).sqrt() * (x.double() - a.sqrt() * MU) / (a * SD ** 2 + 1 - a)).float()
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(n, generator=g, dtype=torch.float64)
    aT = acp[999]
    xT = (aT.sqrt() * MU + (aT * SD ** 2 + 1 - aT).sqrt() * z).float()
    return xT, eps_star, (MU + SD * z).float(), g


def _rms(a, b):
    return float((a.double() - b.double()).pow(2).mean().sqrt())


def test_second_order_converges_faster_than_ddim():
    xT, eps_star, exact, _ = gaussian_problem()
    ratios = {}
    for n in (20, 50):
        d = DDIMOracle(clip_sample=False, set_alpha_to_one=True)
        d.set_timesteps(n)
        xd = xT.clone()
        for t in d.timesteps:
            xd = d.step(eps_star(xd, t), int(t), xd)
        p = DPMOracle()
        p.set_timesteps(n)
        xp = xT.clone()
        for t in p.timesteps:
            xp = p.step(eps_star(xp, t), int(t), xp)
        ratios[n] = _rms(xp, exact) / _rms(xd, exact)
        print(f"Gaussian N={n}: DDIM rms {_rms(xd, exact):.4f}  DPM++ 2M rms {_rms(xp, exact):.4f}  ratio {ratios[n]:.3f}")
    assert ratios[20] <= 0.6 and ratios[50] <= 0.15


def test_sde_form_samples_the_target_distribution():
    xT, eps_star, _, g = gaussian_problem(seed=1)
    p = DPMOracle(algorithm_type="sde-dpmsolver++")
    p.set_timesteps(100)
    x = xT.clone()
    for t in p.timesteps:
        x = p.step(eps_star(x, t), int(t), x, noise=torch.randn(x.shape, generator=g))
    print(f"SDE 100 steps: mean {float(x.mean()):.4f} std {float(x.std()):.4f}")
    assert abs(float(x.mean()) - MU) < 0.01 and abs(float(x.std()) / SD - 1) < 0.05


# -------------------------------------------------------------------------------------------- host logic
def test_unsupported_settings_and_errors():
    from brepgen_b200.schedulers import DPMSolverMultistepScheduler
    for kw in (dict(prediction_type="v_prediction"), dict(prediction_type="sample"), dict(thresholding=True),
               dict(use_karras_sigmas=True), dict(use_lu_lambdas=True), dict(solver_order=3),
               dict(algorithm_type="dpmsolver"), dict(algorithm_type="sde-dpmsolver"), dict(solver_type="heun"),
               dict(final_sigmas_type="sigma_min"), dict(lambda_min_clipped=-5.1), dict(trained_betas=[0.1] * 1000),
               dict(variance_type="learned_range"), dict(beta_schedule="squaredcos_cap_v2")):
        with pytest.raises(NotImplementedError):
            DPMSolverMultistepScheduler(**kw)
    s = DPMSolverMultistepScheduler()
    assert s.num_inference_steps is None and len(s.timesteps) == 1000 and s.init_noise_sigma == 1.0 and len(s) == 1000
    assert s.config.lower_order_final and not s.config.euler_at_final and not s.config.clip_sample
    with pytest.raises(ValueError):
        s.set_timesteps(1001)
    x = torch.zeros(2, 4)
    with pytest.raises(ValueError, match="set_timesteps"):        # diffusers: step before set_timesteps
        s.step(x, 10, x)
    assert s.scale_model_input(x, 5) is x


def test_cascade_config_validation():
    from brepgen_b200.sampler import Cascade, CascadeConfig, check_schedule
    cfg = CascadeConfig()
    assert (cfg.dpm_steps, cfg.dpm_order, cfg.dpm_algorithm) == (20, 2, "dpmsolver++")
    for ok in (dict(dpm_steps=1), dict(dpm_steps=1000), dict(dpm_order=1), dict(dpm_algorithm="sde-dpmsolver++")):
        check_schedule(CascadeConfig(schedule="dpm", **ok))
    check_schedule(CascadeConfig(schedule="ddim", dpm_steps=0, dpm_order=5))     # DPM fields unused by other schedules
    for bad in (dict(dpm_steps=0), dict(dpm_steps=1001), dict(dpm_order=3), dict(dpm_order=0),
                dict(dpm_algorithm="dpmsolver"), dict(dpm_algorithm="heun")):
        with pytest.raises(ValueError):
            check_schedule(CascadeConfig(schedule="dpm", **bad))
        with pytest.raises(ValueError):      # run() rejects the config before it touches a device
            Cascade({}, device="cpu").run(CascadeConfig(schedule="dpm", **bad))
    c = Cascade({}, device="cpu")
    assert (c.dpm.config.clip_sample, c.dpm.config.clip_sample_range, c.dpm.config.solver_order) == (True, 3, 2)
    assert torch.equal(c.dpm.alphas_cumprod, c.ddpm.alphas_cumprod)


def test_replacement_levels():
    """replace_table: the level 1 / (1 + sigma_next^2) each step leaves x at, exactly (1, 0) after the last step"""
    from brepgen_b200.schedulers import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler(clip_sample=True, clip_sample_range=3)
    s.set_timesteps(20)
    tab = s.replace_table(s.timesteps)
    assert tab.shape == (20, 2) and tab[-1].tolist() == [1.0, 0.0]
    sig = s.sigmas.double()
    a = 1 / (1 + sig[1:] ** 2)
    assert torch.allclose(tab.double(), torch.stack([a.sqrt(), (1 - a).sqrt()], 1), atol=1e-6)
    assert s.replace_coefficients(int(s.timesteps[3])) == tuple(tab[3].tolist())
    assert s.replace_coefficients(999, initial=True) == (float(s.alphas_cumprod[999] ** 0.5),
                                                         float((1 - s.alphas_cumprod[999]) ** 0.5))


class _FakeLib:
    """records bg_dpm_step calls instead of launching (host-logic tests run without a device)"""

    def __init__(self):
        self.calls = []

    def bg_dpm_step(self, *a):
        self.calls.append(a)
        return 0


@pytest.fixture
def fake_lib(monkeypatch):
    from brepgen_b200 import _ffi, schedulers
    fake = _FakeLib()
    monkeypatch.setattr(_ffi, "lib", lambda: fake)
    monkeypatch.setattr(_ffi, "current_stream", lambda: 0)
    monkeypatch.setattr(schedulers, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "device", contextlib.nullcontext)
    return fake


# positions in the bg_dpm_step argument list
A_HIST, A_NOISE, A_SEED, A_OFFSET, A_KEYS, A_PER, A_T, A_N, A_C1, A_INV, A_CZ, A_CLIP = 5, 6, 7, 8, 9, 10, 11, 12, 17, 18, 19, 20


@pytest.mark.parametrize("algorithm", ["dpmsolver++", "sde-dpmsolver++"])
def test_generator_and_stream_advance_once_per_step_only_in_sde_mode(fake_lib, algorithm):
    from brepgen_b200.schedulers import DPMSolverMultistepScheduler
    sde = algorithm == "sde-dpmsolver++"
    s = DPMSolverMultistepScheduler(algorithm_type=algorithm, clip_sample=True, clip_sample_range=3)
    s.set_timesteps(10)
    x = torch.zeros(2, 3, 5)
    g = torch.Generator().manual_seed(4)
    st = g.get_state()
    for t in s.timesteps:
        s.step(x, t, x, generator=g)
    ref = torch.Generator().manual_seed(4)
    for _ in range(10 if sde else 0):
        torch.randn(x.shape, generator=ref)
    assert torch.equal(g.get_state(), ref.get_state()) and (sde or torch.equal(g.get_state(), st))
    calls = fake_lib.calls
    assert len(calls) == 10 and all((c[A_NOISE] is not None) == sde for c in calls)
    assert [c[A_C1] == 0.0 for c in calls] == [True] + [False] * 8 + [True]
    assert all(c[A_HIST] is not None and c[A_CLIP] == 3.0 for c in calls)
    assert calls[-1][A_CZ] == 0.0 and (calls[0][A_CZ] > 0.0) == sde
    assert s.step_index == 10 and s.lower_order_nums == 2
    # batch stream: one element-group count per step in SDE mode (the last step included), none for the ODE
    calls.clear()
    s.set_timesteps(4)
    assert s.step_index is None and s.lower_order_nums == 0 and s.model_outputs == [None, None]
    y = torch.zeros(3, 7)                   # n = 21: 6 groups of 4
    s.set_noise_seed(5, 0, 2)
    for t in s.timesteps:
        s.step(y, t, y)
    assert [c[A_OFFSET] for c in calls] == ([0, 6, 12, 18] if sde else [0] * 4)
    assert all(c[A_KEYS] is None and c[A_NOISE] is None for c in calls) and calls[0][A_N] == 21
    assert s._philox_offset == (24 if sde else 0)
    calls.clear()
    s.set_timesteps(4)
    s.set_sample_keys(seed=3, first=10, stage=1)
    s.step(y, s.timesteps[0], y)
    c = calls[0]
    assert (c[A_KEYS] is not None) == sde and c[A_PER] == 7 and c[A_T] == int(s.timesteps[0])


def test_shape_change_restarts_the_solver(fake_lib):
    """the late face-count increase: the step on the doubled sample is first order with a new history buffer"""
    from brepgen_b200.schedulers import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(10)
    x = torch.zeros(2, 3, 6)
    for t in s.timesteps[:5]:
        s.step(x, t, x)
    h = s.hist
    x2 = x.repeat(1, 2, 1)
    for t in s.timesteps[5:]:
        s.step(x2, t, x2)
    assert [c[A_C1] == 0.0 for c in fake_lib.calls] == [True, False, False, False, False, True, False, False, False, True]
    assert s.hist is not h and tuple(s.hist.shape) == (2, 6, 6)


def test_oracle_dpm_cascade_driver():
    """oracle.dpm.run_cascade_dpm with stand-in networks: one forward per step and stage, step noise on every step of the
    SDE form only, the face slots doubled from the first t <= 249 on; with nothing known it is the plain driver"""
    from brepgen_b200.sampler import CascadeConfig, Completion
    from oracle.dpm import run_cascade_dpm
    for use_cf, algo in ((False, "sde-dpmsolver++"), (True, "dpmsolver++")):
        cfg = CascadeConfig(batch_size=2, num_surfaces=3, num_edges=2, use_cf=use_cf, class_label=6, schedule="dpm",
                            dpm_steps=10, dpm_algorithm=algo, dense_masks=True)
        S = 3 if use_cf else 6
        g = torch.Generator().manual_seed(1)
        init = {"surfPos": torch.randn(2, 3, 6, generator=g), "surfZ": torch.randn(2, S, 48, generator=g),
                "edgePos": torch.randn(2, S, 2, 6, generator=g), "edgeZV": torch.randn(2, S, 2, 18, generator=g)}
        seen, bank = {}, {}

        def fwd(kind):
            def f(x, t, *rest):
                seen.setdefault(kind, []).append((int(t), tuple(x.shape)))
                return torch.tanh(x) * 0.5
            return f

        def step_noise(name, k, shape):
            if (name, k) not in bank:
                bank[(name, k)] = torch.randn(tuple(shape), generator=g)
            return bank[(name, k)]
        F = {k: fwd(k) for k in ("surfpos", "surfz", "edgepos", "edgez")}
        out = run_cascade_dpm(None, cfg, init, step_noise, F)
        ts = [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]
        mult = 2 if use_cf else 1
        assert [t for t, _ in seen["surfpos"]] == ts and all(len(v) == 10 for v in seen.values())
        assert [s[1] for _, s in seen["surfpos"]] == [3 if (use_cf or t > 249) else 6 for t in ts]
        assert all(s[0] == 2 * mult for v in seen.values() for _, s in v)
        assert len(bank) == (40 if algo == "sde-dpmsolver++" else 0)
        assert out["surfPos"].shape == (2, S, 6) and out["edgeV"].shape == (2, S, 2, 6)
        assert all(torch.isfinite(v.float()).all() for v in out.values())
        nothing = Completion(n_faces=[0, 0], surfPos=torch.zeros(2, 0, 6))
        cfg.dense_masks = False
        ref = run_cascade_dpm(None, cfg, init, step_noise, F)
        got = run_cascade_dpm(None, cfg, init, step_noise, F, known=nothing,
                              replace_noise=lambda name, k, shape: torch.randn(tuple(shape), generator=g))
        for k in ref:
            assert torch.equal(got[k], ref[k]), (use_cf, k)
