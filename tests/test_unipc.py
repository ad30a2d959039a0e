"""CPU tests of the UniPC scheduler: the oracle against diffusers' published answer, its timestep / sigma tables, the order
and corrector of every step, UniPC = DDIM / DPM-Solver++ 2M where the algebra says so, the Gaussian problem, the
coefficient rows the kernel reads (through a torch model of its arithmetic), the oracle cascade driver, and the host
logic of the UniPCMultistepScheduler drop-in and CascadeConfig(schedule="unipc")."""
import contextlib
import ctypes

import pytest
import torch

from oracle.ddim import DDIMOracle
from oracle.dpm import DPMOracle
from oracle.unipc import UniPCOracle
from test_dpm import _diffusers_timesteps, _rms, gaussian_problem
from test_oracle_sched_kat import dummy_model, dummy_sample_deter

# diffusers' tests/schedulers/test_scheduler_unipc.py::test_full_loop_no_noise: 10 steps of its default test config
# (solver_order 2, bh2, linear betas 1e-4 .. 0.02, the sigma_min end), |x| mean 0.2464.
UNIPC_KAT_MEAN = 0.2464
# The same loop under other settings.  Not published answers: values of an independent restatement of diffusers' code,
# which this oracle reproduces to every printed digit.
UNIPC_VARIANTS = [(dict(final_sigmas_type="zero"), 0.2432), (dict(solver_type="bh1"), 0.2521),
                  (dict(solver_order=3), 0.2474), (dict(solver_order=1), 0.2324), (dict(lower_order_final=False), 0.3334)]


def _full_loop(sch, n=10):
    sch.set_timesteps(n)
    x = dummy_sample_deter()
    for t in sch.timesteps:
        x = sch.step(dummy_model(x, int(t)), int(t), x)
    return x


def test_unipc_oracle_full_loop_matches_diffusers_known_answer():
    assert abs(float(_full_loop(UniPCOracle()).abs().mean()) - UNIPC_KAT_MEAN) < 1e-3
    for kw, mean in UNIPC_VARIANTS:
        got = float(_full_loop(UniPCOracle(**kw)).abs().mean())
        assert abs(got - mean) < 6e-5, (kw, got)


@pytest.mark.parametrize("final", ["sigma_min", "zero"])
@pytest.mark.parametrize("n", [10, 20])
@pytest.mark.parametrize("spacing", ["linspace", "leading", "trailing"])
def test_timestep_and_sigma_tables(spacing, n, final):
    from brepgen_b200.schedulers import UniPCMultistepScheduler
    off = 1 if spacing == "leading" else 0
    s = UniPCMultistepScheduler(timestep_spacing=spacing, steps_offset=off, final_sigmas_type=final)
    s.set_timesteps(n)
    want = _diffusers_timesteps(spacing, n, off)
    assert s.timesteps.tolist() == want and s.timesteps.dtype == torch.int64 and s.num_inference_steps == n
    acp = s.alphas_cumprod.double()
    sig = ((1 - acp) / acp).sqrt()
    assert s.sigmas.dtype == torch.float32 and s.sigmas.shape == (n + 1,)
    assert torch.allclose(s.sigmas[:-1].double(), sig[torch.tensor(want)], rtol=1e-6)
    last = float(s.sigmas[-1])
    assert last == 0.0 if final == "zero" else abs(last - float(sig[0])) < 1e-8
    o = UniPCOracle(timestep_spacing=spacing, steps_offset=off, final_sigmas_type=final)
    o.set_timesteps(n)
    assert torch.equal(s.timesteps, o.timesteps) and torch.equal(s.sigmas, o.sigmas)
    if spacing == "linspace" and n == 10:
        assert want == [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]


def test_order_and_corrector_of_every_step():
    """(corrector order, predictor order) per step: the warm-up, lower_order_final, disable_corrector and a restart"""
    from brepgen_b200.schedulers import UniPCMultistepScheduler as U

    def plan(n=10, restart=None, **kw):
        s = U(**kw)
        s.set_timesteps(n)
        return s.step_plan(0, n, restart)
    assert plan() == [(0, 1)] + [(1, 2)] + [(2, 2)] * 7 + [(2, 1)]
    assert plan(solver_order=3) == [(0, 1), (1, 2), (2, 3)] + [(3, 3)] * 5 + [(3, 2), (2, 1)]
    assert plan(solver_order=3, lower_order_final=False) == [(0, 1), (1, 2), (2, 3)] + [(3, 3)] * 7
    assert plan(solver_order=1) == [(0, 1)] + [(1, 1)] * 9
    assert plan(disable_corrector=[0, 4]) == [(0, 1), (0, 2)] + [(2, 2)] * 3 + [(0, 2)] + [(2, 2)] * 3 + [(2, 1)]
    assert plan(restart=6) == [(0, 1), (1, 2)] + [(2, 2)] * 4 + [(0, 1), (1, 2), (2, 2), (2, 1)]
    s = U(solver_order=3)
    s.set_timesteps(20)
    tab = s.coefficient_table(s.timesteps, restart=12)
    assert tab.shape == (20, 24) and tab.dtype == torch.float32
    assert torch.equal(s.coefficient_table(s.timesteps[12:], restart=0), tab[12:])   # a segment's rows: a slice
    assert tab[:, 2].tolist() == [0, 1, 2] + [3] * 9 + [0, 1, 2] + [3] * 3 + [3, 2]
    assert tab[:, 3].tolist() == [1, 2] + [3] * 10 + [1, 2] + [3] * 4 + [2, 1]
    assert tab[:, 4].tolist() == [k % 3 for k in range(20)]
    assert tab[:, 5].tolist() == [(k - 1) % 3 for k in range(20)]


@pytest.mark.parametrize("final", ["sigma_min", "zero"])
@pytest.mark.parametrize("solver_type", ["bh1", "bh2"])
@pytest.mark.parametrize("order", [1, 2, 3])
def test_every_table_row_is_finite(order, solver_type, final):
    from brepgen_b200.schedulers import UniPCMultistepScheduler
    s = UniPCMultistepScheduler(solver_order=order, solver_type=solver_type, final_sigmas_type=final)
    for n in (1, 2, 3, 10, 25):
        s.set_timesteps(n)
        tab = s.coefficient_table()
        assert torch.isfinite(tab).all(), (n, tab)
        if final == "zero":          # into sigma = 0 the step is x0: c_x = 0, c_m0 = -1
            assert tab[-1, 16:19].tolist() == [0.0, -1.0, 0.0] and tab[-1, 3] == 1


# ---------------------------------------------------------------------------------------------- identities
def test_order_one_without_corrector_is_ddim():
    """UniPC order 1 with the corrector off is DPM-Solver++ first order: the eta = 0 DDIM step from t to abar_t'
    ('leading' with N = 9 steps lands on DDIM's N = 10 table)"""
    g = torch.Generator().manual_seed(0)
    x, eps = torch.randn(4, 500, generator=g) * 2, torch.randn(4, 500, generator=g) * 2
    u = UniPCOracle(solver_order=1, timestep_spacing="leading", final_sigmas_type="zero",
                    disable_corrector=range(10))
    u.set_timesteps(9)
    worst = 0.0
    for k, t in enumerate(u.timesteps.tolist()):
        ddim = DDIMOracle(clip_sample=False, set_alpha_to_one=True)
        ddim.set_timesteps(10 if k < 8 else 9)
        u.restart()
        u.step_index = k
        a, b = u.step(eps, t, x), ddim.step(eps, t, x, eta=0.0)
        err = float((a - b).abs().max() / max(1.0, float(b.abs().max())))
        worst = max(worst, err)
        assert err < 1e-6, (t, err)
    print(f"UniPC order 1 vs DDIM: worst {worst:.2e}")


@pytest.mark.parametrize("n", [10, 20])
def test_order_two_bh2_without_corrector_is_dpm_solver_2m(n):
    g = torch.Generator().manual_seed(n)
    x0 = torch.randn(3, 300, generator=g)
    u = UniPCOracle(solver_order=2, solver_type="bh2", final_sigmas_type="zero", disable_corrector=range(n))
    d = DPMOracle(solver_order=2)
    for o in (u, d):
        o.set_timesteps(n)
    xu, xd = x0.clone(), x0.clone()
    for t in u.timesteps:
        xu = u.step(torch.tanh(xu * 0.7) + 0.1, int(t), xu)
        xd = d.step(torch.tanh(xd * 0.7) + 0.1, int(t), xd)
    err = float((xu - xd).abs().max() / xd.abs().max())
    print(f"UniPC-2 bh2 without corrector vs DPM++ 2M, N={n}: {err:.2e}")
    assert err < 1e-6         # fp32 rounding: the two form the same update from differently rounded scalars


def test_gaussian_problem_corrector_beats_dpm_2m():
    """x0 ~ N(0.7, 0.4^2) with the exact eps-predictor: UniPC-2 (bh2, with its corrector) ends closer to the exact ODE
    solution than DPM-Solver++ 2M with the same network evaluations"""
    xT, eps_star, exact, _ = gaussian_problem()
    for n in (10, 20):
        runs = {}
        for name, o in (("dpm", DPMOracle()), ("unipc2", UniPCOracle(final_sigmas_type="zero")),
                        ("unipc3", UniPCOracle(solver_order=3, final_sigmas_type="zero"))):
            o.set_timesteps(n)
            x = xT.clone()
            for t in o.timesteps:
                x = o.step(eps_star(x, t), int(t), x)
            runs[name] = _rms(x, exact)
        print(f"Gaussian N={n}: " + "  ".join(f"{k} rms {v:.4f}" for k, v in runs.items()))
        assert runs["unipc2"] < runs["dpm"]


# ------------------------------------------------------------------------------------ the rows the kernel reads
def kernel_model(row, e, x, last, hist, clip=0.0):
    """unipc_step_kernel's arithmetic in fp32 torch, one rounding per operation in the kernel's order: (out, new last,
    new hist) from one BG_UNIPC_ROW row"""
    r = [torch.tensor(v, dtype=torch.float32) for v in row.tolist()]
    c, p = int(r[2]), int(r[3])
    sn, s1, s2, s3 = (int(v) for v in r[4:8])
    x0 = (x - r[1] * e) / r[0]
    if clip > 0:
        x0 = x0.clamp(-clip, clip)
    m1, m2, m3 = hist[s1], hist[s2], hist[s3]
    xc = x
    if c > 0:
        tail = r[15] * (x0 - m1)
        res = tail
        if c >= 2:
            res = r[13] * ((m2 - m1) / r[11])
            if c >= 3:
                res = res + r[14] * ((m3 - m1) / r[12])
            res = res + tail
        xc = r[8] * last - r[9] * m1 - r[10] * res
    o = r[16] * xc - r[17] * x0
    if p >= 2:
        res = r[21] * ((m1 - x0) / r[19])
        if p >= 3:
            res = res + r[22] * ((m2 - x0) / r[20])
        o = o - r[18] * res
    hist = hist.clone()
    hist[sn] = x0
    return o, xc, hist


@pytest.mark.parametrize("kw", [dict(), dict(final_sigmas_type="zero"), dict(solver_type="bh1"), dict(solver_order=3),
                                dict(solver_order=1), dict(lower_order_final=False),
                                dict(solver_order=3, solver_type="bh1", final_sigmas_type="zero", clip_sample=True),
                                dict(solver_order=3, disable_corrector=[2, 5])], ids=str)
def test_coefficient_rows_reproduce_the_oracle(kw):
    """the product's coefficient table, evaluated by a model of the kernel's arithmetic, follows the oracle: exactly at
    orders 1 and 2; at order 3 within the rounding of the oracle's einsum"""
    from brepgen_b200.schedulers import UniPCMultistepScheduler
    for n in (10, 20):
        s, o = UniPCMultistepScheduler(**kw), UniPCOracle(**kw)
        s.set_timesteps(n)
        tab = s.coefficient_table()
        clip = float(s.config.clip_sample_range) if s.config.clip_sample else 0.0
        x = xo = dummy_sample_deter() * 4 - 1
        hist, last = torch.zeros((s.config.solver_order,) + x.shape), torch.zeros_like(x)
        o.set_timesteps(n)
        for k, t in enumerate(s.timesteps.tolist()):
            x, last, hist = kernel_model(tab[k], dummy_model(x, t), x, last, hist, clip)
            xo = o.step(dummy_model(xo, t), t, xo)
        err = float((x - xo).abs().max() / xo.abs().max())
        assert err < (1e-6 if s.config.solver_order == 3 else 1e-7) and (s.config.solver_order == 3 or err == 0.0), err


# -------------------------------------------------------------------------------------------- oracle cascade driver
def test_oracle_unipc_cascade_driver():
    """oracle.unipc.run_cascade_unipc with stand-in networks: one forward per step and stage (none for the corrector),
    the face slots doubled from the first t <= 249 on with a restart there; with nothing known it is the plain driver"""
    from brepgen_b200.sampler import CascadeConfig, Completion
    from oracle import unipc as U
    for use_cf in (False, True):
        cfg = CascadeConfig(batch_size=2, num_surfaces=3, num_edges=2, use_cf=use_cf, class_label=6, schedule="unipc",
                            unipc_steps=10, unipc_order=3, dense_masks=True)
        S = 3 if use_cf else 6
        g = torch.Generator().manual_seed(1)
        init = {"surfPos": torch.randn(2, 3, 6, generator=g), "surfZ": torch.randn(2, S, 48, generator=g),
                "edgePos": torch.randn(2, S, 2, 6, generator=g), "edgeZV": torch.randn(2, S, 2, 18, generator=g)}
        seen = {}

        def fwd(kind):
            def f(x, t, *rest):
                seen.setdefault(kind, []).append((int(t), tuple(x.shape)))
                return torch.tanh(x) * 0.5
            return f
        F = {k: fwd(k) for k in ("surfpos", "surfz", "edgepos", "edgez")}
        restarts = []
        real = UniPCOracle.restart

        def spy(self):
            restarts.append(getattr(self, "step_index", None))
            real(self)
        UniPCOracle.restart = spy
        try:
            out = U.run_cascade_unipc(None, cfg, init, F)
        finally:
            UniPCOracle.restart = real
        ts = [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]
        mult = 2 if use_cf else 1
        assert [t for t, _ in seen["surfpos"]] == ts and all(len(v) == 10 for v in seen.values())
        assert [s[1] for _, s in seen["surfpos"]] == [3 if (use_cf or t > 249) else 6 for t in ts]
        assert all(s[0] == 2 * mult for v in seen.values() for _, s in v)
        # set_timesteps restarts at every stage (index None, or 10 after a stage); the late increase once, mid-loop,
        # before the step at t = 200
        assert [r for r in restarts if r is not None and r < 10] == ([] if use_cf else [8])
        assert out["surfPos"].shape == (2, S, 6) and out["edgeV"].shape == (2, S, 2, 6)
        assert all(torch.isfinite(v.float()).all() for v in out.values())
        nothing = Completion(n_faces=[0, 0], surfPos=torch.zeros(2, 0, 6))
        cfg.dense_masks = False
        ref = U.run_cascade_unipc(None, cfg, init, F)
        got = U.run_cascade_unipc(None, cfg, init, F, known=nothing,
                                  replace_noise=lambda name, k, shape: torch.randn(tuple(shape), generator=g))
        for k in ref:
            assert torch.equal(got[k], ref[k]), (use_cf, k)
        from oracle import dpm, variation
        assert dpm.DPMOracle is DPMOracle and variation.DPMOracle is DPMOracle      # the drivers are left as they were


# -------------------------------------------------------------------------------------------------- host logic
def test_unsupported_settings_and_errors():
    from brepgen_b200.schedulers import UniPCMultistepScheduler as U
    for kw in (dict(prediction_type="v_prediction"), dict(prediction_type="sample"), dict(predict_x0=False),
               dict(solver_p=object()), dict(thresholding=True), dict(use_karras_sigmas=True),
               dict(trained_betas=[0.1] * 1000), dict(solver_order=4), dict(solver_order=0), dict(solver_type="bh3"),
               dict(final_sigmas_type="karras"), dict(timestep_spacing="log"), dict(beta_schedule="squaredcos_cap_v2"),
               dict(final_sigmas_type="zero", lower_order_final=False),
               dict(final_sigmas_type="zero", lower_order_final=False, solver_type="bh1", solver_order=3)):
        with pytest.raises(NotImplementedError):
            U(**kw)
    U(final_sigmas_type="zero", lower_order_final=False, solver_order=1)      # a first-order last step has a limit
    assert U(solver_type="midpoint").config.solver_type == "bh2"            # diffusers' mapping
    s = U()
    assert s.num_inference_steps is None and len(s.timesteps) == 1000 and s.init_noise_sigma == 1.0 and len(s) == 1000
    assert s.config.lower_order_final and s.config.final_sigmas_type == "sigma_min" and not s.config.clip_sample
    assert s.last_sample is None and s.model_outputs == [None, None] and s.step_index is None
    with pytest.raises(ValueError):
        s.set_timesteps(1001)
    x = torch.zeros(2, 4)
    with pytest.raises(ValueError, match="set_timesteps"):
        s.step(x, 10, x)
    assert s.scale_model_input(x, 5) is x


def test_cascade_config_validation():
    from brepgen_b200.sampler import (Cascade, CascadeConfig, Interpolation, Variation, check_interpolation,
                                      check_schedule, check_variation, stage_timesteps)
    cfg = CascadeConfig()
    assert (cfg.unipc_steps, cfg.unipc_order, cfg.unipc_solver_type) == (10, 2, "bh2")
    for ok in (dict(unipc_steps=1), dict(unipc_steps=1000), dict(unipc_order=1), dict(unipc_order=3),
               dict(unipc_solver_type="bh1")):
        check_schedule(CascadeConfig(schedule="unipc", **ok))
    check_schedule(CascadeConfig(schedule="dpm", unipc_steps=0, unipc_order=7))    # UniPC fields unused elsewhere
    for bad in (dict(unipc_steps=0), dict(unipc_steps=1001), dict(unipc_order=0), dict(unipc_order=4),
                dict(unipc_solver_type="midpoint"), dict(unipc_solver_type="bh3")):
        with pytest.raises(ValueError):
            check_schedule(CascadeConfig(schedule="unipc", **bad))
        with pytest.raises(ValueError):      # run() rejects the config before it touches a device
            Cascade({}, device="cpu").run(CascadeConfig(schedule="unipc", **bad))
    c = Cascade({}, device="cpu")
    assert (c.unipc.config.clip_sample, c.unipc.config.clip_sample_range, c.unipc.config.solver_order,
            c.unipc.config.solver_type, c.unipc.config.final_sigmas_type) == (True, 3, 2, "bh2", "zero")
    assert torch.equal(c.unipc.alphas_cumprod, c.ddpm.alphas_cumprod)
    u = CascadeConfig(schedule="unipc", unipc_steps=10, batch_size=1, num_surfaces=2, num_edges=2)
    assert stage_timesteps(u).tolist() == [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]
    S = 4
    src = Variation(surfPos=torch.zeros(1, S, 6), surfMask=torch.tensor([[False, True, True, True]]),
                    surfZ=torch.zeros(1, S, 48), edgePos=torch.zeros(1, S, 2, 6), edgeM=torch.zeros(1, S, 2, dtype=torch.bool),
                    edge_z=torch.zeros(1, S, 2, 12), edgeV=torch.zeros(1, S, 2, 6), strength=0.5)
    assert check_variation(u, src) == (0.5,) * 4
    with pytest.raises(NotImplementedError, match="unipc"):       # DDIM inversion stays with the "ddim" schedule
        check_variation(u, Variation(**{**src.__dict__, "start": "invert"}))
    with pytest.raises(NotImplementedError, match="unipc"):
        check_interpolation(u, Interpolation(src, src, [0.5]))


def test_replacement_levels():
    """replace_table: the level 1 / (1 + sigma_next^2) each step leaves x at, exactly (1, 0) after the last step of the
    cascade's "zero" end"""
    from brepgen_b200.schedulers import UniPCMultistepScheduler
    s = UniPCMultistepScheduler(final_sigmas_type="zero", clip_sample=True, clip_sample_range=3)
    s.set_timesteps(10)
    tab = s.replace_table(s.timesteps)
    assert tab.shape == (10, 2) and tab[-1].tolist() == [1.0, 0.0]
    sig = s.sigmas.double()
    a = 1 / (1 + sig[1:] ** 2)
    assert torch.allclose(tab.double(), torch.stack([a.sqrt(), (1 - a).sqrt()], 1), atol=1e-6)


class _FakeLib:
    """records bg_unipc_step calls instead of launching (host-logic tests run without a device)"""

    def __init__(self):
        self.calls = []

    def bg_unipc_step(self, *a):
        row = list((ctypes.c_float * 24).from_address(a[10]))   # a host row: read it now, as the library does
        self.calls.append(a[:10] + (row,) + a[11:])
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


def test_steps_follow_the_plan_and_a_shape_change_restarts(fake_lib):
    """the drop-in's rows are the table's; the late face-count increase: the step on the doubled sample is first order
    without a corrector, with new buffers"""
    from brepgen_b200.schedulers import UniPCMultistepScheduler
    s = UniPCMultistepScheduler(solver_order=3, final_sigmas_type="zero", clip_sample=True, clip_sample_range=3)
    s.set_timesteps(10)
    tab = s.coefficient_table()
    x = torch.zeros(2, 3, 6)
    for t in s.timesteps:
        s.step(x, t, x)
    rows = [c[10] for c in fake_lib.calls]
    assert torch.equal(torch.tensor(rows), tab)
    assert all(c[7] == 3 and c[8] == 18 and c[9] == 36 and c[11] == 3.0 for c in fake_lib.calls)
    assert s.step_index == 10 and s.lower_order_nums == 3 and s.this_order == 1 and s.last_sample is s.last
    assert len(s.model_outputs) == 3 and all(m is not None for m in s.model_outputs)
    fake_lib.calls.clear()
    s.set_timesteps(10)
    assert s.last_sample is None and s.model_outputs == [None] * 3
    for t in s.timesteps[:5]:
        s.step(x, t, x)
    h = s.hist
    x2 = x.repeat(1, 2, 1)
    for t in s.timesteps[5:]:
        s.step(x2, t, x2)
    assert [(int(c[10][2]), int(c[10][3])) for c in fake_lib.calls] == \
        [(0, 1), (1, 2), (2, 3), (3, 3), (3, 3), (0, 1), (1, 2), (2, 3), (3, 2), (2, 1)]
    assert torch.equal(torch.tensor([c[10] for c in fake_lib.calls]), s.coefficient_table(restart=5))
    assert s.hist is not h and tuple(s.hist.shape) == (3, 2, 6, 6) and tuple(s.last.shape) == (2, 6, 6)
