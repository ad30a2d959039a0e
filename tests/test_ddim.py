"""CPU tests of the DDIM scheduler: the oracle against the known answers of diffusers' own DDIM tests, and the host logic of
the DDIMScheduler drop-in and CascadeConfig(schedule="ddim").

diffusers' tests/schedulers/test_scheduler_ddim.py runs full loops of set_timesteps(10), eta = 0, over the deterministic
dummy model of tests/test_oracle_sched_kat.py and checks the |x| sum / mean to 1e-2 / 1e-3 (sum / 768 = mean for each
pair)."""
import contextlib

import numpy as np
import pytest
import torch

from oracle.ddim import DDIMOracle
from test_oracle_sched_kat import dummy_model, dummy_sample_deter

DDIM_KATS = [({}, 172.0067, 0.223967),                                             # test_full_loop_no_noise
             (dict(beta_start=0.01, set_alpha_to_one=True), 149.8295, 0.1951),     # ..._with_set_alpha_to_one
             (dict(beta_start=0.01, set_alpha_to_one=False), 149.0784, 0.1941)]    # ..._with_no_set_alpha_to_one


@pytest.mark.parametrize("kw,kat_sum,kat_mean", DDIM_KATS)
def test_ddim_oracle_full_loop_matches_diffusers_known_answer(kw, kat_sum, kat_mean):
    sch = DDIMOracle(**kw)
    sch.set_timesteps(10)
    x = dummy_sample_deter()
    for t in sch.timesteps:
        x = sch.step(dummy_model(x, int(t)), int(t), x, eta=0.0)
    assert abs(float(x.abs().sum()) - kat_sum) < 1e-2
    assert abs(float(x.abs().mean()) - kat_mean) < 1e-3


def test_timestep_tables():
    from brepgen_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    assert s.num_inference_steps is None and s.timesteps.tolist() == list(range(999, -1, -1))
    s.set_timesteps(10)
    assert s.timesteps.tolist() == [900, 800, 700, 600, 500, 400, 300, 200, 100, 0]
    assert s.timesteps.dtype == torch.int64
    s.set_timesteps(3)
    assert s.timesteps.tolist() == [666, 333, 0]
    s.set_timesteps(1000)
    assert s.timesteps.tolist() == list(range(999, -1, -1))
    off = DDIMScheduler(steps_offset=1)
    off.set_timesteps(5)
    assert off.timesteps.tolist() == [801, 601, 401, 201, 1]
    for n in (1, 7, 50, 333):
        s.set_timesteps(n)
        o = DDIMOracle()
        o.set_timesteps(n)
        assert torch.equal(s.timesteps, o.timesteps), n
    assert len(s) == 1000 and s.init_noise_sigma == 1.0
    x = torch.randn(2, 3)
    assert s.scale_model_input(x, 5) is x


def test_unsupported_settings_and_errors():
    from brepgen_b200.schedulers import DDIMScheduler
    for kw in (dict(prediction_type="v_prediction"), dict(prediction_type="sample"), dict(thresholding=True),
               dict(rescale_betas_zero_snr=True), dict(timestep_spacing="trailing"), dict(timestep_spacing="linspace"),
               dict(beta_schedule="squaredcos_cap_v2")):
        with pytest.raises(NotImplementedError):
            DDIMScheduler(**kw)
    s = DDIMScheduler()
    with pytest.raises(ValueError):
        s.set_timesteps(1001)
    x = torch.zeros(2, 4)
    with pytest.raises(ValueError, match="set_timesteps"):        # diffusers: step before set_timesteps
        s.step(x, 10, x)
    s.set_timesteps(10)
    with pytest.raises(ValueError, match="generator"):
        s.step(x, 900, x, eta=0.5, generator=torch.Generator(), variance_noise=torch.zeros(2, 4))


@pytest.mark.parametrize("set_alpha_to_one", [True, False])
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_step_coefficients_match_oracle(set_alpha_to_one, eta):
    from brepgen_b200.schedulers import DDIMScheduler
    s = DDIMScheduler(clip_sample_range=3, set_alpha_to_one=set_alpha_to_one)
    o = DDIMOracle(clip_sample_range=3, set_alpha_to_one=set_alpha_to_one)
    for n in (1, 10, 50, 1000):
        s.set_timesteps(n)
        o.set_timesteps(n)
        tab = s.coefficient_table(s.timesteps, eta)
        assert tab.shape == (n, 5) and tab.dtype == torch.float32
        for i, t in enumerate(s.timesteps.tolist()):
            ref = [float(c) for c in o.coeffs(t, eta)]
            assert list(s.step_coefficients(t, eta)) == ref, (n, t)
            assert tab[i].tolist() == ref, (n, t)
        sb, sa, sa_prev, c_dir, sigma = s.step_coefficients(int(s.timesteps[-1]), eta)
        assert sa_prev == (1.0 if set_alpha_to_one else float(s.alphas_cumprod[0] ** 0.5))
        if set_alpha_to_one:           # the last step lands on abar = 1: no noise and no direction term
            assert sigma == 0.0 and c_dir == 0.0
    s.set_timesteps(50)
    sb, sa, sa_prev, c_dir, sigma = s.step_coefficients(500, eta)
    a_t, a_p = float(s.alphas_cumprod[500]), float(s.alphas_cumprod[480])
    assert sigma == pytest.approx(eta * np.sqrt((1 - a_p) / (1 - a_t) * (1 - a_t / a_p)), rel=1e-5)
    assert c_dir == pytest.approx(np.sqrt(1 - a_p - sigma ** 2), rel=1e-5)


def test_cascade_config_validation():
    from brepgen_b200.sampler import Cascade, CascadeConfig, check_schedule
    cfg = CascadeConfig()
    assert (cfg.schedule, cfg.ddim_steps, cfg.ddim_eta, cfg.ddpm_steps) == ("reference", 50, 0.0, 1000)
    for ok in (dict(ddim_steps=1), dict(ddim_steps=1000), dict(ddim_eta=0.0), dict(ddim_eta=1.0), dict(ddim_eta=2.5)):
        check_schedule(CascadeConfig(schedule="ddim", **ok))
    check_schedule(CascadeConfig(schedule="ddpm", ddim_steps=0, ddim_eta=-1.0))     # DDIM fields unused by other schedules
    for bad in (dict(ddim_steps=0), dict(ddim_steps=1001), dict(ddim_steps=-3), dict(ddim_eta=-0.1),
                dict(ddim_eta=float("nan"))):
        with pytest.raises(ValueError):
            check_schedule(CascadeConfig(schedule="ddim", **bad))
        with pytest.raises(ValueError):      # run() rejects the config before it touches a device
            Cascade({}, device="cpu").run(CascadeConfig(schedule="ddim", **bad))
    c = Cascade({}, device="cpu")
    assert (c.ddim.config.clip_sample, c.ddim.config.clip_sample_range, c.ddim.config.set_alpha_to_one) == (True, 3, True)
    assert torch.equal(c.ddim.alphas_cumprod, c.ddpm.alphas_cumprod)


class _FakeLib:
    """records bg_ddim_step calls instead of launching (host-logic tests run without a device)"""

    def __init__(self):
        self.calls = []

    def bg_ddim_step(self, *a):
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


# positions in the bg_ddim_step argument list
A_NOISE, A_SEED, A_OFFSET, A_KEYS, A_PER, A_T, A_N, A_SIGMA, A_CLIP, A_USE_CLIPPED = 5, 6, 7, 8, 9, 10, 11, 16, 17, 18


def test_generator_is_advanced_once_per_step_when_eta_positive(fake_lib):
    """diffusers draws randn_tensor on every step when eta > 0, the last one (sigma = 0) included: a seeded CPU generator
    ends where diffusers leaves it"""
    from brepgen_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(10)
    x = torch.zeros(2, 3, 5)
    g = torch.Generator().manual_seed(4)
    for t in s.timesteps:
        s.step(x, t, x, eta=0.5, generator=g)
    ref = torch.Generator().manual_seed(4)
    for _ in range(10):
        torch.randn(x.shape, generator=ref)
    assert torch.equal(g.get_state(), ref.get_state())
    assert all(c[A_NOISE] is not None for c in fake_lib.calls) and len(fake_lib.calls) == 10
    assert fake_lib.calls[-1][A_SIGMA] == 0.0 and fake_lib.calls[0][A_SIGMA] > 0.0
    # eta = 0: deterministic, the generator is not touched and no noise is passed
    g0 = torch.Generator().manual_seed(4)
    st = g0.get_state()
    fake_lib.calls.clear()
    s.step(x, 900, x, eta=0.0, generator=g0)
    assert torch.equal(g0.get_state(), st) and fake_lib.calls[0][A_NOISE] is None and fake_lib.calls[0][A_SIGMA] == 0.0
    # a list of generators, one per sample (diffusers' randn_tensor list branch)
    gens = [torch.Generator().manual_seed(9 + i) for i in range(2)]
    s.step(x, 900, x, eta=1.0, generator=gens)
    for i, gi in enumerate(gens):
        r = torch.Generator().manual_seed(9 + i)
        torch.randn((1, 3, 5), generator=r)
        assert torch.equal(gi.get_state(), r.get_state())


def test_noise_stream_arguments(fake_lib):
    """batch stream: the offset advances by one element group count on every eta > 0 step, last step included, and not
    at all when eta = 0; per-sample keys: passed with per_sample and t, no offset bookkeeping"""
    from brepgen_b200.schedulers import DDIMScheduler
    s = DDIMScheduler(clip_sample_range=3)
    s.set_timesteps(4)
    x = torch.zeros(3, 7)            # n = 21: 6 groups of 4
    s.set_noise_seed(5, 0, 2)
    for t in s.timesteps:
        s.step(x, t, x, eta=0.3, use_clipped_model_output=True)
    assert [c[A_OFFSET] for c in fake_lib.calls] == [0, 6, 12, 18]
    assert len({c[A_SEED] for c in fake_lib.calls}) == 1 and fake_lib.calls[0][A_SEED] != 0
    assert all(c[A_KEYS] is None and c[A_NOISE] is None and c[A_USE_CLIPPED] == 1 and c[A_CLIP] == 3.0
               for c in fake_lib.calls)
    assert [c[A_T] for c in fake_lib.calls] == [750, 500, 250, 0] and fake_lib.calls[0][A_N] == 21
    fake_lib.calls.clear()
    s.step(x, 750, x, eta=0.0)
    assert s._philox_offset == 24 and fake_lib.calls[0][A_SIGMA] == 0.0
    fake_lib.calls.clear()
    s.set_sample_keys(seed=3, first=10, stage=1)
    s.step(x, 500, x, eta=1.0)
    c = fake_lib.calls[0]
    assert c[A_KEYS] is not None and c[A_PER] == 7 and c[A_T] == 500 and c[A_NOISE] is None
    explicit = torch.ones(3, 7)
    s.step(x, 500, x, eta=1.0, variance_noise=explicit)
    assert fake_lib.calls[1][A_NOISE] is not None


def test_oracle_ddim_cascade_driver():
    """oracle.ddim.run_cascade_ddim with stand-in networks: one forward per step and stage, step noise requested on every
    step when eta > 0 and never at eta = 0, the face slots doubled from the first t <= 249 on, CFG batches doubled"""
    from brepgen_b200.sampler import CascadeConfig
    from oracle.ddim import run_cascade_ddim
    for use_cf, eta in ((False, 0.5), (True, 0.0)):
        cfg = CascadeConfig(batch_size=2, num_surfaces=3, num_edges=2, use_cf=use_cf, class_label=6, schedule="ddim",
                            ddim_steps=10, ddim_eta=eta, dense_masks=True)
        S = 3 if use_cf else 6
        g = torch.Generator().manual_seed(1)
        init = {"surfPos": torch.randn(2, 3, 6, generator=g), "surfZ": torch.randn(2, S, 48, generator=g),
                "edgePos": torch.randn(2, S, 2, 6, generator=g), "edgeZV": torch.randn(2, S, 2, 18, generator=g)}
        seen, drawn = {}, []

        def fwd(kind):
            def f(x, t, *rest):
                seen.setdefault(kind, []).append((int(t), tuple(x.shape)))
                return torch.tanh(x) * 0.5
            return f

        def step_noise(name, k, shape):
            drawn.append((name, k))
            return torch.randn(tuple(shape), generator=g)
        out = run_cascade_ddim(None, cfg, init, step_noise, {k: fwd(k) for k in ("surfpos", "surfz", "edgepos", "edgez")})
        ts = list(range(900, -1, -100))
        mult = 2 if use_cf else 1
        assert [t for t, _ in seen["surfpos"]] == ts and all(len(v) == 10 for v in seen.values())
        assert [s[1] for _, s in seen["surfpos"]] == [3 if (use_cf or t > 249) else 6 for t in ts]
        assert all(s[0] == 2 * mult for v in seen.values() for _, s in v)
        assert len(drawn) == (40 if eta > 0 else 0)
        assert out["surfPos"].shape == (2, S, 6) and out["edgeV"].shape == (2, S, 2, 6)
        assert all(torch.isfinite(v.float()).all() for v in out.values())
