"""CPU tests of DDIM inversion and interpolation: the inverse scheduler's timesteps and coefficients, the inverse oracle
pinned by equivalence to DDIMOracle, the fp64 slerp, the oracle drivers and the host checks of Variation(start="invert")
and Interpolation (which raise before anything is launched)."""
import numpy as np
import pytest
import torch

from oracle.ddim import DDIMOracle
from oracle.inversion import DDIMInverseOracle, run_cascade_interpolation, run_cascade_inverted_variation, slerp


# ------------------------------------------------------------------------------------------------------- timesteps
def test_inverse_timesteps_written_out():
    from brepgen_b200.schedulers import DDIMInverseScheduler
    s = DDIMInverseScheduler()
    s.set_timesteps(10)
    assert s.timesteps.tolist() == [0, 100, 200, 300, 400, 500, 600, 700, 800, 900]
    s = DDIMInverseScheduler(steps_offset=1)
    s.set_timesteps(50)
    assert s.timesteps.tolist() == [1 + 20 * k for k in range(50)]
    o = DDIMInverseOracle(steps_offset=1)
    o.set_timesteps(50)
    assert torch.equal(o.timesteps, s.timesteps)


@pytest.mark.parametrize("one", [True, False])
def test_first_step_starts_from_alpha_one_or_alphas_cumprod_0(one):
    from brepgen_b200.schedulers import DDIMInverseScheduler
    s = DDIMInverseScheduler(set_alpha_to_one=one)
    s.set_timesteps(10)
    sb, sa, sa_next, c_dir, sigma = s.step_coefficients(0)
    a0 = 1.0 if one else float(s.alphas_cumprod[0])
    assert sa == pytest.approx(a0 ** 0.5, abs=1e-7) and sb == pytest.approx((1 - a0) ** 0.5, abs=1e-7)
    assert sa_next == float(s.alphas_cumprod[0] ** 0.5) and c_dir == float((1 - s.alphas_cumprod[0]) ** 0.5)
    assert sigma == 0.0
    # a later step: from level t - ratio to t
    sb, sa, sa_next, c_dir, _ = s.step_coefficients(300)
    assert sa == float(s.alphas_cumprod[200] ** 0.5) and sa_next == float(s.alphas_cumprod[300] ** 0.5)
    o = DDIMInverseOracle(set_alpha_to_one=one)
    o.set_timesteps(10)
    for t in (0, 300, 900):
        assert [float(v) for v in o.coeffs(t)] == list(s.step_coefficients(t)[:4])


def test_table_rows_are_the_step_coefficients_with_sigma_zero():
    from brepgen_b200.schedulers import DDIMInverseScheduler
    s = DDIMInverseScheduler(clip_sample_range=3)
    s.set_timesteps(20)
    tab = s.coefficient_table(s.timesteps)
    assert tab.shape == (20, 5) and (tab[:, 4] == 0).all()
    for k, t in enumerate(s.timesteps.tolist()):
        assert tab[k].tolist() == list(torch.tensor(s.step_coefficients(t)).tolist())
    with pytest.raises(ValueError, match="eta must be 0"):
        s.coefficient_table(s.timesteps, 0.5)


def test_unsupported_configurations_raise():
    from brepgen_b200.schedulers import DDIMInverseScheduler
    for kw in (dict(prediction_type="v_prediction"), dict(timestep_spacing="trailing"), dict(thresholding=True),
               dict(rescale_betas_zero_snr=True)):
        with pytest.raises(NotImplementedError):
            DDIMInverseScheduler(**kw)
    with pytest.raises(ValueError):
        DDIMInverseScheduler().step_coefficients(100)       # set_timesteps not called


# ------------------------------------------------------------------------------------------- pinned through DDIM
@pytest.mark.parametrize("dtype,bar", [(torch.float64, 1e-12), (torch.float32, 2e-6)])
@pytest.mark.parametrize("n,offset", [(10, 0), (50, 1), (1000, 0)])
def test_inverse_then_forward_is_the_identity(dtype, bar, n, offset):
    fwd = DDIMOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True, steps_offset=offset)
    inv = DDIMInverseOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True, steps_offset=offset)
    fwd.set_timesteps(n)
    inv.set_timesteps(n)
    g = torch.Generator().manual_seed(n)
    for t in inv.timesteps.tolist()[:: max(1, n // 10)]:
        x0 = (torch.rand(4, 64, generator=g, dtype=torch.float64) * 2 - 1).to(dtype)
        eps = torch.randn(4, 64, generator=g, dtype=torch.float64).to(dtype)
        sb, sa, _, _ = inv.coeffs(t)
        x = (sa.to(dtype) * x0 + sb.to(dtype) * eps)          # a sample at the level below t
        back = fwd.step(eps, t, inv.step(eps, t, x))
        err = float(((back - x).abs().max() / x.abs().max()))
        assert back.dtype == dtype and err <= bar, (t, err)


@pytest.mark.parametrize("n", [10, 50])
def test_constant_eps_inversion_then_ddim_returns_x0(n):
    fwd = DDIMOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True)
    inv = DDIMInverseOracle(clip_sample=True, clip_sample_range=3.0, set_alpha_to_one=True)
    fwd.set_timesteps(n)
    inv.set_timesteps(n)
    g = torch.Generator().manual_seed(1)
    x0 = torch.rand(3, 6, 18, generator=g, dtype=torch.float64) * 6 - 3
    eps = torch.randn(3, 6, 18, generator=g, dtype=torch.float64) * 0.1
    x = x0.clone()
    for t in inv.timesteps:
        x = inv.step(eps, int(t), x)
    for t in fwd.timesteps:
        x = fwd.step(eps, int(t), x)
    assert float((x - x0).abs().max()) < 1e-9


# ------------------------------------------------------------------------------------------------------------ slerp
def test_slerp_endpoints_norm_and_lerp():
    g = torch.Generator().manual_seed(2)
    a, b = torch.randn(3, 5, 4, generator=g), torch.randn(3, 5, 4, generator=g)
    assert torch.equal(slerp(a, b, [0.0, 0.0, 0.0]).float(), a)
    assert torch.equal(slerp(a, b, [1.0, 1.0, 1.0]).float(), b)
    # orthogonal unit vectors: every point of the arc has norm 1 and the angle splits as alpha
    u, v = torch.zeros(1, 2, 2, dtype=torch.float64), torch.zeros(1, 2, 2, dtype=torch.float64)
    u[0, 0, 0] = v[0, 1, 1] = 1.0
    for al in (0.1, 0.25, 0.5, 0.9):
        o = slerp(u, v, [al])
        assert abs(float(o.norm()) - 1.0) < 1e-12 and abs(float(o[0, 0, 0]) - np.cos(al * np.pi / 2)) < 1e-12
    # nearly parallel: the lerp
    w = a + 1e-3 * b
    o = slerp(a, w, [0.3, 0.3, 0.3])
    assert torch.allclose(o, 0.7 * a.double() + 0.3 * w.double(), atol=0, rtol=1e-12)
    # masked tokens are a's and take no part in the angle
    mask = torch.zeros(3, 5, dtype=torch.bool)
    mask[:, 2] = True
    b2 = b.clone()
    b2[:, 2] = 100.0
    o1, o2 = slerp(a, b, [0.4] * 3, mask), slerp(a, b2, [0.4] * 3, mask)
    assert torch.equal(o1, o2) and torch.equal(o1[:, 2], a[:, 2].double())


# ---------------------------------------------------------------------------------------------------- the drivers
def _cfg(**kw):
    from brepgen_b200.sampler import CascadeConfig
    base = dict(batch_size=2, num_surfaces=3, num_edges=3, schedule="ddim", ddim_steps=5, seed=3, decode=False)
    base.update(kw)
    return CascadeConfig(**base)


def _source(cfg, seed, n_valid):
    from brepgen_b200.sampler import Variation
    g = torch.Generator().manual_seed(seed)
    B, S, E = cfg.batch_size, 2 * cfg.num_surfaces if not cfg.use_cf else cfg.num_surfaces, cfg.num_edges
    pos = torch.rand(B, S, 6, generator=g) * 2 - 1
    surfMask = torch.arange(S)[None, :] >= torch.tensor(n_valid)[:, None]
    edgeM = torch.rand(B, S, E, generator=g) < 0.4
    edgeM[..., 0] = False
    edgeM |= surfMask[..., None]
    return Variation(pos, surfMask, torch.randn(B, S, 48, generator=g), torch.rand(B, S, E, 6, generator=g) * 2 - 1,
                     edgeM, torch.randn(B, S, E, 12, generator=g), torch.randn(B, S, E, 6, generator=g), 1.0, "invert")


def _tiny_forwards():
    """cheap deterministic stand-ins for the denoisers (the drivers only need eps of the right shape)"""
    def f(x, t, *cond):
        return 0.1 * torch.tanh(x) + 0.001 * float(t[0])
    return {k: f for k in ("surfpos", "surfz", "edgepos", "edgez")}


def _init(cfg, seed):
    g = torch.Generator().manual_seed(seed)
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    S = S0 if cfg.use_cf else 2 * S0
    return {"surfPos": torch.randn(B, S0, 6, generator=g), "surfZ": torch.randn(B, S, 48, generator=g),
            "edgePos": torch.randn(B, S, E, 6, generator=g), "edgeZV": torch.randn(B, S, E, 18, generator=g)}


def test_oracle_interpolation_at_alpha_0_is_the_inverted_variation_of_a():
    cfg = _cfg()
    a, b = _source(cfg, 1, [2, 3]), _source(cfg, 2, [3, 1])
    init = _init(cfg, 4)
    va = run_cascade_inverted_variation(None, cfg, a, init, forwards=_tiny_forwards())
    iv = run_cascade_interpolation(None, cfg, a, b, [0.0, 0.0], init, forwards=_tiny_forwards())
    for k in va:
        assert torch.equal(va[k], iv[k]), k
    half = run_cascade_interpolation(None, cfg, a, b, [0.5, 0.5], init, forwards=_tiny_forwards())
    assert not torch.equal(half["surfZ"], va["surfZ"])


# ---------------------------------------------------------------------------------------------------- host checks
def _raises(exc, match, cfg, source):
    from brepgen_b200.sampler import Cascade
    with pytest.raises(exc, match=match):
        Cascade({}, device="cpu").run(cfg, source=source)


def test_host_checks_raise_before_any_launch():
    from dataclasses import replace
    from brepgen_b200.sampler import Interpolation
    cfg = _cfg()
    a, b = _source(cfg, 1, [2, 3]), _source(cfg, 2, [3, 1])
    _raises(ValueError, "Variation.start", cfg, replace(a, start="inverse"))
    _raises(NotImplementedError, "schedule 'ddim' with ddim_eta = 0", _cfg(schedule="ddpm", ddpm_steps=5), a)
    _raises(NotImplementedError, "ddim_eta = 0", _cfg(ddim_eta=0.5), a)
    _raises(NotImplementedError, "ddim_eta = 0", _cfg(ddim_eta=0.5), Interpolation(a, b, [0.5, 0.5]))
    empty = replace(a, surfMask=torch.ones_like(a.surfMask), edgeM=torch.ones_like(a.edgeM))
    _raises(ValueError, "no valid face", cfg, empty)
    _raises(ValueError, r"Interpolation.b: .*no valid face", cfg, Interpolation(a, empty, [0.5, 0.5]))
    _raises(ValueError, "surfZ must be a tensor of shape", cfg, Interpolation(a, replace(b, surfZ=b.surfZ[:, :2]),
                                                                              [0.5, 0.5]))
    _raises(ValueError, "alpha has 3 values", cfg, Interpolation(a, b, [0.5, 0.5, 0.5]))
    _raises(ValueError, r"alpha must lie in \[0, 1\]", cfg, Interpolation(a, b, [0.5, 1.5]))
    _raises(ValueError, r"alpha must lie in \[0, 1\]", cfg, Interpolation(a, b, [float("nan"), 0.5]))
    _raises(ValueError, "equal strengths", cfg, Interpolation(a, replace(b, strength=0.6), [0.5, 0.5]))
    zero = (0.0, 0.6, 0.6, 0.6)
    _raises(ValueError, "must all be > 0", cfg, Interpolation(replace(a, strength=zero), replace(b, strength=zero),
                                                              [0.5, 0.5]))
    _raises(ValueError, "must be a Variation", cfg, Interpolation(a, {"surfPos": 1}, [0.5, 0.5]))
    # the face-slot limit, checked for both designs: 4 valid faces do not fit the 3 slots a non-CFG run starts with
    many = _source(cfg, 3, [2, 4])
    _raises(ValueError, r"Interpolation.b: .*face slots", cfg, Interpolation(a, many, [0.5, 0.5]))
    _raises(ValueError, r"Interpolation.a: .*face slots", cfg, Interpolation(many, b, [0.5, 0.5]))
