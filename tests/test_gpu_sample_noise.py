"""GPU tests of the per-sample noise mode (bg_randn_keyed, bg_ddpm_step and bg_ddpm_step_tab with sample keys, and
CascadeConfig(noise="per_sample")).

  * the generator against a numpy Philox4x32-10 of the same counters with float64 Box-Muller, and its statistics;
  * the keyed step forms against each other and against bg_ddpm_step fed the keyed noise, bit for bit;
  * noise that does not depend on the batch: sample b of a batch equals the same sample drawn alone, bit for bit;
  * small cascades: B = 5 equals five B = 1 runs, CFG, graph on / off, two simulated ranks, explicit sample seeds;
  * the benchmark's shape (B = 64, S0 = 50, E = 40) against B = 1 runs of three of its samples;
  * argument errors, and DDPMScheduler.step with a list of CPU generators (diffusers' per-sample generators).
"""
import numpy as np
import pytest
import torch

from brepgen_b200.schedulers import sample_keys, sample_seed

pytestmark = pytest.mark.gpu

M32 = np.uint64(0xFFFFFFFF)


def philox_np(ctr, key):
    """numpy Philox4x32-10: ctr uint64 [n, 4] (32-bit words), key uint64 [n, 2] -> uint64 [n, 4]"""
    c = [ctr[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = key[:, 0].astype(np.uint64), key[:, 1].astype(np.uint64)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & M32, p1 >> np.uint64(32), p1 & M32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return np.stack(c, 1)


def keyed_normals_np(keys, per_sample, domain, t):
    """float64 [len(keys), per_sample]: element j of sample b from counter (j // 4, t, domain), key keys[b]"""
    B = len(keys)
    gps = (per_sample + 3) // 4
    q = np.tile(np.arange(gps, dtype=np.uint64), B)
    kb = np.repeat(np.asarray(keys, dtype=np.uint64), gps)
    ctr = np.stack([q & M32, q >> np.uint64(32), np.full_like(q, t), np.full_like(q, domain)], 1)
    r = philox_np(ctr, np.stack([kb & M32, kb >> np.uint64(32)], 1)).astype(np.float64)
    u1 = (r[:, 0::2] + 1.0) * 2.0 ** -32
    u2 = r[:, 1::2] * 2.0 ** -32
    rr = np.sqrt(-2.0 * np.log(u1))
    z = np.stack([rr[:, 0] * np.cos(2 * np.pi * u2[:, 0]), rr[:, 0] * np.sin(2 * np.pi * u2[:, 0]),
                  rr[:, 1] * np.cos(2 * np.pi * u2[:, 1]), rr[:, 1] * np.sin(2 * np.pi * u2[:, 1])], 1)
    return z.reshape(B, gps * 4)[:, :per_sample]


def keys_dev(seeds, stage):
    return torch.from_numpy(sample_keys(seeds, stage).view(np.int64)).cuda()


def randn_keyed(keys, B, per, domain, t):
    from brepgen_b200 import _ffi as f
    out = torch.full((B, per), float("nan"), device="cuda")
    f.check(f.lib().bg_randn_keyed(keys.data_ptr(), B, per, domain, t, out.data_ptr(), f.current_stream()), "randn_keyed")
    return out


SEEDS = [sample_seed(3, b) for b in range(7)]


# ------------------------------------------------------------------------------------------------------------ generator
@pytest.mark.parametrize("per,domain,t", [(1, 1, 0), (7, 0, 999), (13, 1, 0), (42, 0, 1), (4096, 0, 250)])
def test_randn_keyed_matches_numpy_philox(per, domain, t):
    seeds = SEEDS[:5] + [0, 2 ** 64 - 1]
    keys = sample_keys(seeds, 2)
    got = randn_keyed(keys_dev(seeds, 2), len(seeds), per, domain, t).double().cpu().numpy()
    ref = keyed_normals_np(keys, per, domain, t)
    err = np.abs(got - ref).max()
    print(f"randn_keyed per={per} domain={domain} t={t}: max |err| vs float64 Box-Muller = {err:.3e}")
    assert np.isfinite(got).all()
    # the kernel's fp32 u1 / u2 and __logf / __sincosf: worst measured 7.4e-6 (per = 4096) on an H100; bar = 4x that
    assert err < 3e-5, err


def test_randn_keyed_statistics():
    """2^24 draws: mean, variance, KS; neighbouring samples, consecutive t and the two domains uncorrelated (< 4 sigma)"""
    from scipy import stats
    B, per = 64, 2 ** 18
    N = B * per
    seeds = [sample_seed(11, b) for b in range(B + 1)]
    k = keys_dev(seeds, 0)
    z = randn_keyed(k, B + 1, per, 0, 500).double()
    a = z[:B].flatten()
    sig = 1.0 / np.sqrt(N)
    mean, var = float(a.mean()), float(a.var())
    print(f"mean {mean:.2e} (sigma {sig:.1e})  var-1 {var - 1:.2e} (sigma {np.sqrt(2 / N):.1e})")
    assert abs(mean) < 4 * sig and abs(var - 1) < 4 * np.sqrt(2.0 / N)
    ks = stats.kstest(a.cpu().numpy(), "norm")
    print(f"KS D={ks.statistic:.2e} p={ks.pvalue:.3f}")
    assert ks.pvalue > 1e-3

    def corr(x, y):
        x, y = x - x.mean(), y - y.mean()
        return float((x * y).sum() / (x.norm() * y.norm()))
    nb = corr(z[:B].flatten(), z[1:].flatten())                       # sample b vs sample b + 1, same positions
    zt = randn_keyed(k, B + 1, per, 0, 501).double()
    ct = corr(a, zt[:B].flatten())                                    # t vs t + 1
    z1 = randn_keyed(k, B + 1, per, 1, 500).double()
    cd = corr(a, z1[:B].flatten())                                    # step vs initial-noise domain
    print(f"correlations: neighbours {nb:.2e}, consecutive t {ct:.2e}, domains {cd:.2e} (4 sigma = {4 * sig:.1e})")
    assert max(abs(nb), abs(ct), abs(cd)) < 4 * sig


# ---------------------------------------------------------------------------------------------------- kernels agree
def _step_inputs(B, per, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(B, per, generator=g, device="cuda") * 2 for _ in range(3)]


@pytest.mark.parametrize("cfg_w", [0.0, 0.6])
@pytest.mark.parametrize("per", [7, 13, 1638])
def test_ddpm_step_with_keys_equals_step_fed_keyed_noise_and_table_form(per, cfg_w):
    from brepgen_b200 import _ffi as f
    from brepgen_b200.schedulers import DDPMScheduler
    lib, st = f.lib(), f.current_stream()
    B = 7
    eps_c, eps_u, x = _step_inputs(B, per)
    eps_u = eps_u if cfg_w else None
    k = keys_dev(SEEDS, 1)
    sch = DDPMScheduler(clip_sample=True, clip_sample_range=3)
    ts = torch.tensor([999, 600, 250, 1, 0], dtype=torch.int64)
    coef = sch.coefficient_table(ts).cuda()
    ts_d, step, t_cur = ts.cuda(), torch.full((1,), -1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int64,
                                                                                                          device="cuda")
    for i, t in enumerate(ts.tolist()):
        sb, sa, c_x0, c_x, sigma = sch.step_coefficients(t)
        keyed = torch.full_like(x, float("nan"))
        f.check(lib.bg_ddpm_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), keyed.data_ptr(), None, 0, 0,
                                 k.data_ptr(), per, t, B * per, sb, sa, 3.0, c_x0, c_x, sigma, st), "keyed")
        nz = randn_keyed(k, B, per, 0, t)
        fed = torch.full_like(x, float("nan"))
        f.check(lib.bg_ddpm_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), fed.data_ptr(), nz.data_ptr(), 0, 0,
                                 None, 0, 0, B * per, sb, sa, 3.0, c_x0, c_x, sigma, st), "ddpm_step")
        f.check(lib.bg_step_advance(ts_d.data_ptr(), len(ts), step.data_ptr(), t_cur.data_ptr(), st), "advance")
        tab = torch.full_like(x, float("nan"))
        f.check(lib.bg_ddpm_step_tab(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), tab.data_ptr(), 0, 0, 0,
                                     k.data_ptr(), per, t_cur.data_ptr(), B * per, coef.data_ptr(), step.data_ptr(), 3.0,
                                     st), "tab")
        torch.cuda.synchronize()
        assert torch.isfinite(keyed).all()
        assert torch.equal(keyed, fed), t
        assert torch.equal(tab, keyed), t
        if sigma != 0.0:     # the noise is really there
            quiet = torch.empty_like(x)
            f.check(lib.bg_ddpm_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), quiet.data_ptr(), None, 0, 0,
                                     None, 0, 0, B * per, sb, sa, 3.0, c_x0, c_x, 0.0, st), "ddpm_step")
            torch.cuda.synchronize()
            assert not torch.equal(quiet, keyed)


# ------------------------------------------------------------------------------------------ noise independent of batch
@pytest.mark.parametrize("shape", [(7, 6), (7, 13, 18), (7,), (13,)])
def test_noise_does_not_depend_on_the_batch(shape):
    """sample b of a B = 7 batch == a B = 1 call with sample_base = b: initial noise and step noise (through the scheduler)"""
    from brepgen_b200.sampler import randn_keyed as init_noise
    from brepgen_b200.schedulers import DDPMScheduler
    B = 7
    full = init_noise([sample_seed(5, b) for b in range(B)], 3, (B,) + shape, "cuda")
    zero = torch.zeros((B,) + shape, device="cuda")
    sch = DDPMScheduler(clip_sample=True, clip_sample_range=3)
    sch.set_sample_keys(seed=5, first=0, stage=3)
    step_full = torch.stack([sch.step(zero, t, zero).prev_sample for t in (700, 699)])
    for b in range(B):
        one = init_noise([sample_seed(5, b)], 3, (1,) + shape, "cuda")
        assert torch.equal(one[0], full[b]), b
        s1 = DDPMScheduler(clip_sample=True, clip_sample_range=3)
        s1.set_sample_keys(seed=5, first=b, stage=3)
        step_one = torch.stack([s1.step(zero[:1], t, zero[:1]).prev_sample for t in (700, 699)])
        assert torch.equal(step_one[:, 0], step_full[:, b]), b
    assert not torch.equal(full[0], full[1]) and not torch.equal(step_full[0], step_full[1])
    assert float(step_full.abs().max()) > 0


# ------------------------------------------------------------------------------------------------------- cascades
_MODELS = {}


def _setup(use_cf):
    if use_cf not in _MODELS:
        from brepgen_b200.models import NETS
        from brepgen_b200.spec import denoiser_spec
        from brepgen_b200.synth import synth_state_dict
        from brepgen_b200.vae import build_synthetic_decoders
        ms = {}
        for kind in NETS:
            m = NETS[kind](use_cf)
            m.load_state_dict(synth_state_dict(denoiser_spec(kind, use_cf), seed=11))
            ms[kind] = m.cuda().eval()
        _MODELS[use_cf] = (ms,) + tuple(build_synthetic_decoders(torch.device("cuda")))
    return _MODELS[use_cf]


def _run(cfg):
    from brepgen_b200.sampler import Cascade
    ms, sv, ev = _setup(cfg.use_cf)
    out = Cascade(ms, sv, ev).run(cfg)
    torch.cuda.synchronize()
    return out


def _assert_sample_equal(full, b, one, what=""):
    assert set(full) == set(one)
    for k in full:
        assert torch.equal(full[k][b], one[k][0]), (what, b, k)


def _cfg(**kw):
    from brepgen_b200.sampler import CascadeConfig
    base = dict(num_surfaces=5, num_edges=6, schedule="ddpm", ddpm_steps=4, seed=21, noise="per_sample", class_label=6,
                graph="off")
    base.update(kw)
    return CascadeConfig(**base)


@pytest.mark.parametrize("schedule,use_cf,graph", [("ddpm", False, "off"), ("ddpm", True, "off"), ("ddpm", False, "on"),
                                                   ("reference", False, "auto")])
def test_cascade_sample_equals_sample_run_alone(schedule, use_cf, graph):
    full = _run(_cfg(batch_size=5, schedule=schedule, use_cf=use_cf, graph=graph))
    assert all(torch.isfinite(v.float()).all() for v in full.values())
    assert "surf_ncs" in full and "edge_ncs" in full
    for b in range(5):
        _assert_sample_equal(full, b, _run(_cfg(batch_size=1, sample_base=b, schedule=schedule, use_cf=use_cf, graph=graph)),
                             (schedule, use_cf, graph))
    assert not torch.equal(full["surfPos"][0], full["surfPos"][1])


def test_cascade_graph_on_equals_graph_off():
    for use_cf in (False, True):
        a = _run(_cfg(batch_size=3, use_cf=use_cf, graph="off", ddpm_steps=40))
        b = _run(_cfg(batch_size=3, use_cf=use_cf, graph="on", ddpm_steps=40))
        for k in a:
            assert torch.equal(a[k], b[k]), (use_cf, k)


def test_two_ranks_equal_one_gpu():
    from brepgen_b200.sampler import shard_config
    one = _run(_cfg(batch_size=6))
    parts = [_run(shard_config(_cfg(batch_size=6), 6, r, 2)) for r in range(2)]
    for k in one:
        assert torch.equal(torch.cat([p[k] for p in parts], 0), one[k]), k


def test_explicit_sample_seeds_reproduce_a_sample_anywhere():
    s = [sample_seed(21, 4), 12345, 777]
    a = _run(_cfg(batch_size=3, sample_seeds=s))
    b = _run(_cfg(batch_size=3, sample_seeds=s[::-1]))
    for i in range(3):
        _assert_sample_equal(a, i, {k: v[2 - i:3 - i] for k, v in b.items()}, "reversed")
    default = _run(_cfg(batch_size=1, sample_base=4))         # sample_seed(seed, index) is the default seed of index 4
    _assert_sample_equal(a, 0, default, "default")


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("masks", ["dense", "dedup"])
def test_benchmark_shape_samples_equal_samples_run_alone(masks):
    """B = 64, S0 = 50, E = 40 (the benchmark's cascade, 2 DDPM steps per stage): samples 0, 31, 63 against B = 1 runs,
    bit for bit.  At B = 64 the edge stages' GEMMs run 256-wide tiles and at B = 1 128-wide ones; tools/batch_invariance.py
    shows wgmma rows come out bit-identical on both paths and at any row offset (DESIGN.md section 6)."""
    kw = dict(num_surfaces=50, num_edges=40, ddpm_steps=2, dense_masks=masks == "dense", seed=1000)
    full = _run(_cfg(batch_size=64, **kw))
    for k, v in full.items():
        assert torch.isfinite(v.float().flatten(1)).all(1).all(), k
    from brepgen_b200.sampler import randn_keyed as init_noise
    for b in (0, 31, 63):
        one = _run(_cfg(batch_size=1, sample_base=b, **kw))
        for k in full:
            if full[k].dtype == torch.bool:
                assert torch.equal(full[k][b], one[k][0]), (b, k)
                continue
            err = _rel(full[k][b], one[k][0])
            print(f"B=64 sample {b} {masks} {k}: rel_l2 vs B=1 = {err:.2e}")
            assert torch.equal(full[k][b], one[k][0]), (b, k, err)
        seeds = [sample_seed(1000, b)]
        big = init_noise([sample_seed(1000, i) for i in range(64)], 3, (64, 100, 40, 18), "cuda")
        assert torch.equal(big[b], init_noise(seeds, 3, (1, 100, 40, 18), "cuda")[0])


# --------------------------------------------------------------------------------------------------------- errors
def test_bad_keyed_step_arguments_are_rejected_and_launch_nothing():
    from brepgen_b200 import _ffi as f
    lib, st = f.lib(), f.current_stream()
    B, per = 3, 8
    eps, _, x = _step_inputs(B, per)
    k = keys_dev(SEEDS[:B], 0)
    out = torch.full((B, per), float("nan"), device="cuda")
    coef = torch.ones(1, 5, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    n = B * per

    def step_call(per_sample, t=5, sa=0.8):
        return lib.bg_ddpm_step(eps.data_ptr(), None, 0.0, x.data_ptr(), out.data_ptr(), None, 0, 0, k.data_ptr(),
                                per_sample, t, n, 0.5, sa, 3.0, 0.3, 0.6, 0.1, st)

    def tab_call(per_sample, t_cur_ptr):
        return lib.bg_ddpm_step_tab(eps.data_ptr(), None, 0.0, x.data_ptr(), out.data_ptr(), 0, 0, 0, k.data_ptr(),
                                    per_sample, t_cur_ptr, n, coef.data_ptr(), step.data_ptr(), 3.0, st)
    cases = [
        ("randn NULL keys", lambda: lib.bg_randn_keyed(None, B, per, 0, 5, out.data_ptr(), st)),
        ("randn per_sample 0", lambda: lib.bg_randn_keyed(k.data_ptr(), B, 0, 0, 5, out.data_ptr(), st)),
        ("randn per_sample < 0", lambda: lib.bg_randn_keyed(k.data_ptr(), B, -4, 0, 5, out.data_ptr(), st)),
        ("step per_sample 0", lambda: step_call(0)),
        ("step n % per_sample", lambda: step_call(5)),
        ("step t outside 32 bits", lambda: step_call(per, t=2 ** 32)),
        ("step sqrt_abar 0", lambda: step_call(per, sa=0.0)),
        ("tab per_sample < 0", lambda: tab_call(-1, t_cur.data_ptr())),
        ("tab n % per_sample", lambda: tab_call(7, t_cur.data_ptr())),
        ("tab keyed NULL t_cur", lambda: tab_call(per, None)),
    ]
    l0 = lib.bg_launch_count()
    for name, call in cases:
        assert call() == -1, name               # BG_STATUS_BAD_ARG
        assert lib.bg_last_error(), name
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0
    assert torch.isnan(out).all()


# ------------------------------------------------------------------------------------------------------- drop-in
@pytest.mark.parametrize("cfg_w", [0.0, 0.6])
def test_step_with_a_list_of_cpu_generators(cfg_w):
    """DDPMScheduler.step(generator=[g_0 ... g_{B-1}]) == the step fed per-sample torch.randn draws (diffusers'
    randn_tensor list branch); sample i depends on g_i alone"""
    from brepgen_b200.schedulers import DDPMScheduler
    B, shape = 4, (9, 6)
    g = torch.Generator().manual_seed(1)
    eps_c, eps_u, x = (torch.randn((B,) + shape, generator=g).cuda() for _ in range(3))
    kw = dict(model_output_uncond=eps_u, guidance_w=cfg_w) if cfg_w else {}
    sch = DDPMScheduler(clip_sample=True, clip_sample_range=3)
    gens = [torch.Generator().manual_seed(40 + i) for i in range(B)]
    got = sch.step(eps_c, 500, x, generator=gens, **kw).prev_sample
    nz = torch.cat([torch.randn((1,) + shape, generator=torch.Generator().manual_seed(40 + i)) for i in range(B)])
    ref = sch.step(eps_c, 500, x, noise=nz, **kw).prev_sample
    assert torch.equal(got, ref)
    alone = sch.step(eps_c[2:3], 500, x[2:3], generator=[torch.Generator().manual_seed(42)],
                     **({k: (v[2:3] if torch.is_tensor(v) else v) for k, v in kw.items()})).prev_sample
    assert torch.equal(alone[0], got[2])
    with pytest.raises(ValueError):
        sch.step(eps_c, 500, x, generator=gens[:2], **kw)
