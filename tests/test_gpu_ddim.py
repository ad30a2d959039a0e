"""GPU tests of the DDIM step (bg_ddim_step, bg_ddim_step_tab), the DDIMScheduler drop-in and CascadeConfig(schedule="ddim").

  * the product scheduler reproduces the known answers of diffusers' DDIM tests through the kernel;
  * every output element against a float64 evaluation of the step on the kernel's own fp32 inputs;
  * 10- and 50-step chains against DDIMOracle;
  * the eager, keyed and table forms agree bit for bit, and keyed DDIM draws the keyed DDPM step's normals;
  * eta = 1 over the 1000-step table with clipped eps is the DDPM step;
  * small cascades against oracle.ddim.run_cascade_ddim, graph on / off, per-sample noise, forward counts, the late face increase;
  * argument errors.
"""
import numpy as np
import pytest
import torch

from oracle.ddim import DDIMOracle
from test_ddim import DDIM_KATS
from test_oracle_sched_kat import dummy_model, dummy_sample_deter

pytestmark = pytest.mark.gpu


def _lib():
    from brepgen_b200 import _ffi as f
    return f, f.lib(), f.current_stream()


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------------ known answers
@pytest.mark.parametrize("kw,kat_sum,kat_mean", DDIM_KATS)
def test_product_scheduler_reproduces_diffusers_known_answers(kw, kat_sum, kat_mean):
    from brepgen_b200.schedulers import DDIMScheduler
    s = DDIMScheduler(**kw)
    s.set_timesteps(10)
    x = dummy_sample_deter().cuda()
    for t in s.timesteps:
        x = s.step(dummy_model(x, int(t)), t, x, eta=0.0).prev_sample
    x = x.cpu()
    print(f"DDIM KAT {kw}: sum {float(x.abs().sum()):.5f} mean {float(x.abs().mean()):.7f}")
    assert abs(float(x.abs().sum()) - kat_sum) < 1e-2
    assert abs(float(x.abs().mean()) - kat_mean) < 1e-3


# --------------------------------------------------------------------------------------------------- fp64 parity
def ddim_ref64(eps_c, eps_u, w, x, coefs, clip, use_clipped, noise):
    """float64 DDIM step on the kernel's fp32 inputs and fp32 coefficients"""
    sb, sa, sa_prev, c_dir, sigma = (float(c) for c in coefs)
    e = eps_c.double()
    if eps_u is not None:
        e = e * (1 + float(np.float32(w))) - eps_u.double() * float(np.float32(w))
    x = x.double()
    x0 = (x - sb * e) / sa
    if clip > 0:
        x0 = x0.clamp(-clip, clip)
    if use_clipped:
        e = (x - sa * x0) / sb
    out = sa_prev * x0 + c_dir * e
    if sigma != 0.0:
        out = out + sigma * noise.double()
    return out, x0


# (timestep, num_inference_steps, set_alpha_to_one): first steps, a middle step and the last steps (prev < 0)
PARITY_STEPS = [(999, 1000, True), (900, 10, True), (500, 50, True), (0, 10, True), (0, 10, False), (0, 1000, False)]
PARITY_BAR = 5e-7     # max |out - ref64| / max(1, max |ref64|) per case; worst measured on an H100: 1.41e-7


@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("t,n_steps,set_alpha_to_one", PARITY_STEPS)
def test_step_matches_float64(t, n_steps, set_alpha_to_one, eta):
    from brepgen_b200.schedulers import DDIMScheduler
    f, lib, st = _lib()
    g = torch.Generator(device="cuda").manual_seed(t + n_steps)
    B, per = 5, 1003
    x = torch.randn(B, per, generator=g, device="cuda") * 3
    eps_c, eps_u, nz = (torch.randn(B, per, generator=g, device="cuda") for _ in range(3))
    s = DDIMScheduler(set_alpha_to_one=set_alpha_to_one)
    s.set_timesteps(n_steps)
    coefs = s.step_coefficients(t, eta)
    worst = 0.0
    for clip in (0.0, 3.0):
        for use_clipped in (0, 1):
            for w, u in ((0.0, None), (0.6, eps_u)):
                out = torch.full_like(x, float("nan"))
                f.check(lib.bg_ddim_step(eps_c.data_ptr(), f.ptr(u), w, x.data_ptr(), out.data_ptr(), nz.data_ptr(), 0, 0,
                                         None, 0, t, B * per, *coefs, clip, use_clipped, st), "bg_ddim_step")
                torch.cuda.synchronize()
                ref, x0 = ddim_ref64(eps_c, u, w, x, coefs, clip, use_clipped, nz)
                if clip > 0:
                    assert int((x0.abs() >= clip).sum()) > 0      # the clamp is really exercised
                err = float((out.double() - ref).abs().max() / max(1.0, float(ref.abs().max())))
                worst = max(worst, err)
                assert torch.isfinite(out).all()
                assert err < PARITY_BAR, (clip, use_clipped, w, err)
    print(f"DDIM fp64 parity t={t} N={n_steps} one={set_alpha_to_one} eta={eta}: worst {worst:.3e}")


# --------------------------------------------------------------------------------------------- chains vs the oracle
@pytest.mark.parametrize("eta", [0.0, 0.5])
@pytest.mark.parametrize("shape", [(4, 37, 6), (3, 11, 48)])
@pytest.mark.parametrize("n_steps", [10, 50])
def test_ddim_chain_matches_oracle(n_steps, shape, eta):
    from brepgen_b200.schedulers import DDIMScheduler
    g = torch.Generator().manual_seed(5)
    x = torch.randn(*shape, generator=g)
    sched = DDIMScheduler(clip_sample=True, clip_sample_range=3)
    orc = DDIMOracle(clip_sample=True, clip_sample_range=3)
    sched.set_timesteps(n_steps), orc.set_timesteps(n_steps)
    xo, xg = x.clone(), x.clone().cuda()
    for t in sched.timesteps:
        nz = torch.randn(x.shape, generator=g)
        xo = orc.step(torch.tanh(xo * 0.7) + 0.1, int(t), xo, eta, noise=nz)
        xg = sched.step(torch.tanh(xg * 0.7) + 0.1, t, xg, eta=eta, variance_noise=nz).prev_sample
    err = rel_l2(xg, xo)
    print(f"DDIM chain N={n_steps} {shape} eta={eta}: rel_l2 {err:.2e}")
    assert err < 1e-5


# ---------------------------------------------------------------------------------------------- forms agree exactly
def _keys(seeds, stage):
    from brepgen_b200.schedulers import sample_keys
    return torch.from_numpy(sample_keys(seeds, stage).view(np.int64)).cuda()


@pytest.mark.parametrize("use_clipped", [0, 1])
@pytest.mark.parametrize("cfg_w", [0.0, 0.6])
@pytest.mark.parametrize("per", [7, 13, 1638])
def test_forms_agree_and_draw_the_ddpm_step_noise(per, cfg_w, use_clipped):
    from brepgen_b200.sampler import randn_keyed
    from brepgen_b200.schedulers import DDIMScheduler, sample_seed
    f, lib, st = _lib()
    B, eta = 7, 0.5
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(per)
    eps_c, eps_u, x = (torch.randn(B, per, generator=g, device="cuda") * 2 for _ in range(3))
    eps_u = eps_u if cfg_w else None
    seeds = [sample_seed(3, b) for b in range(B)]
    k = _keys(seeds, 1)
    s = DDIMScheduler(clip_sample_range=3)
    s.set_timesteps(5)
    ts = s.timesteps
    coef = s.coefficient_table(ts, eta).cuda()
    ts_d = ts.cuda()
    step = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    seed, off0, stride = 0x1234567890ABCDEF, 77, (n + 3) // 4

    def new():
        return torch.full_like(x, float("nan"))
    for i, t in enumerate(ts.tolist()):
        c = s.step_coefficients(t, eta)
        nz = randn_keyed(seeds, 1, (B, per), "cuda", domain=0, t=t)
        fed, keyed, tab, batch, tab_b = new(), new(), new(), new(), new()
        f.check(lib.bg_ddim_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), fed.data_ptr(), nz.data_ptr(), 0, 0,
                                 None, 0, t, n, *c, 3.0, use_clipped, st), "fed")
        f.check(lib.bg_ddim_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), keyed.data_ptr(), None, 0, 0,
                                 k.data_ptr(), per, t, n, *c, 3.0, use_clipped, st), "keyed")
        f.check(lib.bg_ddim_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), batch.data_ptr(), None, seed,
                                 off0 + i * stride, None, 0, t, n, *c, 3.0, use_clipped, st), "batch")
        f.check(lib.bg_step_advance(ts_d.data_ptr(), len(ts), step.data_ptr(), t_cur.data_ptr(), st), "advance")
        f.check(lib.bg_ddim_step_tab(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), tab.data_ptr(), 0, 0, 0,
                                     k.data_ptr(), per, t_cur.data_ptr(), n, coef.data_ptr(), step.data_ptr(), 3.0,
                                     use_clipped, st), "tab keyed")
        f.check(lib.bg_ddim_step_tab(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), tab_b.data_ptr(), seed, off0,
                                     stride, None, 0, None, n, coef.data_ptr(), step.data_ptr(), 3.0, use_clipped, st),
                "tab batch")
        torch.cuda.synchronize()
        assert torch.isfinite(fed).all() and torch.isfinite(batch).all()
        assert torch.equal(keyed, fed), t
        assert torch.equal(tab, keyed), t
        assert torch.equal(tab_b, batch), t
        # the batch stream is bg_ddpm_step's: a DDPM step that returns its noise (c_x0 = c_x = 0, sigma = 1) shows the
        # normals the DDIM step added (up to the rounding of sigma * z + rest, which the kernel fuses)
        if c[4] != 0.0:
            assert not torch.equal(batch, fed)
            quiet = new()
            f.check(lib.bg_ddim_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), quiet.data_ptr(), None, 0, 0, None,
                                     0, t, n, *c[:4], 0.0, 3.0, use_clipped, st), "quiet")
            z_ddpm = new()
            zero = torch.zeros_like(x)
            f.check(lib.bg_ddpm_step(zero.data_ptr(), None, 0.0, zero.data_ptr(), z_ddpm.data_ptr(), None, seed,
                                     off0 + i * stride, None, 0, 0, n, 0.5, 1.0, 0.0, 0.0, 0.0, 1.0, st), "ddpm noise")
            torch.cuda.synchronize()
            assert torch.allclose(batch, quiet + c[4] * z_ddpm, rtol=1e-6, atol=1e-6)


def test_scheduler_generator_and_stream_paths():
    """DDIMScheduler.step: a CPU generator gives the step fed the same torch.randn draw; per-sample mode gives the step fed
    bg_randn_keyed(domain 0, t); the batch stream is reproducible from set_noise_seed"""
    from brepgen_b200.sampler import randn_keyed
    from brepgen_b200.schedulers import DDIMScheduler, sample_seed
    s = DDIMScheduler(clip_sample_range=3)
    s.set_timesteps(20)
    g = torch.Generator().manual_seed(2)
    B, shape = 3, (9, 6)
    eps, x = (torch.randn((B,) + shape, generator=g).cuda() for _ in range(2))
    got = s.step(eps, 500, x, eta=0.8, generator=torch.Generator().manual_seed(7)).prev_sample
    ref = s.step(eps, 500, x, eta=0.8, variance_noise=torch.randn((B,) + shape,
                                                                  generator=torch.Generator().manual_seed(7))).prev_sample
    assert torch.equal(got, ref)
    s.set_sample_keys(seed=4, first=2, stage=3)
    keyed = s.step(eps, 500, x, eta=0.8).prev_sample
    nz = randn_keyed([sample_seed(4, 2 + b) for b in range(B)], 3, (B,) + shape, "cuda", domain=0, t=500)
    assert torch.equal(keyed, s.step(eps, 500, x, eta=0.8, variance_noise=nz).prev_sample)
    a, b = DDIMScheduler(), DDIMScheduler()
    for sch in (a, b):
        sch.set_timesteps(20)
        sch.set_noise_seed(9, 0, 1)
    ra = [a.step(eps, t, x, eta=1.0).prev_sample for t in (500, 450)]
    rb = [b.step(eps, t, x, eta=1.0).prev_sample for t in (500, 450)]
    assert torch.equal(ra[0], rb[0]) and torch.equal(ra[1], rb[1]) and not torch.equal(ra[0], ra[1])
    out = torch.empty_like(x)
    r = s.step(eps, 500, x, eta=0.0, out=out, return_dict=False)
    assert r[0] is out


# ------------------------------------------------------------------------------------------------ eta = 1 is DDPM
# The two steps agree in exact arithmetic, not in rounding: the x0 terms of DDIM (sqrt(abar_prev) x0 and the x0 inside e_dir)
# cancel down to DDPM's c_x0 x0, so a coefficient's rounding shows at the scale of the DDIM terms, not of the result.
DDPM_EQ_STEP_ULPS = 6      # |ddim - ddpm| in fp32 ulps of |sqrt(abar_prev) x0| + |c_dir e_dir| + |sigma z| per element;
                           # worst measured on an H100: 1.73 (t = 999, 700, 250); t = 0 reduces to x0 in both exactly
DDPM_EQ_CHAIN_BAR = 3e-5   # rel-L2 of the 1000-step chain; measured on an H100: 7.7e-6


def _ddpm_ddim(clip_range=1.0):
    from brepgen_b200.schedulers import DDIMScheduler, DDPMScheduler
    ddim = DDIMScheduler(clip_sample=True, clip_sample_range=clip_range, set_alpha_to_one=True)
    ddpm = DDPMScheduler(clip_sample=True, clip_sample_range=clip_range)
    ddim.set_timesteps(1000), ddpm.set_timesteps(1000)
    return ddim, ddpm


def test_eta_one_step_is_the_ddpm_step():
    ddim, ddpm = _ddpm_ddim(3.0)
    g = torch.Generator().manual_seed(3)
    x, eps, nz = (torch.randn(6, 500, generator=g).cuda() * 2 for _ in range(3))
    # Not at t = 1..~10: there both schedulers' fp32 coefficients (computed as diffusers computes them) come from 1 - abar
    # ~ 1e-4, which keeps ~3 fewer digits, and the two formulas round differently (measured 475 ulps at t = 1, from the host
    # coefficients, not the kernel).  The 1000-step chain below covers those steps.
    for t in (999, 700, 250, 0):
        a = ddim.step(eps, t, x, eta=1.0, use_clipped_model_output=True, variance_noise=nz).prev_sample
        b = ddpm.step(eps, t, x, noise=nz).prev_sample
        sb, sa, sa_prev, c_dir, sigma = ddim.step_coefficients(t, 1.0)
        x0 = ((x.double() - sb * eps.double()) / sa).clamp(-3, 3)
        e_dir = (x.double() - sa * x0) / sb
        scale = (sa_prev * x0).abs() + (c_dir * e_dir).abs() + (sigma * nz.double()).abs()
        ulps = float(((a.double() - b.double()).abs() / (scale * 2.0 ** -23)).max())
        print(f"eta=1 DDIM vs DDPM t={t}: {ulps:.2f} ulps")
        assert ulps <= DDPM_EQ_STEP_ULPS, (t, ulps)
        if t == 0:
            assert torch.equal(a, b)


def test_eta_one_chain_is_the_ddpm_chain():
    """1000 steps over the dummy model with noise: the clipped-eps DDIM chain is the DDPM chain; without the flag the
    clamp (active on this sample) makes them differ, so the flag is really tested"""
    ddim, ddpm = _ddpm_ddim(1.0)
    g = torch.Generator().manual_seed(0)
    xa = xb = xc = (dummy_sample_deter() * 4).cuda()
    for t in range(999, -1, -1):
        nz = torch.randn(xa.shape, generator=g).cuda()
        xa = ddim.step(dummy_model(xa, t), t, xa, eta=1.0, use_clipped_model_output=True, variance_noise=nz).prev_sample
        xc = ddim.step(dummy_model(xc, t), t, xc, eta=1.0, variance_noise=nz).prev_sample
        xb = ddpm.step(dummy_model(xb, t), t, xb, noise=nz if t > 0 else None).prev_sample
    e_on, e_off = rel_l2(xa, xb), rel_l2(xc, xb)
    print(f"eta=1 1000-step chain: clipped eps {e_on:.2e}, unclipped eps {e_off:.2e}")
    assert e_on < DDPM_EQ_CHAIN_BAR
    assert e_off > 1e-2


# ---------------------------------------------------------------------------------------------------------- cascade
_MODELS = {}


def _models(use_cf):
    if use_cf not in _MODELS:
        from brepgen_b200.models import NETS
        from brepgen_b200.spec import denoiser_spec
        from brepgen_b200.synth import synth_state_dict
        ms, sds = {}, {}
        for kind in NETS:
            sds[kind] = synth_state_dict(denoiser_spec(kind, use_cf), seed=11)
            m = NETS[kind](use_cf)
            m.load_state_dict(sds[kind])
            ms[kind] = m.cuda().eval()
        _MODELS[use_cf] = (ms, sds)
    return _MODELS[use_cf]


def _cfg(**kw):
    from brepgen_b200.sampler import CascadeConfig
    base = dict(batch_size=2, num_surfaces=4, num_edges=3, class_label=6, schedule="ddim", ddim_steps=4, seed=3,
                decode=False, graph="off")
    base.update(kw)
    return CascadeConfig(**base)


@pytest.mark.parametrize("use_cf", [False, True])
@pytest.mark.parametrize("steps", [4, 10])
def test_short_ddim_cascade_matches_oracle(steps, use_cf):
    from oracle.ddim import run_cascade_ddim
    from brepgen_b200.sampler import Cascade
    ms, sds = _models(use_cf)
    cfg = _cfg(use_cf=use_cf, ddim_steps=steps, ddim_eta=0.5)
    S = cfg.num_surfaces if use_cf else 2 * cfg.num_surfaces
    g = torch.Generator().manual_seed(9)
    init = {"surfPos": torch.randn(2, cfg.num_surfaces, 6, generator=g), "surfZ": torch.randn(2, S, 48, generator=g),
            "edgePos": torch.randn(2, S, 3, 6, generator=g), "edgeZV": torch.randn(2, S, 3, 18, generator=g)}
    bank = {}

    def step_noise(name, k, shape):
        key = (name, k)
        if key not in bank:
            bank[key] = torch.randn(tuple(shape), generator=g)
        return bank[key]

    ref = run_cascade_ddim(sds, cfg, init, step_noise)
    n_oracle = len(bank)
    out = Cascade(ms).run(cfg, init_noise=init, step_noise=step_noise)
    assert len(bank) == n_oracle == 4 * steps          # noise on every step when eta > 0, the same draws on both sides
    assert torch.equal(out["surfMask"].cpu(), ref["surfMask"])
    assert torch.equal(out["edgeM"].cpu(), ref["edgeM"])
    sv, ev = ~ref["surfMask"], ~ref["edgeM"]
    valid = {"surfPos": slice(None), "surfZ": sv, "edgePos": sv, "edge_z": ev, "edgeV": ev}
    for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV"):
        err = rel_l2(out[k].cpu()[valid[k]], ref[k][valid[k]])
        print(f"ddim cascade steps={steps} cf={use_cf} {k} rel_l2={err:.3e}")
        assert err < 2e-3, (k, err)


def _run(cfg, ms=None):
    from brepgen_b200.sampler import Cascade
    casc = Cascade(ms if ms is not None else _models(cfg.use_cf)[0])
    out = casc.run(cfg)
    torch.cuda.synchronize()
    return out, casc


@pytest.mark.parametrize("noise", ["batch", "per_sample"])
@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_graph_on_equals_graph_off(eta, noise):
    for use_cf in (False, True):
        kw = dict(batch_size=3, num_surfaces=5, num_edges=6, use_cf=use_cf, ddim_steps=12, ddim_eta=eta, noise=noise)
        a, _ = _run(_cfg(graph="off", **kw))
        b, casc = _run(_cfg(graph="on", **kw))
        assert casc.last_graph_steps == 4 * 12
        for k in a:
            assert torch.equal(a[k], b[k]), (eta, noise, use_cf, k)
    if eta > 0:        # the noise is really there
        c, _ = _run(_cfg(graph="off", **dict(kw, ddim_eta=0.0)))
        assert not torch.equal(a["surfZ"], c["surfZ"])


@pytest.mark.parametrize("graph", ["off", "on"])
def test_per_sample_ddim_cascade_equals_samples_run_alone(graph):
    kw = dict(num_surfaces=5, num_edges=6, use_cf=True, ddim_steps=6, ddim_eta=0.5, noise="per_sample", seed=21,
              graph=graph, decode=True)
    from brepgen_b200.vae import build_synthetic_decoders
    ms = _models(True)[0]
    sv, ev = build_synthetic_decoders(torch.device("cuda"))
    from brepgen_b200.sampler import Cascade

    def run(cfg):
        out = Cascade(ms, sv, ev).run(cfg)
        torch.cuda.synchronize()
        return out
    full = run(_cfg(batch_size=5, **kw))
    assert "surf_ncs" in full and "edge_ncs" in full
    for b in range(5):
        one = run(_cfg(batch_size=1, sample_base=b, **kw))
        for k in full:
            assert torch.equal(full[k][b], one[k][0]), (graph, b, k)
    assert not torch.equal(full["surfPos"][0], full["surfPos"][1])


def test_forward_counts_and_late_face_increase():
    ms = _models(False)[0]
    calls = {}
    for kind, m in ms.items():
        orig = m.forward

        def wrapped(*a, _k=kind, _o=orig, **kw):
            t = None if torch.cuda.is_current_stream_capturing() else int(a[1].reshape(-1)[0])
            calls.setdefault(_k, []).append((t, a[0].shape[1]))
            return _o(*a, **kw)
        m.forward = wrapped
    try:
        N = 10
        out, _ = _run(_cfg(num_surfaces=3, num_edges=2, ddim_steps=N, graph="off"), ms)
        assert {k: len(v) for k, v in calls.items()} == {k: N for k in ("surfpos", "surfz", "edgepos", "edgez")}
        # timesteps 900, 800, ..., 0: the face slots double at the first t <= 249 (t = 200), as in sample.py:140-142
        assert calls["surfpos"] == [(t, 3 if t > 249 else 6) for t in range(900, -1, -100)]
        assert out["surfPos"].shape == (2, 6, 6)
        calls.clear()
        out_g, casc = _run(_cfg(num_surfaces=3, num_edges=2, ddim_steps=N, graph="on"), ms)
        # graphs: warm-up + capture per segment; the surface-position loop has two segments (before / after the increase)
        assert {k: len(v) for k, v in calls.items()} == {"surfpos": 4, "surfz": 2, "edgepos": 2, "edgez": 2}
        assert casc.last_graph_steps == 4 * N
        for k in out:
            assert torch.equal(out[k], out_g[k]), k
    finally:
        for m in ms.values():
            del m.forward


# ----------------------------------------------------------------------------------------------------------- errors
def test_bad_arguments_are_rejected_and_launch_nothing():
    f, lib, st = _lib()
    B, per = 3, 8
    n = B * per
    eps, x = torch.randn(B, per, device="cuda"), torch.randn(B, per, device="cuda")
    k = _keys([1, 2, 3], 0)
    out = torch.full((B, per), float("nan"), device="cuda")
    coef = torch.ones(1, 5, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    c = (0.5, 0.8, 0.9, 0.3, 0.1)

    def eager(eps_p=eps.data_ptr(), x_p=x.data_ptr(), out_p=out.data_ptr(), keys=k.data_ptr(), per_s=per, t=5, nn=n,
              coefs=c):
        return lib.bg_ddim_step(eps_p, None, 0.0, x_p, out_p, None, 1, 0, keys, per_s, t, nn, *coefs, 3.0, 0, st)

    def tab(eps_p=eps.data_ptr(), x_p=x.data_ptr(), out_p=out.data_ptr(), keys=k.data_ptr(), per_s=per, tc=t_cur.data_ptr(),
            nn=n, cf=coef.data_ptr(), sp=step.data_ptr()):
        return lib.bg_ddim_step_tab(eps_p, None, 0.0, x_p, out_p, 1, 0, 6, keys, per_s, tc, nn, cf, sp, 3.0, 0, st)
    cases = [
        ("eager NULL eps", lambda: eager(eps_p=None)), ("eager NULL x", lambda: eager(x_p=None)),
        ("eager NULL out", lambda: eager(out_p=None)), ("eager n 0", lambda: eager(nn=0)),
        ("eager per_sample 0", lambda: eager(per_s=0)), ("eager per_sample < 0", lambda: eager(per_s=-8)),
        ("eager n % per_sample", lambda: eager(per_s=5)), ("eager sqrt_abar 0", lambda: eager(coefs=(0.5, 0.0, 0.9, 0.3, 0.1))),
        ("eager sqrt_abar < 0", lambda: eager(coefs=(0.5, -0.8, 0.9, 0.3, 0.1))), ("eager t < 0", lambda: eager(t=-1)),
        ("eager t > 32 bits", lambda: eager(t=2 ** 32)),
        ("tab NULL eps", lambda: tab(eps_p=None)), ("tab NULL out", lambda: tab(out_p=None)),
        ("tab NULL coef", lambda: tab(cf=None)), ("tab NULL step", lambda: tab(sp=None)),
        ("tab keyed NULL t_cur", lambda: tab(tc=None)), ("tab per_sample 0", lambda: tab(per_s=0)),
        ("tab n % per_sample", lambda: tab(per_s=7)), ("tab n 0", lambda: tab(nn=0)),
    ]
    l0 = lib.bg_launch_count()
    for name, call in cases:
        assert call() == -1, name               # BG_STATUS_BAD_ARG
        assert lib.bg_last_error(), name
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0
    assert torch.isnan(out).all()
    # the same calls with valid arguments launch (the batch forms ignore per_sample and t_cur)
    assert eager(t=2 ** 32 - 1) == 0 and eager(keys=None, per_s=0) == 0 and tab(keys=None, per_s=0, tc=None) == 0
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0 + 3
