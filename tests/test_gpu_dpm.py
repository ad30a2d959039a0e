"""GPU tests of the DPM-Solver++ step (bg_dpm_step, bg_dpm_step_tab), the DPMSolverMultistepScheduler drop-in and
CascadeConfig(schedule="dpm").

  * diffusers' known answer through the product kernel, and this project's answer for final sigma = 0;
  * every output and history element against a float64 evaluation of the step on the kernel's own fp32 inputs;
  * 10- and 20-step chains against DPMOracle; a first-order step is the DDIM step;
  * the eager, keyed and table forms agree bit for bit;
  * the Gaussian convergence and SDE moments through the scheduler and through a graph-replayed loop;
  * small cascades against oracle.dpm.run_cascade_dpm, graph on / off across the late face increase, per-sample noise,
    forward counts, completion;
  * argument errors.
"""
import numpy as np
import pytest
import torch

from oracle.dpm import DPMOracle
from test_dpm import DPM_KAT_MEAN, DPM_ZERO_MEAN, MU, SD, _rms, gaussian_problem
from test_gpu_completion import KNOWN_FIELDS, _n_faces, _nothing_known
from test_gpu_ddim import _keys, _lib, _models, rel_l2
from test_oracle_sched_kat import dummy_model, dummy_sample_deter

pytestmark = pytest.mark.gpu


def _sched(**kw):
    from brepgen_b200.schedulers import DPMSolverMultistepScheduler
    return DPMSolverMultistepScheduler(**kw)


# ------------------------------------------------------------------------------------------------------ known answers
def test_product_scheduler_reproduces_known_answers():
    s = _sched()
    s.set_timesteps(10)
    x = dummy_sample_deter().cuda()
    for t in s.timesteps:
        x = s.step(dummy_model(x, int(t)), t, x).prev_sample
    zero = float(x.abs().mean())
    # diffusers' own test config: final sigma = sigma_min and a second-order last step, through the kernel with the
    # product's coefficients
    f, lib, st = _lib()
    s.set_timesteps(10)
    s.sigmas[-1] = ((1 - s.alphas_cumprod[0]) / s.alphas_cumprod[0]) ** 0.5
    x = dummy_sample_deter().cuda()
    hist = torch.zeros_like(x)
    for k, t in enumerate(s.timesteps.tolist()):
        out = torch.empty_like(x)
        eps = dummy_model(x, t)
        f.check(lib.bg_dpm_step(eps.data_ptr(), None, 0.0, x.data_ptr(), out.data_ptr(), hist.data_ptr(), None, 0, 0, None,
                                0, t, x.numel(), *s.step_coefficients(k, 1 if k == 0 else 2), 0.0, st), "bg_dpm_step")
        x = out
    kat = float(x.abs().mean())
    print(f"DPM KAT: sigma_min config {kat:.6f} (diffusers {DPM_KAT_MEAN}), final sigma 0: {zero:.6f}")
    assert abs(kat - DPM_KAT_MEAN) < 1e-3
    assert abs(zero - DPM_ZERO_MEAN) < 1e-4


# --------------------------------------------------------------------------------------------------- fp64 parity
def dpm_ref64(eps_c, eps_u, w, x, m1, coefs, clip, noise):
    alpha_s, sigma_s, c_x, c_0, c_1, inv_r0, c_z = (float(c) for c in coefs)
    e = eps_c.double()
    if eps_u is not None:
        e = e * (1 + float(np.float32(w))) - eps_u.double() * float(np.float32(w))
    x = x.double()
    x0 = (x - sigma_s * e) / alpha_s
    if clip > 0:
        x0 = x0.clamp(-clip, clip)
    out = c_x * x + c_0 * x0
    if c_1 != 0.0:
        out = out + c_1 * ((x0 - m1.double()) * inv_r0)
    if c_z != 0.0:
        out = out + c_z * noise.double()
    return out, x0


PARITY_BAR = 2e-6     # max |got - ref64| / max(1, |ref64|) per element; for hist (x0) the scale is that of its operands,
                      # max(1, |x0|, (|x| + |sigma_s e|) / alpha_s): at t = 999 x0 = (x - sigma_s e) / alpha_s divides an fp32
                      # difference by alpha_s ~ 0.006, which no fp32 evaluation keeps to 2e-6 of a small |x0|


@pytest.mark.parametrize("algorithm", ["dpmsolver++", "sde-dpmsolver++"])
@pytest.mark.parametrize("k", [0, 10, 19])     # t = 999 (first order), a second-order middle step, the last step
def test_step_matches_float64(k, algorithm):
    f, lib, st = _lib()
    s = _sched(algorithm_type=algorithm)
    s.set_timesteps(20)
    t = int(s.timesteps[k])
    coefs = s.step_coefficients(k, s.step_order(k))
    assert (coefs[4] != 0.0) == (k == 10)
    g = torch.Generator(device="cuda").manual_seed(k)
    B, per = 5, 1003
    x = torch.randn(B, per, generator=g, device="cuda") * 3
    eps_c, eps_u, nz, m1 = (torch.randn(B, per, generator=g, device="cuda") for _ in range(4))
    worst = [0.0, 0.0]
    for clip in (0.0, 3.0):
        for w, u in ((0.0, None), (0.6, eps_u)):
            out = torch.full_like(x, float("nan"))
            hist = m1.clone()
            f.check(lib.bg_dpm_step(eps_c.data_ptr(), f.ptr(u), w, x.data_ptr(), out.data_ptr(), hist.data_ptr(),
                                    nz.data_ptr(), 0, 0, None, 0, t, B * per, *coefs, clip, st), "bg_dpm_step")
            torch.cuda.synchronize()
            ref, x0 = dpm_ref64(eps_c, u, w, x, m1, coefs, clip, nz)
            e64 = eps_c.double() if u is None else eps_c.double() * (1 + float(np.float32(w))) - u.double() * float(np.float32(w))
            x0_scale = torch.maximum(x0.abs(), (x.double().abs() + coefs[1] * e64.abs()) / coefs[0])
            if clip > 0:
                assert int((x0.abs() >= clip).sum()) > 0      # the clamp is really exercised
            for i, (got, want, scale) in enumerate(((out, ref, ref.abs()), (hist, x0, x0_scale))):
                assert torch.isfinite(got).all()
                err = float(((got.double() - want).abs() / scale.clamp_min(1.0)).max())
                worst[i] = max(worst[i], err)
                assert err < PARITY_BAR, (clip, w, i, err)
    print(f"DPM fp64 parity k={k} t={t} {algorithm}: out worst {worst[0]:.3e}, hist worst {worst[1]:.3e}")


# --------------------------------------------------------------------------------------------- chains vs the oracle
@pytest.mark.parametrize("algorithm", ["dpmsolver++", "sde-dpmsolver++"])
@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("n_steps", [10, 20])
def test_dpm_chain_matches_oracle(n_steps, order, algorithm):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(4, 37, 6, generator=g)
    kw = dict(solver_order=order, algorithm_type=algorithm, clip_sample=True, clip_sample_range=3)
    sched, orc = _sched(**kw), DPMOracle(**kw)
    sched.set_timesteps(n_steps), orc.set_timesteps(n_steps)
    xo, xg = x.clone(), x.clone().cuda()
    for t in sched.timesteps:
        nz = torch.randn(x.shape, generator=g)
        xo = orc.step(torch.tanh(xo * 0.7) + 0.1, int(t), xo, noise=nz)
        xg = sched.step(torch.tanh(xg * 0.7) + 0.1, t, xg, variance_noise=nz).prev_sample
    err = rel_l2(xg, xo)
    print(f"DPM chain N={n_steps} order={order} {algorithm}: rel_l2 {err:.2e}")
    assert err < 1e-5


def test_first_order_step_is_the_ddim_step():
    """bg_dpm_step first order from t to t' = bg_ddim_step (eta = 0, clipped eps) to abar_t' within the fp64 bar"""
    from brepgen_b200.schedulers import DDIMScheduler
    f, lib, st = _lib()
    dpm = _sched(solver_order=1, timestep_spacing="leading", clip_sample=True, clip_sample_range=3)
    dpm.set_timesteps(9)
    g = torch.Generator(device="cuda").manual_seed(1)
    B, per = 3, 777
    x, eps = (torch.randn(B, per, generator=g, device="cuda") * 2 for _ in range(2))
    worst = 0.0
    for k, t in enumerate(dpm.timesteps.tolist()):
        ddim = DDIMScheduler(clip_sample=True, clip_sample_range=3, set_alpha_to_one=True)
        ddim.set_timesteps(10 if k < 8 else 9)
        a, b = torch.empty_like(x), torch.empty_like(x)
        f.check(lib.bg_dpm_step(eps.data_ptr(), None, 0.0, x.data_ptr(), a.data_ptr(), None, None, 0, 0, None, 0, t,
                                x.numel(), *dpm.step_coefficients(k, 1), 3.0, st), "dpm")
        f.check(lib.bg_ddim_step(eps.data_ptr(), None, 0.0, x.data_ptr(), b.data_ptr(), None, 0, 0, None, 0, t, x.numel(),
                                 *ddim.step_coefficients(t, 0.0), 3.0, 1, st), "ddim")
        torch.cuda.synchronize()
        err = float(((a.double() - b.double()).abs() / b.double().abs().clamp_min(1.0)).max())
        worst = max(worst, err)
        assert err < PARITY_BAR, (t, err)
    print(f"first-order bg_dpm_step vs bg_ddim_step: worst {worst:.2e}")


# ---------------------------------------------------------------------------------------------- forms agree exactly
@pytest.mark.parametrize("cfg_w", [0.0, 0.6])
@pytest.mark.parametrize("per", [7, 13, 1638])
def test_eager_keyed_and_table_forms_agree(per, cfg_w):
    from brepgen_b200.sampler import randn_keyed
    from brepgen_b200.schedulers import sample_seed
    f, lib, st = _lib()
    B = 7
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(per)
    eps_u = torch.randn(B, per, generator=g, device="cuda") if cfg_w else None
    seeds = [sample_seed(3, b) for b in range(B)]
    k = _keys(seeds, 1)
    s = _sched(algorithm_type="sde-dpmsolver++", clip_sample=True, clip_sample_range=3)
    s.set_timesteps(6)
    ts = s.timesteps
    coef = s.coefficient_table(ts).cuda()
    ts_d = ts.cuda()
    step = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    seed, off0, stride = 0x1234567890ABCDEF, 77, (n + 3) // 4
    hist = {name: torch.zeros(B, per, device="cuda") for name in ("fed", "keyed", "tab", "batch", "tab_b")}
    for i, t in enumerate(ts.tolist()):
        eps_c, x = (torch.randn(B, per, generator=g, device="cuda") * 2 for _ in range(2))
        c = s.step_coefficients(i, s.step_order(i))
        assert list(c) == coef[i].tolist()
        nz = randn_keyed(seeds, 1, (B, per), "cuda", domain=0, t=t)     # the keyed DDPM step's normals at t
        out = {name: torch.full_like(x, float("nan")) for name in hist}
        args = lambda name: (eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), out[name].data_ptr(),
                             hist[name].data_ptr())
        f.check(lib.bg_dpm_step(*args("fed"), nz.data_ptr(), 0, 0, None, 0, t, n, *c, 3.0, st), "fed")
        f.check(lib.bg_dpm_step(*args("keyed"), None, 0, 0, k.data_ptr(), per, t, n, *c, 3.0, st), "keyed")
        f.check(lib.bg_dpm_step(*args("batch"), None, seed, off0 + i * stride, None, 0, t, n, *c, 3.0, st), "batch")
        f.check(lib.bg_step_advance(ts_d.data_ptr(), len(ts), step.data_ptr(), t_cur.data_ptr(), st), "advance")
        f.check(lib.bg_dpm_step_tab(*args("tab"), 0, 0, 0, k.data_ptr(), per, t_cur.data_ptr(), n, coef.data_ptr(),
                                    step.data_ptr(), 3.0, st), "tab keyed")
        f.check(lib.bg_dpm_step_tab(*args("tab_b"), seed, off0, stride, None, 0, None, n, coef.data_ptr(),
                                    step.data_ptr(), 3.0, st), "tab batch")
        torch.cuda.synchronize()
        assert torch.isfinite(out["fed"]).all() and torch.isfinite(out["batch"]).all()
        for a, b in (("keyed", "fed"), ("tab", "keyed"), ("tab_b", "batch")):
            assert torch.equal(out[a], out[b]), (t, a, b)
            assert torch.equal(hist[a], hist[b]), (t, a, b)
        if c[6] != 0.0:
            assert not torch.equal(out["batch"], out["fed"])


# ------------------------------------------------------------------------------------- Gaussian problem on the GPU
def _gaussian_runs(n_steps, algorithm="dpmsolver++", seed=0):
    """(eager scheduler result, graph-replayed result, exact endpoint, xT) of the Gaussian problem of test_dpm.py"""
    from brepgen_b200.sampler import Cascade, CascadeConfig
    xT, _, exact, _ = gaussian_problem(seed=seed)
    acp = _sched().alphas_cumprod.double().cuda()

    def eps_star(x, t):      # t: a device int64 tensor, so the graph can capture it
        a = acp.index_select(0, t.reshape(-1))
        return ((1 - a).sqrt() * (x.double() - a.sqrt() * MU) / (a * SD ** 2 + 1 - a)).float()
    s = _sched(algorithm_type=algorithm)
    s.set_timesteps(n_steps)
    s.set_noise_seed(11)
    x = xT.reshape(1, -1).cuda()
    for t in s.timesteps:
        x = s.step(eps_star(x, t.reshape(1).cuda()), t, x).prev_sample
    eager = x.cpu().reshape(-1)
    s.set_timesteps(n_steps)
    s.set_noise_seed(11)
    cfg = CascadeConfig(graph="on")
    casc = Cascade({})
    tabs = (s.coefficient_table(s.timesteps), s.replace_table(s.timesteps))
    graph = casc._loop_graph(cfg, s, s.timesteps, xT.reshape(1, -1).cuda(), eps_star, None, tabs).cpu().reshape(-1)
    return eager, graph, exact


def test_gaussian_convergence_through_the_product():
    from oracle.ddim import DDIMOracle
    xT, eps_cpu, exact, _ = gaussian_problem()
    for n, bar in ((20, 0.6), (50, 0.15)):
        d = DDIMOracle(clip_sample=False, set_alpha_to_one=True)
        d.set_timesteps(n)
        xd = xT.clone()
        for t in d.timesteps:
            xd = d.step(eps_cpu(xd, t), int(t), xd)
        eager, graph, exact = _gaussian_runs(n)
        assert torch.equal(eager, graph)
        r = _rms(eager, exact) / _rms(xd, exact)
        print(f"GPU Gaussian N={n}: DPM++ 2M rms {_rms(eager, exact):.4f}, DDIM rms {_rms(xd, exact):.4f}, ratio {r:.3f}")
        assert r <= bar


def test_sde_moments_through_the_product():
    eager, graph, _ = _gaussian_runs(100, "sde-dpmsolver++", seed=1)
    assert torch.equal(eager, graph)           # the same batch stream, step for step
    print(f"GPU SDE 100 steps: mean {float(eager.mean()):.4f} std {float(eager.std()):.4f}")
    assert abs(float(eager.mean()) - MU) < 0.01 and abs(float(eager.std()) / SD - 1) < 0.05


# ---------------------------------------------------------------------------------------------------------- cascade
def _cfg(**kw):
    from brepgen_b200.sampler import CascadeConfig
    base = dict(batch_size=2, num_surfaces=4, num_edges=3, class_label=6, schedule="dpm", dpm_steps=4, seed=3,
                decode=False, graph="off")
    base.update(kw)
    return CascadeConfig(**base)


@pytest.mark.parametrize("algorithm", ["dpmsolver++", "sde-dpmsolver++"])
@pytest.mark.parametrize("use_cf", [False, True])
@pytest.mark.parametrize("steps", [4, 10])
def test_short_dpm_cascade_matches_oracle(steps, use_cf, algorithm):
    from oracle.dpm import run_cascade_dpm
    from brepgen_b200.sampler import Cascade
    ms, sds = _models(use_cf)
    cfg = _cfg(use_cf=use_cf, dpm_steps=steps, dpm_algorithm=algorithm)
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

    ref = run_cascade_dpm(sds, cfg, init, step_noise)
    n_oracle = len(bank)
    out = Cascade(ms).run(cfg, init_noise=init, step_noise=step_noise)
    assert len(bank) == n_oracle == (4 * steps if algorithm == "sde-dpmsolver++" else 0)
    assert torch.equal(out["surfMask"].cpu(), ref["surfMask"])
    assert torch.equal(out["edgeM"].cpu(), ref["edgeM"])
    sv, ev = ~ref["surfMask"], ~ref["edgeM"]
    valid = {"surfPos": slice(None), "surfZ": sv, "edgePos": sv, "edge_z": ev, "edgeV": ev}
    for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV"):
        err = rel_l2(out[k].cpu()[valid[k]], ref[k][valid[k]])
        print(f"dpm cascade steps={steps} cf={use_cf} {algorithm} {k} rel_l2={err:.3e}")
        # worst measured on an H100: 2.16e-3 (DPM-4 with CFG, edgeV): the second-order extrapolation over four large steps
        # amplifies the fp16 denoisers' difference from the fp32 oracle more than DDIM's first-order steps (bar 2e-3)
        assert err < 3e-3, (k, err)


def _run(cfg, ms=None, known=None):
    from brepgen_b200.sampler import Cascade
    casc = Cascade(ms if ms is not None else _models(cfg.use_cf)[0])
    out = casc.run(cfg, known=known)
    torch.cuda.synchronize()
    return out, casc


@pytest.mark.parametrize("noise", ["batch", "per_sample"])
@pytest.mark.parametrize("algorithm", ["dpmsolver++", "sde-dpmsolver++"])
def test_graph_on_equals_graph_off(algorithm, noise):
    """12 steps: the surface-position loop crosses the late face increase, so its graph has two segments and the second
    starts first order with a new history"""
    for use_cf in (False, True):
        kw = dict(batch_size=3, num_surfaces=5, num_edges=6, use_cf=use_cf, dpm_steps=12, dpm_algorithm=algorithm,
                  noise=noise)
        a, _ = _run(_cfg(graph="off", **kw))
        b, casc = _run(_cfg(graph="on", **kw))
        assert casc.last_graph_steps == 4 * 12
        for k in a:
            assert torch.equal(a[k], b[k]), (algorithm, noise, use_cf, k)
    if algorithm == "sde-dpmsolver++":        # the noise is really there
        c, _ = _run(_cfg(graph="off", **dict(kw, dpm_algorithm="dpmsolver++")))
        assert not torch.equal(a["surfZ"], c["surfZ"])


@pytest.mark.parametrize("graph", ["off", "on"])
def test_per_sample_dpm_cascade_equals_samples_run_alone(graph):
    kw = dict(num_surfaces=5, num_edges=6, use_cf=False, dpm_steps=12, dpm_algorithm="sde-dpmsolver++",
              noise="per_sample", seed=21, graph=graph)
    full, _ = _run(_cfg(batch_size=5, **kw))
    for b in range(5):
        one, _ = _run(_cfg(batch_size=1, sample_base=b, **kw))
        for k in full:
            assert torch.equal(full[k][b], one[k][0]), (graph, b, k)
    assert not torch.equal(full["surfPos"][0], full["surfPos"][1])


@pytest.mark.parametrize("use_cf", [False, True])
def test_forward_counts_and_late_face_increase(use_cf):
    ms = _models(use_cf)[0]
    calls = {}
    for kind, m in ms.items():
        orig = m.forward

        def wrapped(*a, _k=kind, _o=orig, **kw):
            t = None if torch.cuda.is_current_stream_capturing() else int(a[1].reshape(-1)[0])
            calls.setdefault(_k, []).append((t, a[0].shape[0], a[0].shape[1]))
            return _o(*a, **kw)
        m.forward = wrapped
    try:
        N, B = 10, 2
        out, _ = _run(_cfg(num_surfaces=3, num_edges=2, dpm_steps=N, use_cf=use_cf), ms)
        evaluations = sum(rows // B for v in calls.values() for _, rows, _ in v)
        assert evaluations == (8 * N if use_cf else 4 * N)
        ts = [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]
        assert [(t, s) for t, _, s in calls["surfpos"]] == [(t, 3 if (use_cf or t > 249) else 6) for t in ts]
        calls.clear()
        out_g, casc = _run(_cfg(num_surfaces=3, num_edges=2, dpm_steps=N, use_cf=use_cf, graph="on"), ms)
        assert casc.last_graph_steps == 4 * N
        for k in out:
            assert torch.equal(out[k], out_g[k]), k
    finally:
        for m in ms.values():
            del m.forward


# ------------------------------------------------------------------------------------------------------- completion
@pytest.mark.parametrize("graph", ["off", "on"])
def test_completion_with_dpm(graph):
    from brepgen_b200.sampler import Completion
    kw = dict(batch_size=3, num_surfaces=5, num_edges=4, use_cf=False, dpm_steps=12, dpm_algorithm="sde-dpmsolver++",
              graph=graph)
    a, _ = _run(_cfg(**kw))
    b, _ = _run(_cfg(**kw), known=_nothing_known(_cfg(**kw)))
    for k in a:
        assert torch.equal(a[k], b[k]), k                          # nothing known = the plain run
    known = Completion.from_outputs(a, _n_faces(a, [2, 0, 3]))
    assert sum(known.n_faces) >= 2
    c, _ = _run(_cfg(seed=8, **kw), known=known)
    for i, nf in enumerate(known.n_faces):
        assert not c["surfMask"][i, :nf].any()
        for fk, ok in KNOWN_FIELDS:
            assert torch.equal(c[ok][i, :nf].cpu(), getattr(known, fk)[i, :nf].cpu()), (i, fk)
    assert not torch.equal(c["surfPos"][1], a["surfPos"][1])


def test_completion_matches_oracle():
    from brepgen_b200.sampler import Cascade
    from oracle.dpm import run_cascade_dpm
    ms, sds = _models(False)
    cfg = _cfg(dpm_steps=10)
    g = torch.Generator().manual_seed(9)

    def init():
        return {"surfPos": torch.randn(2, 4, 6, generator=g), "surfZ": torch.randn(2, 8, 48, generator=g),
                "edgePos": torch.randn(2, 8, 3, 6, generator=g), "edgeZV": torch.randn(2, 8, 3, 18, generator=g)}
    a = run_cascade_dpm(sds, cfg, init(), None)
    from brepgen_b200.sampler import Completion
    known = Completion.from_outputs(a, _n_faces(a, [1, 2]))
    init_b = init()
    rbank = {}

    def rnoise(name, k, shape):
        key = (name, k, tuple(shape))
        if key not in rbank:
            rbank[key] = torch.randn(tuple(shape), generator=g)
        return rbank[key]
    ref = run_cascade_dpm(sds, cfg, init_b, None, known=known, replace_noise=rnoise)
    out = Cascade(ms).run(cfg, init_noise=init_b, known=known, replace_noise=rnoise)
    assert torch.equal(out["surfMask"].cpu(), ref["surfMask"]) and torch.equal(out["edgeM"].cpu(), ref["edgeM"])
    sv, ev = ~ref["surfMask"], ~ref["edgeM"]
    valid = {"surfPos": slice(None), "surfZ": sv, "edgePos": sv, "edge_z": ev, "edgeV": ev}
    for k in valid:
        err = rel_l2(out[k].cpu()[valid[k]], ref[k][valid[k]])
        print(f"dpm completion {k} rel_l2={err:.3e}")
        assert err < 1e-3, (k, err)


# ----------------------------------------------------------------------------------------------------------- errors
def test_bad_arguments_are_rejected_and_launch_nothing():
    f, lib, st = _lib()
    B, per = 3, 8
    n = B * per
    eps, x = torch.randn(B, per, device="cuda"), torch.randn(B, per, device="cuda")
    hist = torch.zeros(B, per, device="cuda")
    k = _keys([1, 2, 3], 0)
    out = torch.full((B, per), float("nan"), device="cuda")
    coef = torch.ones(1, 7, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    c = (0.8, 0.5, 0.9, 0.3, 0.1, 1.5, 0.2)

    def eager(eps_p=eps.data_ptr(), x_p=x.data_ptr(), out_p=out.data_ptr(), h_p=hist.data_ptr(), keys=k.data_ptr(),
              per_s=per, t=5, nn=n, coefs=c):
        return lib.bg_dpm_step(eps_p, None, 0.0, x_p, out_p, h_p, None, 1, 0, keys, per_s, t, nn, *coefs, 3.0, st)

    def tab(eps_p=eps.data_ptr(), x_p=x.data_ptr(), out_p=out.data_ptr(), h_p=hist.data_ptr(), keys=k.data_ptr(),
            per_s=per, tc=t_cur.data_ptr(), nn=n, cf=coef.data_ptr(), sp=step.data_ptr()):
        return lib.bg_dpm_step_tab(eps_p, None, 0.0, x_p, out_p, h_p, 1, 0, 6, keys, per_s, tc, nn, cf, sp, 3.0, st)
    cases = [
        ("eager NULL eps", lambda: eager(eps_p=None)), ("eager NULL x", lambda: eager(x_p=None)),
        ("eager NULL out", lambda: eager(out_p=None)), ("eager NULL hist, c_1 != 0", lambda: eager(h_p=None)),
        ("eager n 0", lambda: eager(nn=0)), ("eager per_sample 0", lambda: eager(per_s=0)),
        ("eager per_sample < 0", lambda: eager(per_s=-8)), ("eager n % per_sample", lambda: eager(per_s=5)),
        ("eager alpha_s 0", lambda: eager(coefs=(0.0,) + c[1:])), ("eager alpha_s < 0", lambda: eager(coefs=(-0.8,) + c[1:])),
        ("eager t < 0", lambda: eager(t=-1)), ("eager t > 32 bits", lambda: eager(t=2 ** 32)),
        ("tab NULL eps", lambda: tab(eps_p=None)), ("tab NULL out", lambda: tab(out_p=None)),
        ("tab NULL hist", lambda: tab(h_p=None)), ("tab NULL coef", lambda: tab(cf=None)),
        ("tab NULL step", lambda: tab(sp=None)), ("tab keyed NULL t_cur", lambda: tab(tc=None)),
        ("tab per_sample 0", lambda: tab(per_s=0)), ("tab n % per_sample", lambda: tab(per_s=7)), ("tab n 0", lambda: tab(nn=0)),
    ]
    l0 = lib.bg_launch_count()
    for name, call in cases:
        assert call() == -1, name               # BG_STATUS_BAD_ARG
        assert lib.bg_last_error(), name
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0
    assert torch.isnan(out).all() and (hist == 0).all()
    # valid calls launch: the last 32-bit t, the batch forms (per_sample and t_cur ignored), a first-order step without hist
    assert eager(t=2 ** 32 - 1) == 0 and eager(keys=None, per_s=0) == 0 and tab(keys=None, per_s=0, tc=None) == 0
    assert eager(h_p=None, coefs=c[:4] + (0.0, 0.0, 0.2)) == 0
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0 + 4
