"""GPU tests of the UniPC step (bg_unipc_step, bg_unipc_step_tab), the UniPCMultistepScheduler drop-in and
CascadeConfig(schedule="unipc").

  * diffusers' known answer and the oracle's other full-loop values through the product kernel;
  * every output, last and history element against a float64 evaluation of the step on the kernel's own fp32 inputs;
  * the eager and table forms agree bit for bit;
  * small cascades against oracle.unipc.run_cascade_unipc, graph on / off across the late face increase, per-sample
    noise, forward counts, completion and variations;
  * argument errors.
"""
import pytest
import torch

from oracle.unipc import UniPCOracle, run_cascade_unipc, run_cascade_variation_unipc
from test_gpu_completion import KNOWN_FIELDS, _n_faces, _nothing_known
from test_gpu_ddim import _lib, _models, rel_l2
from test_gpu_variation import _fit, _start_noise, _var
from test_oracle_sched_kat import dummy_model, dummy_sample_deter
from test_unipc import UNIPC_KAT_MEAN, UNIPC_VARIANTS

pytestmark = pytest.mark.gpu


def _sched(**kw):
    from brepgen_b200.schedulers import UniPCMultistepScheduler
    return UniPCMultistepScheduler(**kw)


# ------------------------------------------------------------------------------------------------------ known answers
def test_product_scheduler_reproduces_known_answers():
    for kw, mean in [(dict(), UNIPC_KAT_MEAN)] + UNIPC_VARIANTS + [(dict(solver_order=3, solver_type="bh1",
                                                                        final_sigmas_type="zero"), None)]:
        s, o = _sched(**kw), UniPCOracle(**kw)
        s.set_timesteps(10), o.set_timesteps(10)
        x, xo = dummy_sample_deter().cuda(), dummy_sample_deter()
        for t in s.timesteps:
            x = s.step(dummy_model(x, int(t)), t, x).prev_sample
            xo = o.step(dummy_model(xo, int(t)), int(t), xo)
        got = float(x.abs().mean())
        err = rel_l2(x.cpu(), xo)
        print(f"UniPC full loop {kw}: |x| mean {got:.6f} (oracle {float(xo.abs().mean()):.6f}), rel_l2 {err:.2e}")
        if mean is not None:
            assert abs(got - mean) < (1e-3 if not kw else 6e-5)
        assert err < 1e-6


# --------------------------------------------------------------------------------------------------- fp64 parity
def unipc_ref64(row, e, x, last, hist, clip):
    """(out, last, x0) of one step in float64 from the row's fp32 coefficients, and the same expressions with every value
    and coefficient replaced by its magnitude (the scale an fp32 evaluation's rounding error is bounded by)"""
    r = [float(v) for v in row]
    c, p = int(r[2]), int(r[3])
    m = [hist[int(r[5 + i])].double() for i in range(3)]
    res = {}
    for mode in ("value", "magnitude"):
        A = (lambda v: v.abs()) if mode == "magnitude" else (lambda v: v)
        k = (lambda v: abs(v)) if mode == "magnitude" else (lambda v: v)
        sub = (lambda a, b: a + b) if mode == "magnitude" else (lambda a, b: a - b)
        x0 = sub(A(x.double()), k(r[1]) * A(e.double())) / k(r[0])
        if clip > 0 and mode == "value":
            x0 = x0.clamp(-clip, clip)     # the magnitude stays unclamped: it bounds a value rounded across the clamp
        mm = [A(v) for v in m]
        xc = A(x.double())
        if c > 0:
            tot = k(r[15]) * sub(x0, mm[0])
            if c >= 2:
                tot = tot + k(r[13]) * sub(mm[1], mm[0]) / k(r[11])
            if c >= 3:
                tot = tot + k(r[14]) * sub(mm[2], mm[0]) / k(r[12])
            xc = sub(sub(k(r[8]) * A(last.double()), k(r[9]) * mm[0]), k(r[10]) * tot)
        o = sub(k(r[16]) * xc, k(r[17]) * x0)
        if p >= 2:
            tot = k(r[21]) * sub(mm[0], x0) / k(r[19])
            if p >= 3:
                tot = tot + k(r[22]) * sub(mm[1], x0) / k(r[20])
            o = sub(o, k(r[18]) * tot)
        res[mode] = (o, xc, x0)
    return res["value"], res["magnitude"]


PARITY_ULP = 4        # |got - ref64| <= 4 ulp (2^-23 each) of the magnitude sum, which bounds every partial result of
                      # the chain (CFG, x0, the corrector's terms, the predictor's); worst measured on an H100: 1.51 ulp


@pytest.mark.parametrize("case", [dict(k=0), dict(k=10, solver_order=2, solver_type="bh2"),
                                  dict(k=10, solver_order=2, solver_type="bh1"),
                                  dict(k=10, solver_order=3, solver_type="bh2"),
                                  dict(k=10, solver_order=3, solver_type="bh1"),
                                  dict(k=19, solver_order=3, solver_type="bh1", final_sigmas_type="zero")], ids=str)
def test_step_matches_float64(case):
    """k = 0 (t = 999, first order, no corrector), a middle step with the corrector at orders 2 and 3 under bh1 and bh2,
    and the last step into sigma = 0"""
    f, lib, st = _lib()
    case = dict(case)
    k = case.pop("k")
    s = _sched(**case)
    s.set_timesteps(20)
    R = s.config.solver_order
    row = s.coefficient_table()[k]
    assert (row[2] > 0) == (k > 0) and int(row[3]) == (1 if k in (0, 19) else R)
    g = torch.Generator(device="cuda").manual_seed(k + 7 * R)
    B, per = 5, 1003
    x = torch.randn(B, per, generator=g, device="cuda") * 3
    eps_c, eps_u, last0 = (torch.randn(B, per, generator=g, device="cuda") for _ in range(3))
    hist0 = torch.randn((R, B, per), generator=g, device="cuda")
    worst = [0.0, 0.0, 0.0]
    for clip in (0.0, 3.0):
        for w, u in ((0.0, None), (0.6, eps_u)):
            out = torch.full_like(x, float("nan"))
            last, hist = last0.clone(), hist0.clone()
            f.check(lib.bg_unipc_step(eps_c.data_ptr(), f.ptr(u), w, x.data_ptr(), out.data_ptr(), last.data_ptr(),
                                      hist.data_ptr(), R, per, B * per, row.data_ptr(), clip, st), "bg_unipc_step")
            torch.cuda.synchronize()
            e32 = eps_c                  # the kernel's fp32 CFG combine (two products, one difference) is the input
            if u is not None:
                f32 = lambda v: torch.tensor(v, dtype=torch.float32, device="cuda")
                e32 = eps_c * (f32(1.0) + f32(w)) - u * f32(w)
            (o, xc, x0), (mo, mxc, mx0) = unipc_ref64(row, e32, x, last0, hist0, clip)
            sn = int(row[4])
            untouched = [i for i in range(R) if i != sn]
            assert torch.equal(hist[untouched], hist0[untouched])
            for i, (got, want, mag) in enumerate(((out, o, mo), (last, xc, mxc), (hist[sn], x0, mx0))):
                assert torch.isfinite(got).all()
                err = float(((got.double() - want).abs() / (mag * 2.0 ** -23).clamp_min(1e-30)).max())
                worst[i] = max(worst[i], err)
                assert err <= PARITY_ULP, (clip, w, i, err)
    print(f"UniPC fp64 parity k={k} {case}: out {worst[0]:.2f} ulp, last {worst[1]:.2f} ulp, x0 {worst[2]:.2f} ulp "
          "(of the magnitude sum)")


# ---------------------------------------------------------------------------------------------- forms agree exactly
@pytest.mark.parametrize("cfg_w", [0.0, 0.6])
@pytest.mark.parametrize("per", [7, 13, 1638])
def test_eager_and_table_forms_agree(per, cfg_w):
    f, lib, st = _lib()
    B = 7
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(per)
    eps_u = torch.randn(B, per, generator=g, device="cuda") if cfg_w else None
    s = _sched(solver_order=3, final_sigmas_type="zero", clip_sample=True, clip_sample_range=3)
    s.set_timesteps(7)
    ts = s.timesteps
    coef = s.coefficient_table(ts)
    coef_d = coef.cuda()
    ts_d = ts.cuda()
    step = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    state = {name: (torch.zeros(B, per, device="cuda"), torch.zeros(3, B, per, device="cuda")) for name in ("eager", "tab")}
    for i in range(len(ts)):
        eps_c, x = (torch.randn(B, per, generator=g, device="cuda") * 2 for _ in range(2))
        out = {name: torch.full_like(x, float("nan")) for name in state}
        args = lambda name: (eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), out[name].data_ptr(),
                             state[name][0].data_ptr(), state[name][1].data_ptr())
        f.check(lib.bg_unipc_step(*args("eager"), 3, per, n, coef[i].data_ptr(), 3.0, st), "eager")
        f.check(lib.bg_step_advance(ts_d.data_ptr(), len(ts), step.data_ptr(), t_cur.data_ptr(), st), "advance")
        f.check(lib.bg_unipc_step_tab(*args("tab"), per, n, coef_d.data_ptr(), step.data_ptr(), 3.0, st), "tab")
        torch.cuda.synchronize()
        assert torch.isfinite(out["eager"]).all()
        assert torch.equal(out["eager"], out["tab"]), i
        for j in range(2):
            assert torch.equal(state["eager"][j], state["tab"][j]), (i, j)
    # in place: out aliasing x gives the same result
    x2 = x.clone()
    last, hist = state["eager"][0].clone(), state["eager"][1].clone()
    s.set_timesteps(7)
    row = s.coefficient_table()[3]
    ref = torch.empty_like(x)
    f.check(lib.bg_unipc_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x.data_ptr(), ref.data_ptr(), last.data_ptr(),
                              hist.data_ptr(), 3, per, n, row.data_ptr(), 3.0, st), "ref")
    last, hist = state["eager"][0].clone(), state["eager"][1].clone()
    f.check(lib.bg_unipc_step(eps_c.data_ptr(), f.ptr(eps_u), cfg_w, x2.data_ptr(), x2.data_ptr(), last.data_ptr(),
                              hist.data_ptr(), 3, per, n, row.data_ptr(), 3.0, st), "in place")
    torch.cuda.synchronize()
    assert torch.equal(x2, ref)


# ---------------------------------------------------------------------------------------------------------- cascade
def _cfg(**kw):
    from brepgen_b200.sampler import CascadeConfig
    base = dict(batch_size=2, num_surfaces=4, num_edges=3, class_label=6, schedule="unipc", unipc_steps=4, seed=3,
                decode=False, graph="off")
    base.update(kw)
    return CascadeConfig(**base)


def _init(cfg, seed=9):
    g = torch.Generator().manual_seed(seed)
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    S = S0 if cfg.use_cf else 2 * S0
    return {"surfPos": torch.randn(B, S0, 6, generator=g), "surfZ": torch.randn(B, S, 48, generator=g),
            "edgePos": torch.randn(B, S, E, 6, generator=g), "edgeZV": torch.randn(B, S, E, 18, generator=g)}


# relative L2 bar against the fp32 oracle: the denoisers run in fp16 on the GPU, and UniPC's multistep extrapolation over
# a few large steps amplifies that difference as DPM-Solver++'s second-order steps do, whose bar is 3e-3 (DDIM's
# first-order steps: 2e-3).  Worst measured on an H100: 2.54e-3 (UniPC-4 with CFG, edgePos)
CASCADE_BAR = 3e-3


def _compare(out, ref, label, bar=CASCADE_BAR):
    assert torch.equal(out["surfMask"].cpu(), ref["surfMask"]), label
    assert torch.equal(out["edgeM"].cpu(), ref["edgeM"]), label
    sv, ev = ~ref["surfMask"], ~ref["edgeM"]
    valid = {"surfPos": slice(None), "surfZ": sv, "edgePos": sv, "edge_z": ev, "edgeV": ev}
    for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV"):
        err = rel_l2(out[k].cpu()[valid[k]], ref[k][valid[k]])
        print(f"{label} {k} rel_l2={err:.3e}")
        assert err < bar, (label, k, err)


@pytest.mark.parametrize("order,solver_type", [(2, "bh2"), (3, "bh2"), (2, "bh1")])
@pytest.mark.parametrize("use_cf", [False, True])
@pytest.mark.parametrize("steps", [4, 10])
def test_short_unipc_cascade_matches_oracle(steps, use_cf, order, solver_type):
    from brepgen_b200.sampler import Cascade
    ms, sds = _models(use_cf)
    cfg = _cfg(use_cf=use_cf, unipc_steps=steps, unipc_order=order, unipc_solver_type=solver_type)
    init = _init(cfg)
    ref = run_cascade_unipc(sds, cfg, init)
    out = Cascade(ms).run(cfg, init_noise=init)
    _compare(out, ref, f"unipc cascade steps={steps} cf={use_cf} order={order} {solver_type}")


def _run(cfg, ms=None, known=None):
    from brepgen_b200.sampler import Cascade
    casc = Cascade(ms if ms is not None else _models(cfg.use_cf)[0])
    out = casc.run(cfg, known=known)
    torch.cuda.synchronize()
    return out, casc


@pytest.mark.parametrize("noise", ["batch", "per_sample"])
@pytest.mark.parametrize("order", [2, 3])
def test_graph_on_equals_graph_off(order, noise):
    """12 steps: the surface-position loop crosses the late face increase, so its graph has two segments and the second
    restarts the solver with new buffers"""
    for use_cf in (False, True):
        kw = dict(batch_size=3, num_surfaces=5, num_edges=6, use_cf=use_cf, unipc_steps=12, unipc_order=order,
                  noise=noise)
        a, _ = _run(_cfg(graph="off", **kw))
        b, casc = _run(_cfg(graph="on", **kw))
        assert casc.last_graph_steps == 4 * 12
        for k in a:
            assert torch.equal(a[k], b[k]), (order, noise, use_cf, k)


@pytest.mark.parametrize("graph", ["off", "on"])
def test_per_sample_unipc_cascade_equals_samples_run_alone(graph):
    kw = dict(num_surfaces=5, num_edges=6, use_cf=False, unipc_steps=12, unipc_order=3, noise="per_sample", seed=21,
              graph=graph)
    full, _ = _run(_cfg(batch_size=5, **kw))
    for b in range(5):
        one, _ = _run(_cfg(batch_size=1, sample_base=b, **kw))
        for k in full:
            assert torch.equal(full[k][b], one[k][0]), (graph, b, k)
    assert not torch.equal(full["surfPos"][0], full["surfPos"][1])


@pytest.mark.parametrize("use_cf", [False, True])
def test_forward_counts_and_late_face_increase(use_cf):
    """4 N network evaluations per cascade (the corrector adds none), and the face slots doubled once"""
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
        out, _ = _run(_cfg(num_surfaces=3, num_edges=2, unipc_steps=N, use_cf=use_cf), ms)
        evaluations = sum(rows // B for v in calls.values() for _, rows, _ in v)
        assert evaluations == (8 * N if use_cf else 4 * N)
        ts = [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]
        assert [(t, s) for t, _, s in calls["surfpos"]] == [(t, 3 if (use_cf or t > 249) else 6) for t in ts]
        calls.clear()
        out_g, casc = _run(_cfg(num_surfaces=3, num_edges=2, unipc_steps=N, use_cf=use_cf, graph="on"), ms)
        assert casc.last_graph_steps == 4 * N
        for k in out:
            assert torch.equal(out[k], out_g[k]), k
    finally:
        for m in ms.values():
            del m.forward


# ------------------------------------------------------------------------------------------------------- completion
@pytest.mark.parametrize("graph", ["off", "on"])
def test_completion_with_unipc(graph):
    from brepgen_b200.sampler import Completion
    kw = dict(batch_size=3, num_surfaces=5, num_edges=4, use_cf=False, unipc_steps=12, unipc_order=3, graph=graph)
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
    from brepgen_b200.sampler import Cascade, Completion
    ms, sds = _models(False)
    cfg = _cfg(unipc_steps=10)
    a = run_cascade_unipc(sds, cfg, _init(cfg, 9))
    known = Completion.from_outputs(a, _n_faces(a, [1, 2]))
    init_b = _init(cfg, 10)
    g = torch.Generator().manual_seed(11)
    rbank = {}

    def rnoise(name, k, shape):
        key = (name, k, tuple(shape))
        if key not in rbank:
            rbank[key] = torch.randn(tuple(shape), generator=g)
        return rbank[key]
    ref = run_cascade_unipc(sds, cfg, init_b, known=known, replace_noise=rnoise)
    out = Cascade(ms).run(cfg, init_noise=init_b, known=known, replace_noise=rnoise)
    _compare(out, ref, "unipc completion")
    for i, nf in enumerate(known.n_faces):
        for fk, ok in KNOWN_FIELDS:
            assert torch.equal(out[ok][i, :nf].cpu(), getattr(known, fk)[i, :nf].cpu()), (i, fk)


# ------------------------------------------------------------------------------------------------------- variations
@pytest.mark.parametrize("use_cf", [False, True])
def test_variation_matches_oracle(use_cf):
    from brepgen_b200.sampler import Cascade
    ms, sds = _models(use_cf)
    cfg = _cfg(use_cf=use_cf, unipc_steps=10)
    a, _ = _run(cfg)
    src = _fit(a, cfg, (2, 4))
    for st in ((0.5,) * 4, (0, 0, 0.5, 0.5)):
        init = _start_noise(cfg, st, seed=5)
        ref = run_cascade_variation_unipc(sds, cfg, _var(src, st), init)
        out = Cascade(ms).run(cfg, init_noise=init, source=_var(src, st))
        torch.cuda.synchronize()
        _compare(out, ref, f"unipc variation s={st} cf={use_cf}")
        if st[0] == 0:
            for k in ("surfPos", "surfMask", "surfZ"):
                assert torch.equal(out[k], src[k]), k


# ----------------------------------------------------------------------------------------------------------- errors
def test_bad_arguments_are_rejected_and_launch_nothing():
    f, lib, st = _lib()
    B, per = 3, 8
    n = B * per
    eps, x = torch.randn(B, per, device="cuda"), torch.randn(B, per, device="cuda")
    hist, last = torch.zeros(3, B, per, device="cuda"), torch.zeros(B, per, device="cuda")
    out = torch.full((B, per), float("nan"), device="cuda")
    s = _sched(solver_order=3)
    s.set_timesteps(10)
    tab = s.coefficient_table()
    good = tab[5].clone()
    assert good[2] == 3 and good[3] == 3
    coef_d = tab.cuda()
    step = torch.zeros(1, dtype=torch.int32, device="cuda")

    def row(**kv):
        r = good.clone()
        for i, v in kv.items():
            r[int(i[1:])] = v
        return r

    def eager(eps_p=eps.data_ptr(), x_p=x.data_ptr(), out_p=out.data_ptr(), l_p=last.data_ptr(), h_p=hist.data_ptr(),
              slots=3, per_s=per, nn=n, r=good):
        return lib.bg_unipc_step(eps_p, None, 0.0, x_p, out_p, l_p, h_p, slots, per_s, nn, r.data_ptr() if r is not None
                                 else None, 3.0, st)

    def tab_(eps_p=eps.data_ptr(), x_p=x.data_ptr(), out_p=out.data_ptr(), l_p=last.data_ptr(), h_p=hist.data_ptr(),
             per_s=per, nn=n, cf=coef_d.data_ptr(), sp=step.data_ptr()):
        return lib.bg_unipc_step_tab(eps_p, None, 0.0, x_p, out_p, l_p, h_p, per_s, nn, cf, sp, 3.0, st)
    cases = [
        ("eager NULL eps", lambda: eager(eps_p=None)), ("eager NULL x", lambda: eager(x_p=None)),
        ("eager NULL out", lambda: eager(out_p=None)), ("eager NULL hist", lambda: eager(h_p=None)),
        ("eager NULL row", lambda: eager(r=None)), ("eager corrector without last", lambda: eager(l_p=None)),
        ("eager n 0", lambda: eager(nn=0)), ("eager per_sample 0", lambda: eager(per_s=0)),
        ("eager n % per_sample", lambda: eager(per_s=5)), ("eager n_slots 0", lambda: eager(slots=0)),
        ("eager n_slots 4", lambda: eager(slots=4)), ("eager alpha_s 0", lambda: eager(r=row(r0=0.0))),
        ("eager alpha_s < 0", lambda: eager(r=row(r0=-0.5))), ("eager corrector order 4", lambda: eager(r=row(r2=4.0))),
        ("eager corrector order -1", lambda: eager(r=row(r2=-1.0))), ("eager order 0", lambda: eager(r=row(r3=0.0))),
        ("eager order 4", lambda: eager(r=row(r3=4.0))), ("eager order 1.5", lambda: eager(r=row(r3=1.5))),
        ("eager slot_new out of ring", lambda: eager(r=row(r4=3.0))), ("eager slot read out of ring", lambda: eager(r=row(r7=5.0))),
        ("eager slot < 0", lambda: eager(r=row(r5=-1.0))), ("eager slot past the 2-slot ring", lambda: eager(slots=2)),
        ("tab NULL eps", lambda: tab_(eps_p=None)), ("tab NULL out", lambda: tab_(out_p=None)),
        ("tab NULL last", lambda: tab_(l_p=None)), ("tab NULL hist", lambda: tab_(h_p=None)),
        ("tab NULL coef", lambda: tab_(cf=None)), ("tab NULL step", lambda: tab_(sp=None)),
        ("tab per_sample 0", lambda: tab_(per_s=0)), ("tab n % per_sample", lambda: tab_(per_s=7)),
        ("tab n 0", lambda: tab_(nn=0)),
    ]
    l0 = lib.bg_launch_count()
    for name, call in cases:
        assert call() == -1, name               # BG_STATUS_BAD_ARG
        assert lib.bg_last_error(), name
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0
    assert torch.isnan(out).all() and (hist == 0).all() and (last == 0).all()
    # valid calls launch: the row, the table form, and a first step without a corrector and without last
    first = tab[0].clone()
    assert first[2] == 0
    assert eager() == 0 and tab_() == 0 and eager(l_p=None, r=first, slots=1) == 0
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0 + 3
