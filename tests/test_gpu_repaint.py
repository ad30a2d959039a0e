"""GPU tests of RePaint resampling: the step and undo kernels (bg_repaint_step / _tab, bg_repaint_undo / _tab), the
RePaintScheduler drop-in and CascadeConfig(schedule="repaint").

  * every step output element against a float64 evaluation; unknown elements bit-identical to bg_ddim_step for the same
    noise; the last step ends on the known values bit for bit, signed zeros included;
  * the undo with explicit noise is the fp32 oracle chain bit for bit;
  * keyed normals are bg_randn_keyed's (domain 3 at counter k, domain 4 at k * n + i); the eager, table, keyed, batch and
    explicit forms agree;
  * without resampling the cascade is the DDIM cascade bit for bit; short completions against oracle.repaint;
  * graph on = graph off, a sample does not depend on its batch, forward counts and the late face increase;
  * argument errors launch nothing.
Without trained weights these tests pin the arithmetic and the invariants, not whether resampling improves a completion.
"""
import numpy as np
import pytest
import torch

from test_gpu_completion import KNOWN_FIELDS, _models, _n_faces

pytestmark = pytest.mark.gpu


def _lib():
    from brepgen_b200 import _ffi as f
    return f, f.lib(), f.current_stream()


def _keys(seeds, stage):
    from brepgen_b200.schedulers import sample_keys
    return torch.from_numpy(sample_keys(seeds, stage).view(np.int64)).cuda()


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _step(out, eps_c, eps_u, w, x, known, m, per_token, noise, seed, keys, per, k, coefs, clip):
    f, lib, st = _lib()
    f.check(lib.bg_repaint_step(eps_c.data_ptr(), f.ptr(eps_u), w, x.data_ptr(), out.data_ptr(), f.ptr(known), f.ptr(m),
                                per_token, f.ptr(noise), seed, f.ptr(keys), per, k, x.numel(), *coefs, clip, st),
            "bg_repaint_step")


def _ddim(out, eps_c, eps_u, w, x, noise, coefs, clip):
    f, lib, st = _lib()
    f.check(lib.bg_ddim_step(eps_c.data_ptr(), f.ptr(eps_u), w, x.data_ptr(), out.data_ptr(), f.ptr(noise), 0, 0, None, 0,
                             0, x.numel(), *coefs[:5], clip, 0, st), "bg_ddim_step")


def _mask(kind, B, T, g):
    if kind == "empty":
        return torch.zeros(B, T, dtype=torch.uint8, device="cuda")
    if kind == "full":
        return torch.ones(B, T, dtype=torch.uint8, device="cuda")
    return (torch.rand(B, T, generator=g, device="cuda") < 0.4).to(torch.uint8)


# ---------------------------------------------------------------------------------------------------- fp64 parity
PARITY_BAR = 5e-7     # max |out - ref64| / max(1, max |ref64|), as the DDIM step's bar (its ops plus one fmaf)


@pytest.mark.parametrize("mask_kind", ["random", "empty", "full"])
@pytest.mark.parametrize("eta", [0.0, 0.8])
@pytest.mark.parametrize("per_token,tokens", [(6, 7), (18, 13), (48, 101)])
def test_step_matches_float64_and_ddim(per_token, tokens, eta, mask_kind):
    from brepgen_b200.schedulers import RePaintScheduler
    g = torch.Generator(device="cuda").manual_seed(per_token * 1000 + tokens)
    B = 3
    per = per_token * tokens
    x = torch.randn(B, per, generator=g, device="cuda") * 3
    eps_c, eps_u, known, nz = (torch.randn(B, per, generator=g, device="cuda") for _ in range(4))
    m = _mask(mask_kind, B, tokens, g)
    sel = m.bool().repeat_interleave(per_token, 1)
    s = RePaintScheduler(eta=eta)
    s.set_timesteps(10, 2, 3)
    worst = 0.0
    for t in (900, 500, 0):
        coefs = s.step_coefficients(t)
        sb, sa, sa_prev, c_dir, sigma, sb_prev = coefs
        for w, u in ((0.0, None), (0.6, eps_u)):
            out, ref_d = (torch.full_like(x, float("nan")) for _ in range(2))
            _step(out, eps_c, u, w, x, known, m, per_token, nz, 0, None, per, 5, coefs, 3.0)
            _ddim(ref_d, eps_c, u, w, x, nz, coefs, 3.0)
            torch.cuda.synchronize()
            e = eps_c.double()
            if u is not None:
                e = e * (1 + float(np.float32(w))) - u.double() * float(np.float32(w))
            x0 = ((x.double() - sb * e) / sa).clamp(-3, 3)
            unk = sa_prev * x0 + c_dir * e + sigma * nz.double()
            kn = sa_prev * known.double() + sb_prev * nz.double()
            ref = torch.where(sel, kn, unk)
            err = float((out.double() - ref).abs().max() / max(1.0, float(ref.abs().max())))
            worst = max(worst, err)
            assert err < PARITY_BAR, (t, w, err)
            assert torch.equal(out[~sel].view(torch.int32), ref_d[~sel].view(torch.int32)), (t, w)   # DDIM bit for bit
            if t == 0:
                assert torch.equal(out[sel].view(torch.int32), known[sel].view(torch.int32))
    print(f"repaint step fp64 per_token={per_token} tokens={tokens} eta={eta} {mask_kind}: worst {worst:.3e}")


def test_last_step_ends_on_known_signed_zeros():
    from brepgen_b200.schedulers import RePaintScheduler
    s = RePaintScheduler(eta=1.0, clip_sample_range=3.0)
    s.set_timesteps(10, 2, 3)
    x = torch.randn(2, 4, 6, device="cuda")
    known = torch.randn(2, 4, 6, device="cuda")
    known[:, :, ::2] = -0.0
    known[:, :, 1::4] = 0.0
    mask = torch.ones(2, 4, dtype=torch.bool, device="cuda")
    mask[1, 3] = False
    out = s.step(torch.randn_like(x), 0, x, known, mask).prev_sample
    torch.cuda.synchronize()
    assert torch.equal(out[mask].view(torch.int32), known[mask].view(torch.int32))


# --------------------------------------------------------------------------------------------------------- undo
@pytest.mark.parametrize("N,t_last", [(50, 300), (250, 0), (250, 988), (20, 450)])
def test_undo_is_the_fp32_chain_bit_for_bit(N, t_last):
    from brepgen_b200.schedulers import RePaintScheduler
    from oracle.repaint import RePaintOracle
    s, o = RePaintScheduler(), RePaintOracle()
    s.set_timesteps(N)
    o.set_timesteps(N)
    n = s.undo_transitions
    g = torch.Generator().manual_seed(N + t_last)
    x = torch.randn(3, 37, 18, generator=g) * 2
    nz = torch.randn((n,) + tuple(x.shape), generator=g)
    got = s.undo_step(x.cuda(), t_last, noise=nz.cuda())
    torch.cuda.synchronize()
    want = o.undo_step(x, t_last, nz)
    assert torch.equal(got.cpu().view(torch.int32), want.view(torch.int32))


# ------------------------------------------------------------------------------------------------- noise forms
@pytest.mark.parametrize("per_token,tokens", [(6, 7), (18, 13)])
def test_noise_forms_agree(per_token, tokens):
    """keyed step normals = bg_randn_keyed(domain 3, k); keyed undo normals = bg_randn_keyed(domain 4, k * n + i); the
    batch key is one sample over the whole tensor; the table forms, advanced over the whole list, equal the eager forms"""
    from brepgen_b200.sampler import randn_keyed
    from brepgen_b200.schedulers import RePaintScheduler, repaint_entries
    f, lib, st = _lib()
    B = 5
    per = per_token * tokens
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(tokens)
    x, eps, known = (torch.randn(B, per, generator=g, device="cuda") for _ in range(3))
    m = (torch.rand(B, tokens, generator=g, device="cuda") < 0.5).to(torch.uint8)
    seeds = [11, 12, 13, 14, 15]
    keys = _keys(seeds, 3)
    seed = 0x0123456789ABCDEF
    kb = torch.from_numpy(np.array([seed], dtype=np.uint64).view(np.int64)).cuda()
    s = RePaintScheduler(eta=0.5, clip_sample_range=3.0)
    s.set_timesteps(10, 2, 2)
    ents = repaint_entries(s.timesteps)
    nt = s.undo_transitions
    coef, utab = s.coefficient_table().cuda(), s.undo_table().cuda()
    ts_d = s.timesteps.cuda()
    step = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    for k, (is_step, t) in enumerate(ents):
        f.check(lib.bg_step_advance(ts_d.data_ptr(), len(ents), step.data_ptr(), t_cur.data_ptr(), st), "advance")
        outs = {key: x.clone() for key in ("keyed", "fed", "batch", "fed_b", "tab", "tab_b")}
        if is_step:
            coefs = s.step_coefficients(t)
            z = randn_keyed(seeds, 3, (B, per), "cuda", domain=3, t=k)
            zb = torch.empty(n, device="cuda")
            f.check(lib.bg_randn_keyed(kb.data_ptr(), 1, n, 3, k, zb.data_ptr(), st), "randn batch key")
            args = (eps, None, 0.0, x, known, m, per_token)
            _step(outs["keyed"], *args, None, 0, keys, per, k, coefs, 3.0)
            _step(outs["fed"], *args, z, 0, None, per, k, coefs, 3.0)
            _step(outs["batch"], *args, None, seed, None, 0, k, coefs, 3.0)
            _step(outs["fed_b"], *args, zb, 0, None, 0, k, coefs, 3.0)
            for name, sd, kk in (("tab", 0, keys), ("tab_b", seed, None)):
                f.check(lib.bg_repaint_step_tab(eps.data_ptr(), None, 0.0, x.data_ptr(), outs[name].data_ptr(),
                                                known.data_ptr(), m.data_ptr(), per_token, sd, f.ptr(kk), per, n,
                                                coef.data_ptr(), step.data_ptr(), 3.0, st), "step tab")
        else:
            cf = s.undo_coefficients(t).cuda()
            z = torch.stack([randn_keyed(seeds, 3, (B, per), "cuda", domain=4, t=k * nt + i) for i in range(nt)])
            zb = torch.empty(nt, n, device="cuda")
            for i in range(nt):
                f.check(lib.bg_randn_keyed(kb.data_ptr(), 1, n, 4, k * nt + i, zb[i].data_ptr(), st), "randn batch")
            for name, nz, sd, kk in (("keyed", None, 0, keys), ("fed", z, 0, None), ("batch", None, seed, None),
                                     ("fed_b", zb, 0, None)):
                f.check(lib.bg_repaint_undo(outs[name].data_ptr(), n, nt, cf.data_ptr(), f.ptr(nz), sd, f.ptr(kk), per, k,
                                            st), "undo")
            for name, sd, kk in (("tab", 0, keys), ("tab_b", seed, None)):
                f.check(lib.bg_repaint_undo_tab(outs[name].data_ptr(), n, nt, sd, f.ptr(kk), per, utab.data_ptr(),
                                                step.data_ptr(), st), "undo tab")
        torch.cuda.synchronize()
        assert torch.equal(outs["keyed"], outs["fed"]), k
        assert torch.equal(outs["batch"], outs["fed_b"]), k
        assert torch.equal(outs["tab"], outs["keyed"]), k
        assert torch.equal(outs["tab_b"], outs["batch"]), k
        if not (is_step and t == 0):         # the last step draws nothing: sigma = 0 and the known part is exact
            assert not torch.equal(outs["keyed"], outs["batch"]), k
    z3 = randn_keyed(seeds, 3, (B, per), "cuda", domain=3, t=7)
    assert float((z3 - randn_keyed(seeds, 3, (B, per), "cuda", domain=0, t=7)).abs().max()) > 1.0


# ---------------------------------------------------------------------------------------------------------- cascade
def _cfg(**kw):
    from brepgen_b200.sampler import CascadeConfig
    base = dict(batch_size=2, num_surfaces=4, num_edges=3, class_label=6, schedule="repaint", repaint_steps=10,
                repaint_jump_length=2, repaint_jump_n_sample=3, repaint_eta=0.5, seed=3, decode=False, graph="off")
    base.update(kw)
    return CascadeConfig(**base)


def _run(cfg, known=None, ms=None):
    from brepgen_b200.sampler import Cascade
    casc = Cascade(ms if ms is not None else _models(cfg.use_cf)[0])
    out = casc.run(cfg, known=known)
    torch.cuda.synchronize()
    return out, casc


@pytest.mark.parametrize("graph", ["off", "on"])
@pytest.mark.parametrize("noise", ["batch", "per_sample"])
def test_without_resampling_is_the_ddim_cascade(noise, graph):
    for use_cf in (False, True):
        kw = dict(batch_size=3, num_surfaces=5, num_edges=4, use_cf=use_cf, noise=noise, graph=graph)
        a, _ = _run(_cfg(repaint_steps=12, repaint_jump_n_sample=1, repaint_eta=0.0, **kw))
        b, _ = _run(_cfg(schedule="ddim", ddim_steps=12, **kw))
        assert set(a) == set(b)
        for k in a:
            assert torch.equal(a[k], b[k]), (use_cf, k)


def _known_source(cfg, sds):
    from brepgen_b200.sampler import Completion
    from oracle.repaint import run_cascade_repaint
    g = torch.Generator().manual_seed(9)
    S = cfg.num_surfaces if cfg.use_cf else 2 * cfg.num_surfaces
    init = {"surfPos": torch.randn(2, cfg.num_surfaces, 6, generator=g), "surfZ": torch.randn(2, S, 48, generator=g),
            "edgePos": torch.randn(2, S, 3, 6, generator=g), "edgeZV": torch.randn(2, S, 3, 18, generator=g)}
    nz = lambda name, k, shape: torch.randn(tuple(shape), generator=g)
    a = run_cascade_repaint(sds, _cfg(use_cf=cfg.use_cf, repaint_steps=4, repaint_jump_n_sample=1), init, nz, nz)
    return Completion.from_outputs(a, _n_faces(a, [1, 2]))


@pytest.mark.parametrize("use_cf", [False, True])
@pytest.mark.parametrize("steps,jn,eta", [(4, 2, 0.0), (4, 3, 1.0), (10, 2, 1.0), (10, 3, 0.0)])
def test_short_completion_matches_oracle(steps, jn, eta, use_cf):
    from brepgen_b200.sampler import Cascade
    from oracle.repaint import run_cascade_repaint
    ms, sds = _models(use_cf)
    cfg = _cfg(use_cf=use_cf, repaint_steps=steps, repaint_jump_n_sample=jn, repaint_eta=eta)
    known = _known_source(cfg, sds)
    assert sum(known.n_faces) >= 2
    S = cfg.num_surfaces if use_cf else 2 * cfg.num_surfaces
    g = torch.Generator().manual_seed(19)
    init = {"surfPos": torch.randn(2, cfg.num_surfaces, 6, generator=g), "surfZ": torch.randn(2, S, 48, generator=g),
            "edgePos": torch.randn(2, S, 3, 6, generator=g), "edgeZV": torch.randn(2, S, 3, 18, generator=g)}
    banks = ({}, {})

    def bank(i):
        def f(name, k, shape):
            key = (name, k, tuple(shape))
            if key not in banks[i]:
                banks[i][key] = torch.randn(tuple(shape), generator=g)
            return banks[i][key]
        return f
    ref = run_cascade_repaint(sds, cfg, init, bank(0), bank(1), known=known)
    sizes = (len(banks[0]), len(banks[1]))
    out = Cascade(ms).run(cfg, init_noise=init, step_noise=bank(0), undo_noise=bank(1), known=known)
    assert (len(banks[0]), len(banks[1])) == sizes and sizes[1] > 0      # the same draws on both sides
    assert torch.equal(out["surfMask"].cpu(), ref["surfMask"])
    assert torch.equal(out["edgeM"].cpu(), ref["edgeM"])
    sv, ev = ~ref["surfMask"], ~ref["edgeM"]
    valid = {"surfPos": slice(None), "surfZ": sv, "edgePos": sv, "edge_z": ev, "edgeV": ev}
    for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV"):
        err = rel_l2(out[k].cpu()[valid[k]], ref[k][valid[k]])
        print(f"repaint completion N={steps} jn={jn} eta={eta} cf={use_cf} {k} rel_l2={err:.3e}")
        assert err < 2e-3, (k, err)
    for i, nf in enumerate(known.n_faces):
        for fk, ok in KNOWN_FIELDS:
            assert torch.equal(out[ok][i, :nf].cpu(), getattr(known, fk)[i, :nf]), (i, fk)


@pytest.mark.parametrize("noise", ["batch", "per_sample"])
def test_graph_on_equals_graph_off(noise):
    """N = 10, jump 2 x 3: the surface-position list crosses the late face increase and jumps back above 249, so its
    graphs come in two segments"""
    from brepgen_b200.sampler import Completion
    from brepgen_b200.schedulers import repaint_timesteps
    L = len(repaint_timesteps(10, 2, 3))
    for use_cf in (False, True):
        kw = dict(batch_size=3, num_surfaces=5, num_edges=4, use_cf=use_cf, noise=noise)
        src, _ = _run(_cfg(seed=7, **kw))
        known = Completion.from_outputs(src, _n_faces(src, [2, 0, 3]))
        a, _ = _run(_cfg(graph="off", **kw), known=known)
        b, casc = _run(_cfg(graph="on", **kw), known=known)
        assert casc.last_graph_steps == 4 * L
        for k in a:
            assert torch.equal(a[k], b[k]), (use_cf, k)
        plain, _ = _run(_cfg(graph="off", **kw))
        assert not torch.equal(a["surfPos"], plain["surfPos"])
        for i, nf in enumerate(known.n_faces):
            for fk, ok in KNOWN_FIELDS:
                assert torch.equal(a[ok][i, :nf].cpu(), getattr(known, fk)[i, :nf].cpu()), (i, fk)


@pytest.mark.parametrize("graph", ["off", "on"])
def test_sample_does_not_depend_on_its_batch(graph):
    from brepgen_b200.sampler import Completion
    kw = dict(num_surfaces=5, num_edges=4, use_cf=False, noise="per_sample", seed=21, graph=graph)
    src, _ = _run(_cfg(batch_size=5, **dict(kw, seed=4)))
    known = Completion.from_outputs(src, _n_faces(src, [0, 1, 2, 3, 4]))
    full, _ = _run(_cfg(batch_size=5, **kw), known=known)
    for b in range(5):
        one_known = Completion(n_faces=[known.n_faces[b]], **{f: getattr(known, f)[b:b + 1] for f, _ in KNOWN_FIELDS})
        one, _ = _run(_cfg(batch_size=1, sample_base=b, **kw), known=one_known)
        for k in full:
            assert torch.equal(full[k][b], one[k][0]), (graph, b, k)


@pytest.mark.parametrize("use_cf", [False, True])
def test_forward_counts_and_late_face_increase(use_cf):
    from brepgen_b200.schedulers import repaint_entries, repaint_timesteps
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
        B = 2
        step_ts = [t for s, t in repaint_entries(repaint_timesteps(10, 2, 3)) if s]
        out, _ = _run(_cfg(num_surfaces=3, num_edges=2, use_cf=use_cf), ms=ms)
        for kind, v in calls.items():
            assert [t for t, _, _ in v] == step_ts, kind
            assert all(rows == (2 * B if use_cf else B) for _, rows, _ in v)
        first = next(i for i, t in enumerate(step_ts) if t <= 249)
        assert max(step_ts[first:]) > 249
        want = [3] * len(step_ts) if use_cf else [3] * first + [6] * (len(step_ts) - first)
        assert [s for _, _, s in calls["surfpos"]] == want
        calls.clear()
        out_g, casc = _run(_cfg(num_surfaces=3, num_edges=2, use_cf=use_cf, graph="on"), ms=ms)
        assert len(calls["surfpos"]) == (2 if use_cf else 4)     # warm-up + capture of the step body per segment
        for k in out:
            assert torch.equal(out[k], out_g[k]), k
    finally:
        for m in ms.values():
            del m.forward


# ----------------------------------------------------------------------------------------------------------- errors
def test_bad_arguments_are_rejected_and_launch_nothing():
    f, lib, st = _lib()
    B, per_token, tokens = 3, 6, 4
    per = per_token * tokens
    n = B * per
    x = torch.full((B, per), float("nan"), device="cuda")
    e, known = torch.zeros(B, per, device="cuda"), torch.zeros(B, per, device="cuda")
    m = torch.ones(B, tokens, dtype=torch.uint8, device="cuda")
    k = _keys([1, 2, 3], 0)
    coef = torch.ones(1, 6, device="cuda")
    ucoef = torch.ones(4, 2, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    cf = (0.5, 0.5, 0.5, 0.5, 0.0, 0.5)

    def eager(e_p=e.data_ptr(), x_p=x.data_ptr(), o_p=x.data_ptr(), kn=known.data_ptr(), m_p=m.data_ptr(), pt=per_token,
              keys=k.data_ptr(), ps=per, kk=5, nn=n, sa=0.5):
        return lib.bg_repaint_step(e_p, None, 0.0, x_p, o_p, kn, m_p, pt, None, 1, keys, ps, kk, nn, 0.5, sa,
                                   *cf[2:], 3.0, st)

    def tab(e_p=e.data_ptr(), x_p=x.data_ptr(), kn=known.data_ptr(), m_p=m.data_ptr(), pt=per_token, keys=k.data_ptr(),
            ps=per, nn=n, c=coef.data_ptr(), sp=step.data_ptr()):
        return lib.bg_repaint_step_tab(e_p, None, 0.0, x_p, x_p, kn, m_p, pt, 1, keys, ps, nn, c, sp, 3.0, st)

    def undo(x_p=x.data_ptr(), nn=n, nt=4, c=ucoef.data_ptr(), keys=k.data_ptr(), ps=per, kk=5):
        return lib.bg_repaint_undo(x_p, nn, nt, c, None, 1, keys, ps, kk, st)

    def undo_tab(x_p=x.data_ptr(), nn=n, nt=4, keys=k.data_ptr(), ps=per, c=ucoef.data_ptr(), sp=step.data_ptr()):
        return lib.bg_repaint_undo_tab(x_p, nn, nt, 1, keys, ps, c, sp, st)
    cases = [
        ("step NULL eps", lambda: eager(e_p=None)), ("step NULL x", lambda: eager(x_p=None)),
        ("step NULL out", lambda: eager(o_p=None)), ("step n 0", lambda: eager(nn=0)),
        ("step known without mask", lambda: eager(m_p=None)), ("step mask without known", lambda: eager(kn=None)),
        ("step per_token 0", lambda: eager(pt=0)), ("step n % per_token", lambda: eager(pt=7)),
        ("step per_sample 0", lambda: eager(ps=0)), ("step per_sample % per_token", lambda: eager(ps=8)),
        ("step per_sample not dividing n", lambda: eager(ps=2 * per)), ("step k < 0", lambda: eager(kk=-1)),
        ("step k > 32 bits", lambda: eager(kk=2 ** 32)), ("step sqrt_abar 0", lambda: eager(sa=0.0)),
        ("tab NULL eps", lambda: tab(e_p=None)), ("tab NULL x", lambda: tab(x_p=None)),
        ("tab NULL coef", lambda: tab(c=None)), ("tab NULL step", lambda: tab(sp=None)),
        ("tab known without mask", lambda: tab(m_p=None)), ("tab n % per_token", lambda: tab(pt=5)),
        ("tab per_sample % per_token", lambda: tab(ps=8)), ("tab n 0", lambda: tab(nn=0)),
        ("undo NULL x", lambda: undo(x_p=None)), ("undo NULL coef", lambda: undo(c=None)),
        ("undo n 0", lambda: undo(nn=0)), ("undo n_trans 0", lambda: undo(nt=0)),
        ("undo per_sample 0", lambda: undo(ps=0)), ("undo per_sample not dividing n", lambda: undo(ps=7)),
        ("undo k < 0", lambda: undo(kk=-1)), ("undo counter > 32 bits", lambda: undo(kk=2 ** 30)),
        ("undo tab NULL x", lambda: undo_tab(x_p=None)), ("undo tab NULL coef", lambda: undo_tab(c=None)),
        ("undo tab NULL step", lambda: undo_tab(sp=None)), ("undo tab n_trans 0", lambda: undo_tab(nt=0)),
        ("undo tab per_sample not dividing n", lambda: undo_tab(ps=7)),
    ]
    l0 = lib.bg_launch_count()
    for name, call in cases:
        assert call() == -1, name               # BG_STATUS_BAD_ARG
        assert lib.bg_last_error(), name
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0
    assert torch.isnan(x).all()
    # the same calls with valid arguments launch (the batch forms ignore per_sample; nothing known needs no per_token)
    assert eager(kk=2 ** 32 - 1) == 0 and eager(keys=None, ps=0) == 0 and eager(kn=None, m_p=None, pt=0) == 0
    assert tab(keys=None, ps=0) == 0 and undo(kk=2 ** 30 - 1) == 0 and undo_tab(keys=None, ps=0) == 0
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0 + 6
