"""GPU tests of B-rep completion: the replacement kernel (bg_replace_known, bg_replace_known_tab), the schedulers'
replace_known and Cascade.run(known=...).

  * every replaced element against a float64 evaluation, every other element untouched;
  * the explicit, keyed, batch-key and table forms agree bit for bit, and draw domain-2 normals;
  * short completed cascades against oracle.completion.run_cascade_completion;
  * round trip: the known parts of a completed run are those of the run they came from, bit for bit;
  * nothing known is a plain run, graph on is graph off, a sample does not depend on its batch;
  * argument errors launch nothing.
"""
import numpy as np
import pytest
import torch

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


# ---------------------------------------------------------------------------------------------------- fp64 parity
PARITY_BAR = 1.2e-7   # |out - ref64| / (|sa known| + |sb z|): fmaf(sa, known, sb*z) rounds twice, <= 2^-23


def _mask(kind, B, T, g):
    if kind == "empty":
        return torch.zeros(B, T, dtype=torch.uint8, device="cuda")
    if kind == "full":
        return torch.ones(B, T, dtype=torch.uint8, device="cuda")
    return (torch.rand(B, T, generator=g, device="cuda") < 0.4).to(torch.uint8)


@pytest.mark.parametrize("mask_kind", ["random", "empty", "full"])
@pytest.mark.parametrize("tokens", [7, 13, 1638])
@pytest.mark.parametrize("per_token", [6, 48, 18])
def test_kernel_matches_float64(per_token, tokens, mask_kind):
    f, lib, st = _lib()
    B = 3
    per = tokens * per_token
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(per_token * 10_000 + tokens)
    x, known, nz = (torch.randn(B, per, generator=g, device="cuda") * 2 for _ in range(3))
    m = _mask(mask_kind, B, tokens, g)
    sel = m.bool().repeat_interleave(per_token, 1)
    k = _keys([5, 6, 7], 2)
    worst = 0.0
    for sa, sb in ((0.3, 0.95), (0.999, 0.04), (1.0, 0.0)):
        for keyed in (False, True):
            out = x.clone()
            f.check(lib.bg_replace_known(out.data_ptr(), known.data_ptr(), m.data_ptr(), n, per_token,
                                         None if keyed else nz.data_ptr(), 0, k.data_ptr() if keyed else None, per, 321,
                                         sa, sb, st), "bg_replace_known")
            z = nz
            if keyed:
                from brepgen_b200.sampler import randn_keyed
                z = randn_keyed([5, 6, 7], 2, (B, per), "cuda", domain=2, t=321)
            torch.cuda.synchronize()
            a, b = float(np.float32(sa)), float(np.float32(sb))
            ref = a * known.double() + b * z.double()
            scale = (a * known.double()).abs() + (b * z.double()).abs()
            err = ((out.double() - ref).abs() / scale.clamp_min(1e-30))[sel]
            if err.numel():
                worst = max(worst, float(err.max()))
                assert float(err.max()) <= PARITY_BAR, (sa, sb, keyed, float(err.max()))
            assert torch.equal(out[~sel].view(torch.int32), x[~sel].view(torch.int32))   # untouched, bit for bit
            if sb == 0.0:
                assert torch.equal(out[sel], known[sel])
    print(f"replace fp64 per_token={per_token} tokens={tokens} {mask_kind}: worst {worst:.3e}")


def test_known_signed_zero_survives_the_last_step():
    f, lib, st = _lib()
    x = torch.ones(1, 12, device="cuda")
    known = torch.full((1, 12), -0.0, device="cuda")
    m = torch.ones(1, 2, dtype=torch.uint8, device="cuda")
    f.check(lib.bg_replace_known(x.data_ptr(), known.data_ptr(), m.data_ptr(), 12, 6, None, 99, None, 0, 0, 1.0, 0.0, st),
            "bg_replace_known")
    torch.cuda.synchronize()
    assert torch.equal(x.view(torch.int32), known.view(torch.int32))


# ------------------------------------------------------------------------------------------------ noise forms agree
@pytest.mark.parametrize("per_token,tokens", [(6, 7), (18, 13), (48, 1638)])
def test_noise_forms_agree(per_token, tokens):
    from brepgen_b200.sampler import randn_keyed
    from brepgen_b200.schedulers import DDIMScheduler
    f, lib, st = _lib()
    B = 5
    per = tokens * per_token
    n = B * per
    g = torch.Generator(device="cuda").manual_seed(tokens)
    x, known = (torch.randn(B, per, generator=g, device="cuda") for _ in range(2))
    m = (torch.rand(B, tokens, generator=g, device="cuda") < 0.5).to(torch.uint8)
    sel = m.bool().repeat_interleave(per_token, 1)
    seeds = [11, 12, 13, 14, 15]
    k = _keys(seeds, 3)
    seed = 0x0123456789ABCDEF
    s = DDIMScheduler(clip_sample_range=3)
    s.set_timesteps(7)
    ts = s.timesteps
    rtab = s.replace_table(ts).cuda()
    ts_d = ts.cuda()
    step = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    for t in ts.tolist():
        sa, sb = s.replace_coefficients(t)
        keyed, fed, batch, fed_b, tab, tab_b = (x.clone() for _ in range(6))
        z = randn_keyed(seeds, 3, (B, per), "cuda", domain=2, t=t)
        zb = torch.empty(n, device="cuda")
        kb = torch.from_numpy(np.array([seed], dtype=np.uint64).view(np.int64)).cuda()
        f.check(lib.bg_randn_keyed(kb.data_ptr(), 1, n, 2, t, zb.data_ptr(), st), "randn batch key")
        call = lambda out, noise, sd, keys: lib.bg_replace_known(out.data_ptr(), known.data_ptr(), m.data_ptr(), n,
                                                                 per_token, noise, sd, keys, per, t, sa, sb, st)
        f.check(call(keyed, None, 0, k.data_ptr()), "keyed")
        f.check(call(fed, z.data_ptr(), 0, None), "fed")
        f.check(call(batch, None, seed, None), "batch")
        f.check(call(fed_b, zb.data_ptr(), 0, None), "fed batch")
        f.check(lib.bg_step_advance(ts_d.data_ptr(), len(ts), step.data_ptr(), t_cur.data_ptr(), st), "advance")
        f.check(lib.bg_replace_known_tab(tab.data_ptr(), known.data_ptr(), m.data_ptr(), n, per_token, 0, k.data_ptr(),
                                         per, t_cur.data_ptr(), rtab.data_ptr(), step.data_ptr(), st), "tab keyed")
        f.check(lib.bg_replace_known_tab(tab_b.data_ptr(), known.data_ptr(), m.data_ptr(), n, per_token, seed, None, 0,
                                         t_cur.data_ptr(), rtab.data_ptr(), step.data_ptr(), st), "tab batch")
        torch.cuda.synchronize()
        assert torch.equal(keyed, fed), t
        assert torch.equal(batch, fed_b), t
        assert torch.equal(tab, keyed), t
        assert torch.equal(tab_b, batch), t
        if sb != 0.0:
            assert not torch.equal(keyed[sel], batch[sel])
            z0 = randn_keyed(seeds, 3, (B, per), "cuda", domain=0, t=t)     # the step noise at the same t
            assert not torch.equal(z0, z)
            assert float((z0 - z).abs().max()) > 1.0


def test_scheduler_replace_known_streams():
    """DDPMScheduler.replace_known: keyed mode is the kernel fed bg_randn_keyed(domain 2, t) (t + 1 before the loop); the
    batch key follows set_noise_seed and leaves the step stream where it was; out= writes in place"""
    from brepgen_b200.sampler import randn_keyed
    from brepgen_b200.schedulers import DDPMScheduler, sample_seed
    s = DDPMScheduler(clip_sample_range=3)
    s.set_timesteps(10)
    g = torch.Generator().manual_seed(4)
    B = 3
    x, known = (torch.randn(B, 9, 6, generator=g).cuda() for _ in range(2))
    mask = torch.rand(B, 9, generator=g).cuda() < 0.5
    s.set_sample_keys(seed=4, first=2, stage=1)
    seeds = [sample_seed(4, 2 + b) for b in range(B)]
    for t, initial in ((500, False), (900, True)):
        got = s.replace_known(x, known, mask, t, initial=initial)
        z = randn_keyed(seeds, 1, x.shape, "cuda", domain=2, t=t + 1 if initial else t)
        assert torch.equal(got, s.replace_known(x, known, mask, t, noise=z, initial=initial))
        assert torch.equal(got[~mask], x[~mask]) and not torch.equal(got[mask], x[mask])
    a, b = DDPMScheduler(), DDPMScheduler()
    for sch in (a, b):
        sch.set_timesteps(10)
        sch.set_noise_seed(9, 0, 1)
    eps = torch.randn(x.shape, generator=g).cuda()
    xa = a.step(eps, 500, x).prev_sample
    a.replace_known(xa, known, mask, 500, out=xa)
    ya = a.step(eps, 400, xa).prev_sample
    yb = b.step(eps, 400, b.step(eps, 500, x).prev_sample).prev_sample
    assert a._philox_offset == b._philox_offset
    assert torch.equal(ya[~mask], yb[~mask]) and not torch.equal(ya, yb)       # the same step noise on both
    zb = b.step(torch.zeros_like(x), 400, torch.zeros_like(x)).prev_sample     # sigma * z of a's and b's next draw
    za = a.step(torch.zeros_like(x), 400, torch.zeros_like(x)).prev_sample
    assert torch.equal(za, zb)


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


def _run(cfg, known=None, decoders=False):
    from brepgen_b200.sampler import Cascade
    ms = _models(cfg.use_cf)[0]
    if decoders:
        from brepgen_b200.vae import build_synthetic_decoders
        sv, ev = build_synthetic_decoders(torch.device("cuda"))
        casc = Cascade(ms, sv, ev)
    else:
        casc = Cascade(ms)
    out = casc.run(cfg, known=known)
    torch.cuda.synchronize()
    return out, casc


def _n_faces(out, want):
    nv = (~out["surfMask"]).sum(1).cpu().tolist()
    return [min(w, v) for w, v in zip(want, nv)]


KNOWN_FIELDS = (("surfPos", "surfPos"), ("surfZ", "surfZ"), ("edgePos", "edgePos"), ("edge_z", "edge_z"),
                ("edgeV", "edgeV"), ("edge_mask", "edgeM"))


@pytest.mark.parametrize("use_cf", [False, True])
@pytest.mark.parametrize("schedule,steps", [("ddpm", 4), ("ddim", 4), ("ddim", 10)])
def test_short_completion_matches_oracle(schedule, steps, use_cf):
    from brepgen_b200.sampler import Cascade, Completion
    from oracle.completion import run_cascade_completion
    ms, sds = _models(use_cf)
    cfg = _cfg(use_cf=use_cf, schedule=schedule, ddpm_steps=steps, ddim_steps=steps, ddim_eta=0.5)
    S = cfg.num_surfaces if use_cf else 2 * cfg.num_surfaces
    g = torch.Generator().manual_seed(9)

    def init():
        return {"surfPos": torch.randn(2, cfg.num_surfaces, 6, generator=g), "surfZ": torch.randn(2, S, 48, generator=g),
                "edgePos": torch.randn(2, S, 3, 6, generator=g), "edgeZV": torch.randn(2, S, 3, 18, generator=g)}
    bank = {}

    def noise(name, k, shape):
        key = (name, k, tuple(shape))
        if key not in bank:
            bank[key] = torch.randn(tuple(shape), generator=g)
        return bank[key]
    a = run_cascade_completion(sds, cfg, init(), noise, forwards=None)
    known = Completion.from_outputs(a, _n_faces(a, [1, 2]))
    assert sum(known.n_faces) >= 2
    init_b = init()
    rbank = {}

    def rnoise(name, k, shape):
        key = (name, k, tuple(shape))
        if key not in rbank:
            rbank[key] = torch.randn(tuple(shape), generator=g)
        return rbank[key]
    ref = run_cascade_completion(sds, cfg, init_b, noise, known=known, replace_noise=rnoise)
    n_r = len(rbank)
    out = Cascade(ms).run(cfg, init_noise=init_b, step_noise=noise, known=known, replace_noise=rnoise)
    assert len(rbank) == n_r == 4 * (steps + 1)          # every stage replaces: edges given; the same draws on both sides
    assert torch.equal(out["surfMask"].cpu(), ref["surfMask"])
    assert torch.equal(out["edgeM"].cpu(), ref["edgeM"])
    sv, ev = ~ref["surfMask"], ~ref["edgeM"]
    valid = {"surfPos": slice(None), "surfZ": sv, "edgePos": sv, "edge_z": ev, "edgeV": ev}
    for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV"):
        err = rel_l2(out[k].cpu()[valid[k]], ref[k][valid[k]])
        print(f"completion {schedule}-{steps} cf={use_cf} {k} rel_l2={err:.3e}")
        assert err < 1e-3, (k, err)
    for i, nf in enumerate(known.n_faces):
        for fk, ok in KNOWN_FIELDS:
            assert torch.equal(out[ok][i, :nf].cpu(), getattr(known, fk)[i, :nf]), (i, fk)


@pytest.mark.parametrize("edges", [True, False])
def test_round_trip_keeps_known_parts_bit_for_bit(edges):
    from brepgen_b200.sampler import Completion
    kw = dict(batch_size=5, num_surfaces=8, num_edges=5, schedule="ddim", ddim_steps=10, noise="per_sample", decode=True)
    a, _ = _run(_cfg(seed=1, **kw), decoders=True)
    n = _n_faces(a, [0, 1, 3, 5, 7])
    assert n[-1] >= 5
    known = Completion.from_outputs(a, n, edges=edges)
    b, _ = _run(_cfg(seed=2, **kw), known=known, decoders=True)
    for i, nf in enumerate(n):
        assert not b["surfMask"][i, :nf].any()
        fields = KNOWN_FIELDS if edges else KNOWN_FIELDS[:2]
        for fk, ok in fields:
            assert torch.equal(b[ok][i, :nf], a[ok][i, :nf]), (i, ok)
        assert torch.equal(b["surf_ncs"][i, :nf], a["surf_ncs"][i, :nf]), i
        if edges:
            assert torch.equal(b["edge_ncs"][i, :nf], a["edge_ncs"][i, :nf]), i
    assert not torch.equal(b["surfPos"][0], a["surfPos"][0])      # the unknown parts are generated anew


def _nothing_known(cfg):
    from brepgen_b200.sampler import Completion
    B, E = cfg.batch_size, cfg.num_edges
    return Completion(n_faces=[0] * B, surfPos=torch.zeros(B, 1, 6), surfZ=torch.zeros(B, 1, 48),
                      edgePos=torch.zeros(B, 1, E, 6), edge_z=torch.zeros(B, 1, E, 12), edgeV=torch.zeros(B, 1, E, 6),
                      edge_mask=torch.zeros(B, 1, E, dtype=torch.bool))


@pytest.mark.parametrize("noise", ["batch", "per_sample"])
@pytest.mark.parametrize("graph", ["off", "on"])
@pytest.mark.parametrize("schedule", ["ddpm", "ddim"])
def test_nothing_known_is_a_plain_run(schedule, graph, noise):
    for use_cf in (False, True):
        cfg = _cfg(batch_size=3, num_surfaces=5, num_edges=4, use_cf=use_cf, schedule=schedule, ddpm_steps=12,
                   ddim_steps=12, ddim_eta=0.5, graph=graph, noise=noise)
        a, _ = _run(cfg)
        b, casc = _run(cfg, known=_nothing_known(cfg))
        if graph == "on":
            assert casc.last_graph_steps == 4 * 12
        assert set(a) == set(b)
        for k in a:
            assert torch.equal(a[k], b[k]), (use_cf, k)


@pytest.mark.parametrize("noise", ["batch", "per_sample"])
@pytest.mark.parametrize("schedule", ["ddpm", "ddim"])
def test_graph_on_equals_graph_off(schedule, noise):
    from brepgen_b200.sampler import Completion
    for use_cf in (False, True):
        kw = dict(batch_size=3, num_surfaces=5, num_edges=4, use_cf=use_cf, schedule=schedule, ddpm_steps=12,
                  ddim_steps=12, ddim_eta=0.5, noise=noise)
        src, _ = _run(_cfg(seed=7, **kw))
        known = Completion.from_outputs(src, _n_faces(src, [2, 0, 3]))
        a, _ = _run(_cfg(graph="off", **kw), known=known)
        b, casc = _run(_cfg(graph="on", **kw), known=known)
        assert casc.last_graph_steps == 4 * 12
        for k in a:
            assert torch.equal(a[k], b[k]), (use_cf, k)
        plain, _ = _run(_cfg(graph="off", **kw))
        assert not torch.equal(a["surfPos"], plain["surfPos"])        # the replacement is really there


@pytest.mark.parametrize("graph", ["off", "on"])
def test_completed_sample_does_not_depend_on_its_batch(graph):
    from brepgen_b200.sampler import Completion
    kw = dict(num_surfaces=5, num_edges=4, use_cf=False, schedule="ddim", ddim_steps=12, ddim_eta=0.5, noise="per_sample",
              seed=21, graph=graph)
    src, _ = _run(_cfg(batch_size=5, seed=4, **{k: v for k, v in kw.items() if k != "seed"}))
    known = Completion.from_outputs(src, _n_faces(src, [0, 1, 2, 3, 4]))
    full, _ = _run(_cfg(batch_size=5, **kw), known=known)
    for b in range(5):
        one_known = Completion(n_faces=[known.n_faces[b]],
                               **{f: getattr(known, f)[b:b + 1] for f, _ in KNOWN_FIELDS})
        one, _ = _run(_cfg(batch_size=1, sample_base=b, **kw), known=one_known)
        for k in full:
            assert torch.equal(full[k][b], one[k][0]), (graph, b, k)


def test_duplicate_known_faces_are_rejected():
    from brepgen_b200.sampler import Completion
    cfg = _cfg()
    pos = torch.rand(2, 3, 6, generator=torch.Generator().manual_seed(0))
    pos[1, 2] = pos[1, 0] + 0.001
    f, lib, _ = _lib()
    l0 = lib.bg_launch_count()
    with pytest.raises(ValueError, match=r"samples \[1\]"):
        _run(cfg, known=Completion(n_faces=[3, 3], surfPos=pos))
    assert lib.bg_launch_count() == l0 + 1          # the de-duplication check only


# ----------------------------------------------------------------------------------------------------------- errors
def test_bad_arguments_are_rejected_and_launch_nothing():
    f, lib, st = _lib()
    B, per_token, tokens = 3, 6, 4
    per = per_token * tokens
    n = B * per
    x = torch.full((B, per), float("nan"), device="cuda")
    known = torch.zeros(B, per, device="cuda")
    m = torch.ones(B, tokens, dtype=torch.uint8, device="cuda")
    k = _keys([1, 2, 3], 0)
    coef = torch.ones(1, 2, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    t_cur = torch.zeros(1, dtype=torch.int64, device="cuda")

    def eager(x_p=x.data_ptr(), k_p=known.data_ptr(), m_p=m.data_ptr(), nn=n, pt=per_token, keys=k.data_ptr(), ps=per,
              t=5):
        return lib.bg_replace_known(x_p, k_p, m_p, nn, pt, None, 1, keys, ps, t, 0.5, 0.5, st)

    def tab(x_p=x.data_ptr(), k_p=known.data_ptr(), m_p=m.data_ptr(), nn=n, pt=per_token, keys=k.data_ptr(), ps=per,
            tc=t_cur.data_ptr(), cf=coef.data_ptr(), sp=step.data_ptr()):
        return lib.bg_replace_known_tab(x_p, k_p, m_p, nn, pt, 1, keys, ps, tc, cf, sp, st)
    cases = [
        ("eager NULL x", lambda: eager(x_p=None)), ("eager NULL known", lambda: eager(k_p=None)),
        ("eager NULL mask", lambda: eager(m_p=None)), ("eager n 0", lambda: eager(nn=0)),
        ("eager per_token 0", lambda: eager(pt=0)), ("eager per_token < 0", lambda: eager(pt=-6)),
        ("eager n % per_token", lambda: eager(pt=7)), ("eager per_sample 0", lambda: eager(ps=0)),
        ("eager per_sample % per_token", lambda: eager(ps=8)), ("eager per_sample not dividing n", lambda: eager(ps=2 * per)),
        ("eager t < 0", lambda: eager(t=-1)), ("eager t > 32 bits", lambda: eager(t=2 ** 32)),
        ("tab NULL x", lambda: tab(x_p=None)), ("tab NULL known", lambda: tab(k_p=None)),
        ("tab NULL mask", lambda: tab(m_p=None)), ("tab NULL t_cur", lambda: tab(tc=None)),
        ("tab NULL coef", lambda: tab(cf=None)), ("tab NULL step", lambda: tab(sp=None)),
        ("tab per_token 0", lambda: tab(pt=0)), ("tab n % per_token", lambda: tab(pt=5)),
        ("tab per_sample 0", lambda: tab(ps=0)), ("tab per_sample % per_token", lambda: tab(ps=8)),
        ("tab per_sample not dividing n", lambda: tab(ps=2 * per)),
    ]
    l0 = lib.bg_launch_count()
    for name, call in cases:
        assert call() == -1, name               # BG_STATUS_BAD_ARG
        assert lib.bg_last_error(), name
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0
    assert torch.isnan(x).all()
    # the same calls with valid arguments launch (the batch forms ignore per_sample)
    assert eager(t=2 ** 32 - 1) == 0 and eager(keys=None, ps=0) == 0 and tab(keys=None, ps=0) == 0
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0 + 3
