"""GPU tests of DDIM inversion and interpolation (Variation(start="invert"), Interpolation):

  * the inverse step is bg_ddim_step / bg_ddim_step_tab with sigma = 0: fp64 parity, eager = table bit for bit, and the
    forward DDIM step undoes it;
  * bg_slerp against float64 torch: endpoints, masked tokens, the lerp branch, per-sample independence, in-place, bad
    arguments;
  * with eps constant (the final Linear of every fc_out zeroed) an inverted variation at strength 1 reconstructs its source;
  * short inverted variations and an interpolation match oracle.inversion; alpha 0 / 1 are the inverted variations of a /
    b; graph on = graph off; a per-sample interpolation does not depend on its batch.
"""
import pytest
import torch

from test_gpu_completion import _lib, _models, rel_l2
from test_gpu_variation import FIELDS, _cfg, _fit, _start_noise

pytestmark = pytest.mark.gpu
NAN = float("nan")


# ---------------------------------------------------------------------------------------------------- inverse step
def _ref64(eps_c, eps_u, w, x, coefs, clip):
    sb, sa, sa_next, c_dir, _ = (float(c) for c in coefs)
    e = eps_c.double() if eps_u is None else eps_c.double() * (1 + w) - eps_u.double() * w
    x0 = (x.double() - sb * e) / sa
    if clip > 0:
        x0 = x0.clamp(-clip, clip)
    return sa_next * x0 + c_dir * e, x0


@pytest.mark.parametrize("t,n_steps,one", [(0, 10, True), (0, 10, False), (500, 10, True), (900, 10, True),
                                           (980, 50, True), (999, 1000, True)])
def test_inverse_step_matches_float64_and_table_form(t, n_steps, one):
    from brepgen_b200.schedulers import DDIMInverseScheduler
    f, lib, st = _lib()
    g = torch.Generator(device="cuda").manual_seed(t + n_steps)
    B, per = 5, 1003
    s = DDIMInverseScheduler(set_alpha_to_one=one, clip_sample_range=3.0)
    s.set_timesteps(n_steps)
    coefs = s.step_coefficients(t)
    x0 = torch.rand(B, per, generator=g, device="cuda") * 7 - 3.5          # partly outside the clip range
    eps_c, eps_u = (torch.randn(B, per, generator=g, device="cuda") for _ in range(2))
    x = (coefs[1] * x0 + coefs[0] * eps_c).contiguous()                    # a sample at the level below t
    tab = s.coefficient_table(torch.tensor([t])).cuda()
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    worst = 0.0
    for w, u in ((0.0, None), (0.6, eps_u)):
        res = s.step(eps_c, t, x, model_output_uncond=u, guidance_w=w)
        out, px0 = res.prev_sample, res.pred_original_sample
        ref, rx0 = _ref64(eps_c, u, w, x, coefs, 3.0)
        err = float((out.double() - ref).abs().max() / max(1.0, float(ref.abs().max())))
        worst = max(worst, err)
        assert err < 1.5e-7, (w, err)
        # x0 divides the rounded x - sb*e by sa: its error scales with (|x| + sb |e|) / sa, not with x0
        ae = eps_c.double().abs() * (1 + w) + (0.0 if u is None else u.double().abs() * w)
        scale = (x.double().abs() + coefs[0] * ae) / coefs[1]
        assert bool(((px0.double() - rx0).abs() <= 2.0 ** -22 * scale).all())
        o2 = torch.full_like(x, NAN)
        f.check(lib.bg_ddim_step_tab(eps_c.data_ptr(), f.ptr(u), w, x.data_ptr(), o2.data_ptr(), 0, 0, 0, None, 0, None,
                                     B * per, tab.data_ptr(), step.data_ptr(), 3.0, 0, st), "bg_ddim_step_tab")
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), o2.view(torch.int32))
    print(f"inverse step fp64 parity t={t} N={n_steps} one={one}: worst {worst:.3e}")


@pytest.mark.parametrize("n_steps", [10, 50])
def test_forward_step_undoes_the_inverse_step(n_steps):
    from brepgen_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    inv = DDIMInverseScheduler(clip_sample_range=3.0)
    fwd = DDIMScheduler(clip_sample_range=3.0)
    inv.set_timesteps(n_steps)
    fwd.set_timesteps(n_steps)
    g = torch.Generator(device="cuda").manual_seed(n_steps)
    worst = 0.0
    for t in inv.timesteps.tolist()[:: max(1, n_steps // 5)]:
        sb, sa = inv.step_coefficients(t)[:2]
        x0 = torch.rand(4, 999, generator=g, device="cuda") * 2 - 1
        eps = torch.randn(4, 999, generator=g, device="cuda")
        x = (sa * x0 + sb * eps).contiguous()
        back = fwd.step(eps, t, inv.step(eps, t, x).prev_sample).prev_sample
        ulps = float((back - x).abs().max() / (2.0 ** -23 * max(1.0, float(x.abs().max()))))
        worst = max(worst, ulps)
        assert ulps <= 8, (t, ulps)
    print(f"inverse then forward N={n_steps}: worst {worst:.2f} ulp of max(1, |x|)")


# ------------------------------------------------------------------------------------------------------------ slerp
def _slerp(a, b, alpha, mask=None, out=None, per_token=None):
    f, lib, st = _lib()
    B = a.shape[0]
    out = torch.full_like(a, NAN) if out is None else out
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    f.check(lib.bg_slerp(a.data_ptr(), b.data_ptr(), alpha.data_ptr(), f.ptr(m), B, a.numel() // B,
                         a.shape[-1] if per_token is None else per_token, out.data_ptr(), st), "bg_slerp")
    torch.cuda.synchronize()
    return out


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("shape", [(5, 37, 18), (3, 50, 6), (2, 4000, 48)])
@pytest.mark.parametrize("masked", [False, True])
def test_slerp_matches_float64(shape, masked):
    from oracle.inversion import slerp
    g = torch.Generator(device="cuda").manual_seed(shape[1])
    a, b = torch.randn(shape, generator=g, device="cuda"), torch.randn(shape, generator=g, device="cuda")
    B = shape[0]
    alpha = torch.linspace(0.1, 0.9, B, device="cuda")
    mask = (torch.rand(shape[:-1], generator=g, device="cuda") < 0.3) if masked else None
    got = _slerp(a, b, alpha, mask)
    ref = slerp(a.cpu(), b.cpu(), alpha.cpu().double(), None if mask is None else mask.cpu())
    err = (got.cpu().double() - ref).abs()
    assert bool((err <= 2.0 ** -23 * ref.abs() + 1e-9).all()), float(err.max())
    if masked:
        assert torch.equal(_bits(got[mask]), _bits(a[mask]))


def test_slerp_endpoints_lerp_independence_and_in_place():
    from oracle.inversion import slerp
    g = torch.Generator(device="cuda").manual_seed(3)
    a, b = torch.randn(4, 60, 6, generator=g, device="cuda"), torch.randn(4, 60, 6, generator=g, device="cuda")
    mask = torch.rand(4, 60, generator=g, device="cuda") < 0.25
    al = torch.tensor([0.0, 1.0, 0.3, 0.7], device="cuda")
    got = _slerp(a, b, al, mask)
    assert torch.equal(_bits(got[0]), _bits(a[0]))
    keep = ~mask[1]
    assert torch.equal(_bits(got[1][keep]), _bits(b[1][keep])) and torch.equal(_bits(got[1][~keep]), _bits(a[1][~keep]))
    # the lerp: b nearly parallel to a
    near = a + 1e-3 * b
    lp = _slerp(a, near, al)
    ref = (1 - al.double().cpu())[:, None, None] * a.double().cpu() + al.double().cpu()[:, None, None] * near.double().cpu()
    assert bool(((lp.cpu().double() - ref).abs() <= 2.0 ** -23 * ref.abs() + 1e-9).all())
    assert torch.allclose(slerp(a.cpu(), near.cpu(), al.cpu().double()), ref, rtol=1e-12, atol=0)
    # one sample's output depends on its own a, b and alpha only
    b2, al2 = b.clone(), al.clone()
    b2[3] = torch.randn(60, 6, generator=g, device="cuda")
    al2[3] = 0.5
    other = _slerp(a, b2, al2, mask)
    assert torch.equal(_bits(other[:3]), _bits(got[:3]))
    # out aliasing a
    a2 = a.clone()
    _slerp(a2, b, al, mask, out=a2)
    assert torch.equal(_bits(a2), _bits(got))


def test_bad_slerp_arguments_launch_nothing():
    f, lib, st = _lib()
    a = torch.zeros(3, 12, device="cuda")
    al = torch.zeros(3, device="cuda")
    out = torch.full_like(a, NAN)

    def call(pa=a.data_ptr(), pb=a.data_ptr(), pal=al.data_ptr(), n=3, per=12, tok=6, po=out.data_ptr()):
        return lib.bg_slerp(pa, pb, pal, None, n, per, tok, po, st)
    cases = [("NULL a", lambda: call(pa=None)), ("NULL b", lambda: call(pb=None)), ("NULL alpha", lambda: call(pal=None)),
             ("NULL out", lambda: call(po=None)), ("n_samples 0", lambda: call(n=0)), ("per_sample 0", lambda: call(per=0)),
             ("per_token 0", lambda: call(tok=0)), ("per_token -6", lambda: call(tok=-6)),
             ("per_sample not a multiple", lambda: call(tok=5)), ("n_samples 2^31", lambda: call(n=2 ** 31))]
    l0 = lib.bg_launch_count()
    for name, c in cases:
        assert c() == -1, name
        assert lib.bg_last_error(), name
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0 and torch.isnan(out).all()
    assert call() == 0
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0 + 1 and torch.equal(out, a)


# ---------------------------------------------------------------------------------------------------------- cascade
def _run(cfg, source=None, init_noise=None, models=None):
    from brepgen_b200.sampler import Cascade
    casc = Cascade(models if models is not None else _models(cfg.use_cf)[0])
    out = casc.run(cfg, init_noise=init_noise, source=source)
    torch.cuda.synchronize()
    return out, casc


def _var(out, st):
    from brepgen_b200.sampler import Variation
    return Variation.from_outputs(out, st, start="invert")


def _interp(a, b, st, alpha):
    from brepgen_b200.sampler import Interpolation, Variation
    return Interpolation(Variation.from_outputs(a, st), Variation.from_outputs(b, st), alpha)


def _constant_eps_models(use_cf):
    """the synthetic denoisers with the final Linear of fc_out zeroed: eps is its bias whatever x, t and conditioning"""
    from brepgen_b200.models import NETS
    from brepgen_b200.spec import denoiser_spec
    from brepgen_b200.synth import synth_state_dict
    ms = {}
    for kind in NETS:
        sd = synth_state_dict(denoiser_spec(kind, use_cf), seed=11)
        sd["fc_out.3.weight"] = torch.zeros_like(sd["fc_out.3.weight"])
        m = NETS[kind](use_cf)
        m.load_state_dict(sd)
        ms[kind] = m.cuda().eval()
    return ms


@pytest.mark.parametrize("use_cf", [False, True])
def test_strength_one_inversion_reconstructs_the_source(use_cf):
    cfg = _cfg(use_cf=use_cf, ddim_steps=10)
    a, _ = _run(cfg)
    src = _fit(a, cfg, (2, 4))
    # valid slots that are not contiguous: drop the first valid face of sample 1
    first = int(torch.nonzero(~src["surfMask"][1]).flatten()[0])
    if int((~src["surfMask"][1]).sum()) > 1:
        src["surfMask"][1, first] = True
        src["edgeM"][1, first] = True
    out, _ = _run(cfg, _var(src, 1.0), models=_constant_eps_models(use_cf))
    for b in range(cfg.batch_size):
        fs, fo = torch.nonzero(~src["surfMask"][b]).flatten(), torch.nonzero(~out["surfMask"][b]).flatten()
        assert len(fs) == len(fo), b
        for k in ("surfPos", "surfZ"):
            assert float((out[k][b, fo] - src[k][b, fs]).abs().max()) < 1e-5, (b, k)
        for j_s, j_o in zip(fs.tolist(), fo.tolist()):
            es, eo = torch.nonzero(~src["edgeM"][b, j_s]).flatten(), torch.nonzero(~out["edgeM"][b, j_o]).flatten()
            assert len(es) == len(eo), (b, j_s)
            for k in ("edgePos", "edge_z", "edgeV"):
                assert float((out[k][b, j_o, eo] - src[k][b, j_s, es]).abs().max()) < 1e-5, (b, j_s, k)


def _check_oracle(out, ref, what, bar=2e-3):
    assert torch.equal(out["surfMask"].cpu(), ref["surfMask"]), what
    assert torch.equal(out["edgeM"].cpu(), ref["edgeM"]), what
    sv, ev = ~ref["surfMask"], ~ref["edgeM"]
    valid = {"surfPos": slice(None), "surfZ": sv, "edgePos": sv, "edge_z": ev, "edgeV": ev}
    for k in valid:
        err = rel_l2(out[k].cpu()[valid[k]], ref[k][valid[k]])
        print(f"{what} {k} rel_l2={err:.3e}")
        assert err < bar, (what, k, err)


@pytest.mark.parametrize("use_cf", [False, True])
def test_inverted_variation_and_interpolation_match_oracle(use_cf):
    from oracle.inversion import run_cascade_interpolation, run_cascade_inverted_variation
    sds = _models(use_cf)[1]
    cfg = _cfg(use_cf=use_cf, ddim_steps=10)
    a, _ = _run(cfg)
    b, _ = _run(_cfg(use_cf=use_cf, ddim_steps=10, seed=9))
    A, Bs = _fit(a, cfg, (2, 4)), _fit(b, cfg, (3, 1))
    # strength 1 inverts up to t = 900 and denoises back from there: both divide the fp16-GEMM error of eps by
    # sqrt(abar_900) = 0.017, which the fp32 oracle amplifies alike from a 3e-4 perturbation of eps to 2.4e-3 (surfPos)
    # and 6.6e-3 (surfZ), and the edge stages compound it (worst on an H100: 1.9e-2, edge_z without CFG); the shorter
    # round trips keep the 2e-3 bar of the other cascade tests
    for st, bar in (((1.0,) * 4, 4e-2), ((0.6,) * 4, 2e-3), ((0, 0, 0.6, 0.6), 2e-3)):
        init = _start_noise(cfg, st, seed=5)
        ref = run_cascade_inverted_variation(sds, cfg, _var(A, st), init)
        out, _ = _run(cfg, _var(A, st), init_noise=init)
        _check_oracle(out, ref, f"inverted variation cf={use_cf} s={st}", bar)
    st = (0.6,) * 4
    init = _start_noise(cfg, st, seed=6)
    alpha = [0.5, 0.5]
    ref = run_cascade_interpolation(sds, cfg, _var(A, st), _var(Bs, st), alpha, init)
    out, _ = _run(cfg, _interp(A, Bs, st, alpha), init_noise=init)
    _check_oracle(out, ref, f"interpolation cf={use_cf}")


@pytest.mark.parametrize("use_cf", [False, True])
def test_interpolation_endpoints_are_the_inverted_variations(use_cf):
    cfg = _cfg(use_cf=use_cf, ddim_steps=10, noise="per_sample")
    a, _ = _run(cfg)
    b, _ = _run(_cfg(use_cf=use_cf, ddim_steps=10, noise="per_sample", seed=9))
    A, Bs = _fit(a, cfg, (2, 4)), _fit(b, cfg, (3, 1))
    st = (0.7,) * 4
    va, _ = _run(cfg, _var(A, st))
    vb, _ = _run(cfg, _var(Bs, st))
    i0, _ = _run(cfg, _interp(A, Bs, st, [0.0, 0.0]))
    i1, _ = _run(cfg, _interp(A, Bs, st, [1.0, 1.0]))
    for k in FIELDS:
        assert torch.equal(i0[k], va[k]), k
    # alpha = 1: slots without a source keep a's inversion; every valid token is b's
    assert torch.equal(i1["surfMask"], vb["surfMask"]) and torch.equal(i1["edgeM"], vb["edgeM"])
    sv, ev = ~vb["surfMask"], ~vb["edgeM"]
    for k, m in (("surfPos", slice(None)), ("surfZ", sv), ("edgePos", sv), ("edge_z", ev), ("edgeV", ev)):
        assert torch.equal(i1[k][m], vb[k][m]), k


@pytest.mark.parametrize("noise", ["batch", "per_sample"])
def test_graph_on_equals_graph_off(noise):
    for use_cf in (False, True):
        kw = dict(batch_size=3, num_surfaces=5, num_edges=4, use_cf=use_cf, ddim_steps=12, noise=noise)
        a, _ = _run(_cfg(seed=7, **kw))
        b, _ = _run(_cfg(seed=8, **kw))
        A, Bs = _fit(a, _cfg(**kw), (3, 1, 5)), _fit(b, _cfg(**kw), (2, 5, 1))
        for src in (_var(A, 0.5), _var(A, (0, 0, 0.25, 0.75)), _interp(A, Bs, 0.5, [0.2, 0.5, 0.9])):
            off, _ = _run(_cfg(graph="off", **kw), src)
            on, casc = _run(_cfg(graph="on", **kw), src)
            assert casc.last_graph_steps > 0
            for k in off:
                assert torch.equal(off[k], on[k]), (use_cf, k)


@pytest.mark.parametrize("graph", ["off", "on"])
def test_per_sample_interpolation_does_not_depend_on_its_batch(graph):
    kw = dict(num_surfaces=5, num_edges=4, use_cf=False, ddim_steps=12, noise="per_sample", graph=graph)
    a, _ = _run(_cfg(batch_size=4, seed=4, **kw))
    b, _ = _run(_cfg(batch_size=4, seed=5, **kw))
    A, Bs = _fit(a, _cfg(**kw), (1, 2, 3, 4)), _fit(b, _cfg(**kw), (4, 3, 2, 1))
    alpha = [0.1, 0.4, 0.6, 0.95]
    full, _ = _run(_cfg(batch_size=4, seed=21, **kw), _interp(A, Bs, 0.5, alpha))
    for i in range(4):
        one = lambda o: {k: o[k][i:i + 1] for k in FIELDS}
        single, _ = _run(_cfg(batch_size=1, seed=21, sample_base=i, **kw), _interp(one(A), one(Bs), 0.5, [alpha[i]]))
        for k in full:
            assert torch.equal(full[k][i], single[k][0]), (i, k)
