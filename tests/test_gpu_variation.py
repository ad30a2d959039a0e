"""GPU tests of B-rep variations (Cascade.run(source=Variation(...))): the start kernels and the cascade.

  * bg_add_noise_gather is the fp32 torch expression of add_noise on the gathered, scaled source, bit for bit; -1 tokens
    are z; keyed z is bg_randn_keyed's; an out-of-range index poisons only its token; bad arguments launch nothing;
  * bg_fill_index is the reference's pad_repeat (fill_golden.npz) and the oracle's fill;
  * bg_dedup_surfaces_index is bg_dedup_surfaces bit for bit, plus the slot of every survivor;
  * kept stages come out as given, forward counts follow the strengths, short variations match oracle.variation;
  * graph on is graph off, and a per-sample variation does not depend on its batch.
"""
import os

import numpy as np
import pytest
import torch

from test_gpu_completion import _keys, _lib, _models, rel_l2

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float("nan")


def _gather(src, index, dim, scale, sa, sb, noise=None, keys=None, tps=0, n_src=None, out=None):
    f, lib, st = _lib()
    n_tok = index.numel()
    out = torch.empty(n_tok, dim, device="cuda") if out is None else out
    f.check(lib.bg_add_noise_gather(src.data_ptr(), src.numel() // dim if n_src is None else n_src, index.data_ptr(),
                                    n_tok, dim, scale, sa, sb, f.ptr(noise), f.ptr(keys), tps, 1, 0, out.data_ptr(), st),
            "bg_add_noise_gather")
    torch.cuda.synchronize()
    return out


def _torch_add_noise(src, index, scale, sa, sb, z):
    """the fp32 torch expression: add_noise(scale * src[index], z) (index -1: z)"""
    i = index.long()
    g = src[i.clamp(min=0)]
    return torch.where((i == -1)[:, None], z, sa * (scale * g) + sb * z)


def _coefs(t):
    from brepgen_b200.schedulers import DDPMScheduler
    return DDPMScheduler().replace_coefficients(t, initial=True)


# -------------------------------------------------------------------------------------------------- gather kernel
@pytest.mark.parametrize("dim,n_tok", [(6, 50), (48, 333), (18, 4000)])
@pytest.mark.parametrize("scale", [1.0, 3.0])
def test_gather_is_the_torch_expression_bit_for_bit(dim, n_tok, scale):
    g = torch.Generator(device="cuda").manual_seed(dim * 7 + n_tok)
    n_src = n_tok // 2 + 3
    src = torch.randn(n_src, dim, generator=g, device="cuda") * 0.7
    index = torch.randint(-1, n_src, (n_tok,), generator=g, device="cuda", dtype=torch.int32)
    z = torch.randn(n_tok, dim, generator=g, device="cuda")
    for t in (999, 500, 101, 0):
        sa, sb = _coefs(t)
        got = _gather(src, index, dim, scale, sa, sb, noise=z)
        ref = _torch_add_noise(src, index, scale, sa, sb, z)
        assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), t
        assert torch.equal(got[index == -1], z[index == -1])


@pytest.mark.parametrize("dim,tokens", [(6, 50), (18, 13), (48, 7)])
def test_keyed_z_is_randn_keyed(dim, tokens):
    from brepgen_b200.sampler import randn_keyed
    seeds = [3, 5, 8, 13, 21]
    B = len(seeds)
    g = torch.Generator(device="cuda").manual_seed(tokens)
    src = torch.randn(B * tokens, dim, generator=g, device="cuda")
    index = torch.randint(-1, B * tokens, (B * tokens,), generator=g, device="cuda", dtype=torch.int32)
    index[:tokens] = -1                          # sample 0: pure noise
    sa, sb = _coefs(420)
    for stage in (0, 2):
        k = _keys(seeds, stage)
        got = _gather(src, index, dim, 3.0, sa, sb, keys=k, tps=tokens)
        z = randn_keyed(seeds, stage, (B, tokens * dim), "cuda", domain=1, t=0).reshape(-1, dim)
        assert torch.equal(got[:tokens], z[:tokens])
        assert torch.equal(got, _torch_add_noise(src, index, 3.0, sa, sb, z))


def test_out_of_range_index_poisons_only_its_token():
    dim, n_src = 18, 20
    g = torch.Generator(device="cuda").manual_seed(1)
    src = torch.randn(n_src, dim, generator=g, device="cuda")
    index = torch.arange(40, device="cuda", dtype=torch.int32) % n_src
    bad = torch.tensor([3, 17, 25, 39], device="cuda")
    index[bad] = torch.tensor([-2, n_src, 2 ** 31 - 1, -7], device="cuda", dtype=torch.int32)
    z = torch.randn(40, dim, generator=g, device="cuda")
    sa, sb = _coefs(300)
    got = _gather(src, index, dim, 1.0, sa, sb, noise=z)
    poisoned = torch.zeros(40, dtype=torch.bool, device="cuda")
    poisoned[bad] = True
    assert torch.isnan(got[poisoned]).all()
    good = index.clone()
    good[bad] = 0
    assert torch.equal(got[~poisoned], _torch_add_noise(src, good, 1.0, sa, sb, z)[~poisoned])


def test_bad_arguments_are_rejected_and_launch_nothing():
    f, lib, st = _lib()
    dim, n_tok, B = 6, 12, 3
    src = torch.zeros(n_tok, dim, device="cuda")
    index = torch.zeros(n_tok, dtype=torch.int32, device="cuda")
    out = torch.full((n_tok, dim), NAN, device="cuda")
    z = torch.zeros(n_tok, dim, device="cuda")
    k = _keys([1, 2, 3], 0)
    mask = torch.zeros(n_tok, 8, dtype=torch.uint8, device="cuda")
    fill = torch.full((n_tok, 8), -5, dtype=torch.int32, device="cuda")
    pos = torch.rand(B, 4, 6, device="cuda")
    opos, omask = torch.empty_like(pos), torch.empty(B, 4, dtype=torch.uint8, device="cuda")

    def gather(s=src.data_ptr(), ns=n_tok, ix=index.data_ptr(), nt=n_tok, d=dim, nz=z.data_ptr(), keys=None, tps=0,
               dom=1, t=0, o=out.data_ptr()):
        return lib.bg_add_noise_gather(s, ns, ix, nt, d, 1.0, 0.5, 0.5, nz, keys, tps, dom, t, o, st)

    def fill_index(m=mask.data_ptr(), rm=None, rows=n_tok, ns=n_tok, ins=8, outs=8, o=fill.data_ptr()):
        return lib.bg_fill_index(m, rm, rows, ns, ins, outs, o, st)
    cases = [
        ("gather NULL src", lambda: gather(s=None)), ("gather NULL index", lambda: gather(ix=None)),
        ("gather NULL out", lambda: gather(o=None)), ("gather n_src 0", lambda: gather(ns=0)),
        ("gather n_tokens 0", lambda: gather(nt=0)), ("gather dim 0", lambda: gather(d=0)),
        ("gather both noises", lambda: gather(keys=k.data_ptr(), tps=4)),
        ("gather no noise", lambda: gather(nz=None)),
        ("gather keyed tps 0", lambda: gather(nz=None, keys=k.data_ptr(), tps=0)),
        ("gather keyed tps not dividing", lambda: gather(nz=None, keys=k.data_ptr(), tps=5)),
        ("gather domain < 0", lambda: gather(dom=-1)), ("gather t < 0", lambda: gather(t=-1)),
        ("gather t > 32 bits", lambda: gather(t=2 ** 32)),
        ("fill NULL mask", lambda: fill_index(m=None)), ("fill NULL out", lambda: fill_index(o=None)),
        ("fill rows 0", lambda: fill_index(rows=0)), ("fill n_src 0", lambda: fill_index(ns=0)),
        ("fill in_slots 0", lambda: fill_index(ins=0)), ("fill in_slots 257", lambda: fill_index(ins=257)),
        ("fill out_slots 0", lambda: fill_index(outs=0)),
        ("fill rows > n_src without a map", lambda: fill_index(ns=n_tok - 1)),
        ("dedup index NULL", lambda: lib.bg_dedup_surfaces_index(pos.data_ptr(), B, 4, 0.08, opos.data_ptr(),
                                                                 omask.data_ptr(), None, st)),
    ]
    l0 = lib.bg_launch_count()
    for name, call in cases:
        assert call() == -1, name               # BG_STATUS_BAD_ARG
        assert lib.bg_last_error(), name
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0
    assert torch.isnan(out).all() and (fill == -5).all()
    assert gather() == 0 and gather(nz=None, keys=k.data_ptr(), tps=4) == 0 and fill_index() == 0
    torch.cuda.synchronize()
    assert lib.bg_launch_count() == l0 + 3


# ------------------------------------------------------------------------------------------------------- fill map
def _fill(mask, out_slots, row_map=None):
    from brepgen_b200.sampler import fill_index
    return fill_index(mask, out_slots, row_map).cpu()


def test_fill_index_is_the_reference_pad_repeat():
    gold = np.load(os.path.join(ROOT, "tests", "golden", "fill_golden.npz"))
    for key in gold.files:
        S = int(key[1:])
        n = torch.arange(1, S + 1)
        mask = (torch.arange(S)[None, :] >= n[:, None]).cuda()           # row n - 1: the first n slots valid
        got = _fill(mask, S)
        assert torch.equal(got, torch.from_numpy(gold[key]).int() + torch.arange(S, dtype=torch.int32)[:, None] * S), key


@pytest.mark.parametrize("in_slots,out_slots", [(10, 5), (10, 10), (40, 40), (100, 50), (256, 256)])
@pytest.mark.parametrize("row_map", [False, True])
def test_fill_index_matches_oracle(in_slots, out_slots, row_map):
    from oracle.variation import fill_rows
    g = torch.Generator().manual_seed(in_slots + out_slots)
    n_src = 37
    p = torch.rand(n_src, 1, generator=g)
    mask = torch.rand(n_src, in_slots, generator=g) < p                    # densities 0..1 per row
    nv = (~mask).sum(1)
    mask[nv > out_slots] = True                                           # rows that fit (overflow: below)
    mask[nv > out_slots, :out_slots // 2] = False
    mask[5] = True                                                         # a row without a valid slot
    rm = torch.randint(-1, n_src, (60,), generator=g, dtype=torch.int32) if row_map else None
    got = _fill(mask.cuda(), out_slots, rm.cuda() if row_map else None)
    ref = torch.tensor(fill_rows(mask.numpy(), out_slots, None if rm is None else rm.tolist()), dtype=torch.int32)
    assert torch.equal(got, ref)


def test_fill_index_overflow_and_bad_rows_are_poisoned():
    mask = torch.zeros(3, 8, dtype=torch.bool)
    mask[1, 3:] = True                                                     # 3 valid: fits 4 slots; rows 0, 2: 8 do not
    got = _fill(mask.cuda(), 4, torch.tensor([0, 1, 2, -1, 3, -2], dtype=torch.int32).cuda())
    assert got[0].tolist() == [-2] * 4 and got[2].tolist() == [-2] * 4 and got[3].tolist() == [-1] * 4
    assert got[1].tolist() == [8, 8, 9, 10]
    assert got[4].tolist() == [-2] * 4 and got[5].tolist() == [-2] * 4    # row map entries out of range


# ------------------------------------------------------------------------------------------------------ index dedup
@pytest.mark.parametrize("kind", ["random", "duplicates"])
@pytest.mark.parametrize("B,S", [(3, 7), (16, 100), (4, 256)])
def test_dedup_index_keeps_positions_and_mask(kind, B, S):
    from brepgen_b200.sampler import dedup_surfaces, dedup_surfaces_index
    from oracle.variation import dedup_surfaces_survivors
    g = torch.Generator().manual_seed(B * S)
    x = torch.rand(B, S, 6, generator=g) * 2 - 1
    if kind == "duplicates":                 # copies of a few boxes, some corner-swapped, some within the threshold
        src = torch.randint(0, 4, (B, S), generator=g)
        x = x.gather(1, src[..., None].expand(B, S, 6)) + (torch.rand(B, S, 1, generator=g) < 0.3) * 0.02
        swap = torch.rand(B, S, generator=g) < 0.3
        x[swap] = torch.cat([x[swap][:, 3:], x[swap][:, :3]], -1)
    xd = x.cuda()
    p0, m0 = dedup_surfaces(xd, 0.08)
    p1, m1, idx = dedup_surfaces_index(xd, 0.08)
    assert torch.equal(p0.view(torch.int32), p1.view(torch.int32)) and torch.equal(m0, m1)
    n = (~m1).sum(1)
    assert torch.equal((idx >= 0), ~m1)
    r4 = torch.round(xd * 10000.0) / torch.full_like(xd, 10000.0)     # a true division (a scalar divisor is a reciprocal)
    i = idx.long().clamp(min=0)
    kept = r4.gather(1, i[..., None].expand(B, S, 6))
    assert torch.equal(kept[~m1].view(torch.int32), p1[~m1].view(torch.int32))
    _, _, slots = dedup_surfaces_survivors(x.numpy(), np.float32(0.08))
    for b in range(B):
        assert idx[b, :int(n[b])].tolist() == slots[b] and (idx[b, int(n[b]):] == -1).all()
    if kind == "duplicates":
        assert int(n.max()) < S


# -------------------------------------------------------------------------------------------------------- cascade
def _cfg(**kw):
    from brepgen_b200.sampler import CascadeConfig
    base = dict(batch_size=2, num_surfaces=4, num_edges=3, class_label=6, schedule="ddim", ddim_steps=10, seed=3,
                decode=False, graph="off")
    base.update(kw)
    return CascadeConfig(**base)


class _Counted:
    def __init__(self, m):
        self.m, self.calls = m, 0

    def __call__(self, *a):
        self.calls += 1
        return self.m(*a)


def _run(cfg, source=None, decoders=False, init_noise=None, step_noise=None, counted=False):
    from brepgen_b200.sampler import Cascade
    ms = _models(cfg.use_cf)[0]
    if counted:
        ms = {k: _Counted(m) for k, m in ms.items()}
    sv = ev = None
    if decoders:
        from brepgen_b200.vae import build_synthetic_decoders
        sv, ev = build_synthetic_decoders(torch.device("cuda"))
    casc = Cascade(ms, sv, ev)
    out = casc.run(cfg, init_noise=init_noise, step_noise=step_noise, source=source)
    torch.cuda.synchronize()
    return out, casc, ms


def _fit(out, cfg, n=(2, 4)):
    """a plain run's output with sample b cut to at most its first n[b] valid faces, so that it fits the num_surfaces slots
    a non-CFG variation starting above t = 249 has"""
    o = {k: v.clone() for k, v in out.items()}
    S = o["surfMask"].shape[1]
    for b, nb in enumerate(n):
        valid = torch.nonzero(~o["surfMask"][b]).flatten()
        cut = valid[min(nb, cfg.num_surfaces):]
        o["surfMask"][b, cut] = True
        o["edgeM"][b, cut] = True
    assert int((~o["surfMask"]).sum(1).max()) <= cfg.num_surfaces and S == o["edgeM"].shape[1]
    return o


def _var(out, st):
    from brepgen_b200.sampler import Variation
    return Variation.from_outputs(out, st)


FIELDS = ("surfPos", "surfMask", "surfZ", "edgePos", "edgeM", "edge_z", "edgeV")


@pytest.mark.parametrize("use_cf", [False, True])
@pytest.mark.parametrize("schedule", ["ddpm", "ddim", "dpm"])
def test_zero_strengths_return_the_source_and_its_decodes(schedule, use_cf):
    cfg = _cfg(use_cf=use_cf, schedule=schedule, ddpm_steps=10, dpm_steps=10, decode=True, noise="per_sample")
    a, _, _ = _run(cfg, decoders=True)
    b, _, ms = _run(cfg, source=_var(a, 0.0), decoders=True, counted=True)
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert all(m.calls == 0 for m in ms.values())


@pytest.mark.parametrize("schedule,steps,s", [("ddpm", 10, 0.5), ("ddim", 10, 0.6), ("dpm", 10, 0.5), ("ddim", 50, 0.3)])
def test_kept_prefix_and_forward_counts(schedule, steps, s):
    cfg = _cfg(schedule=schedule, ddpm_steps=steps, ddim_steps=steps, dpm_steps=steps)
    a, _, _ = _run(cfg)
    for st in ((0, 0, s, s), (0, s, s, s), (s, s, s, s), (0, 0, 0, s)):
        src = _fit(a, cfg) if st[0] > 0 else a
        b, _, ms = _run(cfg, source=_var(src, st), counted=True)
        want = [int(steps * v) for v in st]
        assert [ms[k].calls for k in ("surfpos", "surfz", "edgepos", "edgez")] == want, st
        kept = {0: ("surfPos", "surfMask"), 1: ("surfZ",), 2: ("edgePos", "edgeM"), 3: ("edge_z", "edgeV")}
        for i, v in enumerate(st):
            for k in kept[i]:
                if v == 0:
                    assert torch.equal(b[k], src[k]), (st, k)
        assert not torch.equal(b["edge_z"], src["edge_z"]), st


def _noise_bank(seed):
    g = torch.Generator().manual_seed(seed)
    bank = {}

    def noise(name, k, shape):
        key = (name, k, tuple(shape))
        if key not in bank:
            bank[key] = torch.randn(tuple(shape), generator=g)
        return bank[key]
    return noise


def _start_noise(cfg, st, seed):
    from brepgen_b200.sampler import stage_timesteps, start_slots
    from brepgen_b200.schedulers import strength_timesteps
    g = torch.Generator().manual_seed(seed)
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    S = S0 if cfg.use_cf else 2 * S0
    S1 = start_slots(cfg, int(strength_timesteps(stage_timesteps(cfg), st[0])[0])) if st[0] > 0 else S0
    return {"surfPos": torch.randn(B, S1, 6, generator=g), "surfZ": torch.randn(B, S, 48, generator=g),
            "edgePos": torch.randn(B, S, E, 6, generator=g), "edgeZV": torch.randn(B, S, E, 18, generator=g)}


ORACLE_CASES = [("ddpm", dict(ddpm_steps=10), 0.5, 2e-3), ("ddim", dict(ddim_steps=10, ddim_eta=0.0), 0.6, 2e-3),
                ("ddim", dict(ddim_steps=10, ddim_eta=1.0), 0.6, 2e-3),
                ("dpm", dict(dpm_steps=10, dpm_algorithm="dpmsolver++"), 0.5, 3e-3),
                ("dpm", dict(dpm_steps=10, dpm_algorithm="sde-dpmsolver++"), 0.5, 3e-3)]


@pytest.mark.parametrize("use_cf", [False, True])
@pytest.mark.parametrize("schedule,kw,s,bar", ORACLE_CASES, ids=["ddpm", "ddim-eta0", "ddim-eta1", "dpm-ode", "dpm-sde"])
def test_short_variation_matches_oracle(schedule, kw, s, bar, use_cf):
    from oracle.variation import run_cascade_variation
    sds = _models(use_cf)[1]
    cfg = _cfg(use_cf=use_cf, schedule=schedule, **kw)
    a, _, _ = _run(cfg)
    src = _fit(a, cfg, (2, 4))
    for st in ((s,) * 4, (0, 0, s, s)):
        init = _start_noise(cfg, st, seed=5)
        noise = _noise_bank(7)
        ref = run_cascade_variation(sds, cfg, _var(src, st), init, noise)
        out, _, _ = _run(cfg, source=_var(src, st), init_noise=init, step_noise=noise)
        assert torch.equal(out["surfMask"].cpu(), ref["surfMask"]), st
        assert torch.equal(out["edgeM"].cpu(), ref["edgeM"]), st
        sv, ev = ~ref["surfMask"], ~ref["edgeM"]
        valid = {"surfPos": slice(None), "surfZ": sv, "edgePos": sv, "edge_z": ev, "edgeV": ev}
        for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV"):
            err = rel_l2(out[k].cpu()[valid[k]], ref[k][valid[k]])
            print(f"variation {schedule} {kw} s={st} cf={use_cf} {k} rel_l2={err:.3e}")
            assert err < bar, (st, k, err)


@pytest.mark.parametrize("noise", ["batch", "per_sample"])
@pytest.mark.parametrize("schedule", ["ddpm", "ddim", "dpm"])
def test_graph_on_equals_graph_off(schedule, noise):
    for use_cf in (False, True):
        kw = dict(batch_size=3, num_surfaces=5, num_edges=4, use_cf=use_cf, schedule=schedule, ddpm_steps=12,
                  ddim_steps=12, dpm_steps=12, ddim_eta=0.5, dpm_algorithm="sde-dpmsolver++", noise=noise)
        a, _, _ = _run(_cfg(seed=7, **kw))
        src = _fit(a, _cfg(**kw), (3, 1, 5))
        for st in ((0.5,) * 4, (0, 0, 0.25, 0.75)):
            off, _, _ = _run(_cfg(graph="off", **kw), source=_var(src, st))
            on, casc, _ = _run(_cfg(graph="on", **kw), source=_var(src, st))
            assert casc.last_graph_steps == sum(int(12 * v) for v in st)
            for k in off:
                assert torch.equal(off[k], on[k]), (use_cf, st, k)


@pytest.mark.parametrize("graph", ["off", "on"])
@pytest.mark.parametrize("schedule", ["ddim", "dpm"])
def test_per_sample_variation_does_not_depend_on_its_batch(schedule, graph):
    kw = dict(num_surfaces=5, num_edges=4, use_cf=False, schedule=schedule, ddim_steps=12, ddim_eta=0.5, dpm_steps=12,
              noise="per_sample", graph=graph)
    a, _, _ = _run(_cfg(batch_size=5, seed=4, **kw))
    src = _fit(a, _cfg(**kw), (1, 2, 3, 4, 5))
    full, _, _ = _run(_cfg(batch_size=5, seed=21, **kw), source=_var(src, 0.5))
    for b in range(5):
        one_src = {k: src[k][b:b + 1] for k in FIELDS}
        one, _, _ = _run(_cfg(batch_size=1, seed=21, sample_base=b, **kw), source=_var(one_src, 0.5))
        for k in full:
            assert torch.equal(full[k][b], one[k][0]), (b, k)
