"""CPU tests of B-rep variations (Cascade.run(source=Variation(...))): strength_timesteps written out, the oracle's slot fill
against the reference's own pad_repeat (tests/golden/fill_golden.npz), the variation oracle's kept stages, the host checks
(nothing launched) and, with a recording stand-in for the library, what each stage launches."""
import ctypes
import os

import numpy as np
import pytest
import torch

from brepgen_b200.sampler import Cascade, CascadeConfig, Variation, check_variation
from brepgen_b200.schedulers import (DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler, dpm_timesteps,
                                     sample_keys, strength_timesteps)
from oracle.variation import fill_rows, pad_repeat_positions, run_cascade_variation
from test_completion import _RecordingLib, _bank, _init, _stand_ins, fake_lib  # noqa: F401  (fake_lib: fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGES = ("surfPos", "surfZ", "edgePos", "edgeZV")


# ------------------------------------------------------------------------------------------------ strength -> steps
def test_strength_timesteps_written_out():
    s = DDPMScheduler()
    s.set_timesteps(1000)
    assert strength_timesteps(s.timesteps, 0.25).tolist() == list(range(249, -1, -1))
    d = DDIMScheduler()
    d.set_timesteps(50)
    assert strength_timesteps(d.timesteps, 0.3).tolist() == list(range(280, -1, -20))
    assert len(strength_timesteps(d.timesteps, 0.3)) == 15
    ts = dpm_timesteps(1000, 20, "linspace")
    assert strength_timesteps(torch.from_numpy(ts), 0.5).tolist() == ts[10:].tolist()
    p = DPMSolverMultistepScheduler()
    p.set_timesteps(20)
    assert strength_timesteps(p.timesteps, 0.5).tolist() == ts[10:].tolist()
    for full in (s.timesteps, d.timesteps, p.timesteps):
        assert torch.equal(strength_timesteps(full, 1.0), full)
        assert len(strength_timesteps(full, 0.0)) == 0
    assert len(strength_timesteps(d.timesteps, 0.999)) == 49          # int(50 * 0.999) = 49, as diffusers truncates


@pytest.mark.parametrize("strength,n", [(-0.1, 50), (1.01, 50), (0.01, 50), (0.09, 10), (float("nan"), 10)])
def test_strength_timesteps_errors(strength, n):
    d = DDIMScheduler()
    d.set_timesteps(n)
    with pytest.raises(ValueError):
        strength_timesteps(d.timesteps, strength)


# ---------------------------------------------------------------------------------------------------- fill layout
def test_oracle_fill_equals_reference_pad_repeat():
    gold = np.load(os.path.join(ROOT, "tests", "golden", "fill_golden.npz"))
    assert sorted(gold.files) == ["S100", "S30", "S40", "S50"]
    for key in gold.files:
        S = int(key[1:])
        assert gold[key].shape == (S, S)
        for n in range(1, S + 1):
            assert pad_repeat_positions(n, S) == gold[key][n - 1].tolist(), (S, n)


def test_fill_rows_takes_valid_slots_in_order():
    mask = np.array([[False, True, False, True], [True, True, True, True], [False, False, False, False]])
    got = fill_rows(mask, 5, row_map=[0, 1, -1, 2])
    assert got[0] == [0, 0, 0, 2, 2] and got[1] == [-1] * 5 and got[2] == [-1] * 5
    assert got[3] == [8, 8, 9, 10, 11]


# ---------------------------------------------------------------------------------------------------------- oracle
def _cfg(**kw):
    base = dict(batch_size=2, num_surfaces=5, num_edges=4, schedule="ddim", ddim_steps=6, decode=False, graph="off")
    base.update(kw)
    return CascadeConfig(**base)


def _source(cfg, seed=1):
    from oracle.ddim import run_cascade_ddim
    n, _ = _bank(seed)
    return run_cascade_ddim(None, cfg, _init(cfg, seed), n, _stand_ins())


def _start_noise(cfg, st, seed=3):
    """start noise of every varied stage, in its starting shape"""
    g = torch.Generator().manual_seed(seed)
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    S = S0 if cfg.use_cf else 2 * S0
    d = DDIMScheduler()
    d.set_timesteps(cfg.ddim_steps)
    t0 = int(strength_timesteps(d.timesteps, st[0])[0]) if st[0] > 0 else 0
    S1 = S0 if (not cfg.use_cf and t0 > 249) else S
    return {"surfPos": torch.randn(B, S1, 6, generator=g), "surfZ": torch.randn(B, S, 48, generator=g),
            "edgePos": torch.randn(B, S, E, 6, generator=g), "edgeZV": torch.randn(B, S, E, 18, generator=g)}


@pytest.mark.parametrize("use_cf", [False, True])
def test_oracle_with_zero_strengths_returns_the_source(use_cf):
    cfg = _cfg(use_cf=use_cf, class_label=3)
    out = _source(cfg)
    n, bank = _bank(5)
    got = run_cascade_variation(None, cfg, Variation.from_outputs(out, 0.0), {}, n, _stand_ins())
    assert not bank
    for k in out:
        assert torch.equal(got[k], out[k]), k


@pytest.mark.parametrize("st", [(0, 0, 0.5, 0.5), (0, 0, 0, 1.0), (0, 0.5, 0.5, 0.5), (0.34, 0.5, 0.5, 0.5)])
def test_oracle_keeps_a_zero_prefix(st):
    cfg = _cfg(ddim_eta=0.5)
    out = _source(cfg)
    n, bank = _bank(5)
    got = run_cascade_variation(None, cfg, Variation.from_outputs(out, st), _start_noise(cfg, st), n, _stand_ins())
    kept = {"surfPos": ("surfPos", "surfMask"), "surfZ": ("surfZ",), "edgePos": ("edgePos", "edgeM"),
            "edgeZV": ("edge_z", "edgeV")}
    for name, s in zip(STAGES, st):
        for k in kept[name]:
            if s == 0:
                assert torch.equal(got[k], out[k]), (name, k)
            elif got[k].dtype != torch.bool:          # a varied stage's masks may come out as they were
                assert not torch.equal(got[k], out[k]), (name, k)
    assert {name for name, _, _ in bank} == {name for name, s in zip(STAGES, st) if s > 0}


# -------------------------------------------------------------------------------------------------- host checks
def _var(cfg, strength=0.5, **over):
    g = torch.Generator().manual_seed(0)
    B, E = cfg.batch_size, cfg.num_edges
    S = cfg.num_surfaces if cfg.use_cf else 2 * cfg.num_surfaces
    fields = dict(surfPos=torch.rand(B, S, 6, generator=g), surfMask=torch.arange(S)[None, :].expand(B, S) >= 3,
                  surfZ=torch.randn(B, S, 48, generator=g), edgePos=torch.rand(B, S, E, 6, generator=g),
                  edgeM=torch.arange(E)[None, None, :].expand(B, S, E) >= 2, edge_z=torch.randn(B, S, E, 12, generator=g),
                  edgeV=torch.randn(B, S, E, 6, generator=g))
    fields.update(over)
    return Variation(**fields, strength=strength)


def _bad_cases():
    c = _cfg()
    many = torch.arange(10)[None, :].expand(2, 10) >= 7          # 7 valid faces, more than num_surfaces = 5
    slot0 = _var(c).edgeM.clone()
    slot0[1, 2, 0] = True
    return [
        ("schedule reference", dict(schedule="reference"), _var(c), NotImplementedError),
        ("schedule repaint", dict(schedule="repaint"), _var(c), NotImplementedError),
        ("dense masks", dict(dense_masks=True), _var(c), ValueError),
        ("ragged masks", dict(ragged_masks=True), _var(c), ValueError),
        ("batch size", dict(batch_size=3), _var(c), ValueError),
        ("num_edges", dict(num_edges=5), _var(c), ValueError),
        ("cfg slots", dict(use_cf=True), _var(c), ValueError),
        ("surfZ shape", {}, _var(c, surfZ=torch.zeros(2, 10, 47)), ValueError),
        ("edgeV shape", {}, _var(c, edgeV=torch.zeros(2, 10, 4, 5)), ValueError),
        ("surfMask dtype", {}, _var(c, surfMask=torch.zeros(2, 10)), ValueError),
        ("edgeM dtype", {}, _var(c, edgeM=torch.zeros(2, 10, 4, dtype=torch.uint8)), ValueError),
        ("surfZ dtype", {}, _var(c, surfZ=torch.zeros(2, 10, 48, dtype=torch.int32)), ValueError),
        ("three strengths", {}, _var(c, strength=(0.5, 0.5, 0.5)), ValueError),
        ("strength > 1", {}, _var(c, strength=1.5), ValueError),
        ("strength < 0", {}, _var(c, strength=(0, 0, -0.1, 0.5)), ValueError),
        ("strength without a step", {}, _var(c, strength=(0.1, 0.5, 0.5, 0.5)), ValueError),
        ("zero after a varied stage", {}, _var(c, strength=(0.5, 0, 0.5, 0.5)), ValueError),
        ("zero last", {}, _var(c, strength=(0, 0, 0.5, 0)), ValueError),
        ("more faces than the starting slots", {}, _var(c, strength=0.9, surfMask=many), ValueError),
        ("edge slot 0 padded on a valid face", {}, _var(c, edgeM=slot0), ValueError),
    ]


@pytest.mark.parametrize("name,cfg_kw,source,exc", _bad_cases(), ids=[c[0] for c in _bad_cases()])
def test_bad_variations_raise_before_any_launch(fake_lib, name, cfg_kw, source, exc):
    with pytest.raises(exc):
        Cascade({}, device="cpu").run(_cfg(**cfg_kw), source=source)
    assert fake_lib.calls == []


def test_variation_with_completion_is_rejected(fake_lib):
    from test_completion import _known
    with pytest.raises(ValueError, match="known"):
        Cascade({}, device="cpu").run(_cfg(num_edges=4), source=_var(_cfg()), known=_known(n=(1, 1), K=3, E=4))
    assert fake_lib.calls == []


def test_more_faces_fit_when_the_list_starts_after_the_late_increase():
    """7 valid faces exceed num_surfaces = 5 but fit the 10 slots a non-CFG run has from t <= 249 on"""
    many = torch.arange(10)[None, :].expand(2, 10) >= 7
    c = _cfg()
    with pytest.raises(ValueError, match="below 0.5"):              # DDIM-6: 166, 0 start at t <= 249: s < 3/6
        check_variation(c, _var(c, strength=0.5, surfMask=many))
    assert check_variation(c, _var(c, strength=(0.34, 0.5, 1, 1), surfMask=many)) == (0.34, 0.5, 1.0, 1.0)


# ------------------------------------------------------------------------------------------- what the stages launch
class _ReadingLib(_RecordingLib):
    """_RecordingLib that also copies, at call time, the keys and the explicit noise of every bg_add_noise_gather (host
    pointers of CPU tensors here)"""

    def __init__(self):
        super().__init__()
        self.starts = []

    def bg_add_noise_gather(self, src, n_src, index, n_tok, dim, scale, sa, sb, noise, keys, tps, domain, t, out, st):
        rec = dict(n_tok=n_tok, dim=dim, scale=scale, sa=sa, sb=sb, tps=tps, domain=domain, t=t, keys=None, noise=None)
        if keys is not None:
            rec["keys"] = list((ctypes.c_uint64 * (n_tok // tps)).from_address(keys))
        if noise is not None:
            rec["noise"] = torch.tensor(list((ctypes.c_float * (n_tok * dim)).from_address(noise)))
        self.starts.append(rec)
        self.calls.append(("bg_add_noise_gather", None))
        return 0


@pytest.fixture
def reading_lib(fake_lib, monkeypatch):
    from brepgen_b200 import _ffi
    lib = _ReadingLib()
    monkeypatch.setattr(_ffi, "lib", lambda: lib)
    return lib


def _stand_in_models(counts):
    def net(kind):
        def f(x, t, *rest):
            counts[kind] += 1
            return torch.zeros_like(x)
        return f
    return {k: net(k) for k in ("surfpos", "surfz", "edgepos", "edgez")}


@pytest.mark.parametrize("st", [(0.5, 0.5, 0.5, 0.5), (0, 0, 0.5, 1.0), (0, 0, 0, 0)])
def test_per_sample_starts_take_the_stage_keys_at_domain_1(reading_lib, st):
    cfg = _cfg(noise="per_sample", seed=4, sample_base=2)
    counts = dict.fromkeys(("surfpos", "surfz", "edgepos", "edgez"), 0)
    Cascade(_stand_in_models(counts), device="cpu").run(cfg, source=_var(cfg, strength=st))
    from brepgen_b200.sampler import per_sample_seeds
    seeds = per_sample_seeds(cfg)
    varied = [i for i, s in enumerate(st) if s > 0]
    assert len(reading_lib.starts) == len(varied)
    for rec, i in zip(reading_lib.starts, varied):
        assert rec["keys"] == sample_keys(seeds, i).tolist() and rec["noise"] is None
        assert (rec["domain"], rec["t"], rec["scale"]) == (1, 0, 3.0 if i in (0, 2) else 1.0)
        assert rec["n_tok"] == cfg.batch_size * rec["tps"]
    # forwards: int(N * s) per varied stage, none per kept one
    want = [int(6 * s) for s in st]
    assert [counts[k] for k in ("surfpos", "surfz", "edgepos", "edgez")] == want


def test_batch_mode_kept_stages_draw_nothing(reading_lib):
    cfg = _cfg(seed=9)
    st = (0, 0, 0.5, 0.5)
    Cascade(_stand_in_models(dict.fromkeys(("surfpos", "surfz", "edgepos", "edgez"), 0)), device="cpu").run(
        cfg, source=_var(cfg, strength=st))
    g = torch.Generator().manual_seed(9)
    B, S, E = 2, 10, 4
    assert len(reading_lib.starts) == 2
    for rec, shape in zip(reading_lib.starts, ((B, S, E, 6), (B, S, E, 18))):
        assert rec["keys"] is None and torch.equal(rec["noise"], torch.randn(shape, generator=g).flatten())
        a = DDPMScheduler().alphas_cumprod[332]                      # DDIM-6 at s = 0.5: 332, 166, 0
        assert (rec["sa"], rec["sb"]) == (float(a ** 0.5), float((1 - a) ** 0.5))


def test_init_noise_overrides_the_start_noise(reading_lib):
    cfg = _cfg(noise="per_sample")
    z = torch.randn(2, 10, 4, 18)
    Cascade(_stand_in_models(dict.fromkeys(("surfpos", "surfz", "edgepos", "edgez"), 0)), device="cpu").run(
        cfg, source=_var(cfg, strength=(0, 0, 0, 0.5)), init_noise={"edgeZV": z})
    (rec,) = reading_lib.starts
    assert rec["keys"] is None and torch.equal(rec["noise"], z.flatten())


def test_dpm_graph_table_of_a_truncated_list_starts_first_order(fake_lib, monkeypatch):
    seen = []

    def loop_graph(self, cfg, sched, timesteps, x, fwd, known=None, tables=None):
        seen.append((timesteps.tolist(), tables[0].clone()))
        return x
    monkeypatch.setattr(Cascade, "_loop_graph", loop_graph)
    cfg = _cfg(schedule="dpm", dpm_steps=10, graph="on", use_cf=True, num_surfaces=10)
    Cascade(_stand_in_models(dict.fromkeys(("surfpos", "surfz", "edgepos", "edgez"), 0)), device="cpu").run(
        cfg, source=_var(cfg, strength=(0, 0, 0.5, 0.5)))
    p = DPMSolverMultistepScheduler(solver_order=2)
    p.set_timesteps(10)
    assert [ts for ts, _ in seen] == [p.timesteps[5:].tolist()] * 2
    for _, tab in seen:
        assert tab.shape == (5, 7)
        assert tab[0, 4] == 0 and tab[0, 5] == 0                       # c_1 = inv_r0 = 0: first order
        assert (tab[1:-1, 4] != 0).all()                              # then second order up to the last step
        assert torch.equal(tab[1:], p.coefficient_table(p.timesteps)[6:])
