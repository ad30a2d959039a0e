"""Per-sample classifier-free guidance, host side (no GPU): the forward-batch layout of sampler.Guidance, the host checks
of check_guidance, shard_config's slicing, the rows and combines a whole cascade issues (recorded by a stand-in library),
and the stacked oracle of oracle/guidance.py against one batched oracle run."""
import math

import pytest
import torch

from brepgen_b200.sampler import (TEXT2INT, Cascade, CascadeConfig, Guidance, check_guidance, per_sample_guidance,
                                  shard_config)
from test_completion import fake_lib  # noqa: F401  (fixture)


def _cfg(**kw):
    base = dict(batch_size=4, num_surfaces=3, num_edges=2, use_cf=True, class_label=6, schedule="ddpm", ddpm_steps=3,
                decode=False, graph="off")
    base.update(kw)
    return CascadeConfig(**base)


def _labels(g):
    return g.label.flatten().tolist()


# ------------------------------------------------------------------------------------------------ layout
def test_scalar_mode_is_the_reference_layout():
    g = Guidance(_cfg(guidance_w=0.6), "cpu")
    assert not g.per_sample and g.rows == 8
    assert _labels(g) == [6] * 4 + [0] * 4
    assert g.label.dtype == torch.int64 and g.label.shape == (8, 1)
    t = torch.arange(4.0)
    assert torch.equal(g.double(t), torch.cat([t, t]))
    pred = torch.randn(8, 5)
    pc, pu, w = g.split(pred)
    assert torch.equal(pc, pred[:4]) and torch.equal(pu, pred[4:]) and w == 0.6


def test_scalar_negative_label_only_changes_the_labels():
    g = Guidance(_cfg(negative_label="chair"), "cpu")
    assert not g.per_sample and _labels(g) == [6] * 4 + [TEXT2INT["chair"]] * 4 and g.rows == 8


def test_no_cfg_is_the_batch_itself():
    g = Guidance(_cfg(use_cf=False), "cpu")
    t = torch.randn(4, 3)
    assert g.label is None and g.rows == 4 and g.double(t) is t
    assert g.split(t)[0] is t and g.split(t)[1] is None


def test_mixed_labels_and_zero_weights():
    g = Guidance(_cfg(class_label=["chair", 10, 9, 1], guidance_w=[0.5, 0.0, 2.0, 0.0], negative_label=[0, 0, 6, 3]),
                 "cpu")
    assert g.per_sample and g.G == 2 and g.rows == 6
    assert _labels(g) == [6, 10, 9, 1, 0, 6]            # conditional rows, then the guided samples' negatives
    assert g.g.tolist() == [0, 2]
    assert g.uncond_row.tolist() == [0, -1, 1, -1] and g.uncond_row.dtype == torch.int32
    assert g.w_dev.tolist() == [0.5, 0.0, 2.0, 0.0] and g.w_dev.dtype == torch.float32
    t = torch.arange(4.0)[:, None]
    assert g.double(t).flatten().tolist() == [0, 1, 2, 3, 0, 2]


def test_all_zero_weights_need_no_unconditional_rows():
    g = Guidance(_cfg(guidance_w=[0.0] * 4), "cpu")
    t = torch.randn(4, 2)
    assert g.G == 0 and g.rows == 4 and _labels(g) == [6] * 4 and g.double(t) is t


def test_uniform_per_sample_fields_keep_every_row():
    g = Guidance(_cfg(guidance_w=[0.6] * 4), "cpu")
    assert g.per_sample and g.rows == 8 and _labels(g) == [6] * 4 + [0] * 4 and g.uncond_row.tolist() == [0, 1, 2, 3]


def test_copies_are_guided_as_their_sample():
    """an interpolation inverts both designs of sample b under sample b's fields"""
    g = Guidance(_cfg(batch_size=2, class_label=[1, 2], guidance_w=[0.0, 1.5], negative_label=[0, 4]), "cpu", n=4)
    assert _labels(g) == [1, 2, 1, 2, 4, 4] and g.uncond_row.tolist() == [-1, 0, -1, 1]


def test_names_resolve_through_text2int():
    cls, neg, w = check_guidance(_cfg(class_label=["bathtub", "table", 3, "uncond"], negative_label="lamp"))
    assert cls == [1, 10, 3, 0] and neg == [8] * 4 and w == [0.6] * 4


def test_per_sample_mode_is_on_when_any_field_is_a_sequence():
    assert not per_sample_guidance(_cfg())
    assert per_sample_guidance(_cfg(negative_label=(0, 0, 0, 0)))
    assert per_sample_guidance(_cfg(guidance_w=torch.full((4,), 0.6)))


# ------------------------------------------------------------------------------------------------ host checks
@pytest.mark.parametrize("kw,exc", [
    (dict(class_label=[6, 6, 6]), ValueError),                               # wrong length
    (dict(guidance_w=[0.6] * 5), ValueError),
    (dict(negative_label=[0, 0]), ValueError),
    (dict(use_cf=False, class_label=[6] * 4), ValueError),                   # per-sample fields without CFG
    (dict(use_cf=False, guidance_w=[0.0] * 4), ValueError),
    (dict(use_cf=False, negative_label=3), ValueError),                      # a negative label without CFG
    (dict(class_label=11), ValueError),                                      # outside the embedding's rows
    (dict(class_label=[0, 1, -1, 2]), ValueError),
    (dict(negative_label=[0, 0, 0, 12]), ValueError),
    (dict(class_label=2.5), ValueError),
    (dict(class_label=["chair", "spaceship", 0, 0]), KeyError),              # unknown names, as config_from_eval_args
    (dict(negative_label="spaceship"), KeyError),
    (dict(guidance_w=[0.6, math.inf, 0.6, 0.6]), ValueError),                # non-finite w
    (dict(guidance_w=math.nan), ValueError),
])
def test_bad_guidance_raises_before_any_launch(fake_lib, kw, exc):
    with pytest.raises(exc):
        Cascade({}, device="cpu").run(_cfg(**kw))
    assert fake_lib.calls == []


def test_no_cfg_accepts_the_defaults():
    assert check_guidance(_cfg(use_cf=False, class_label=3, negative_label="uncond")) is None


def test_shard_config_slices_the_per_sample_fields():
    cfg = _cfg(batch_size=5, class_label=[1, 2, 3, 4, 5], guidance_w=[0.0, 0.1, 0.2, 0.3, 0.4], negative_label=7)
    parts = [shard_config(cfg, 5, r, 2) for r in range(2)]
    assert [p.class_label for p in parts] == [[1, 2, 3], [4, 5]]
    assert [p.guidance_w for p in parts] == [[0.0, 0.1, 0.2], [0.3, 0.4]]
    assert [p.negative_label for p in parts] == [7, 7]
    assert [p.sample_base for p in parts] == [0, 3]
    with pytest.raises(ValueError, match="class_label"):
        shard_config(_cfg(class_label=[1, 2, 3]), 4, 0, 2)


# ------------------------------------------------------------------------------------------------ whole cascades
def _recording_models(rows):
    def net(kind):
        def f(x, t, *rest):
            rows.append((kind, x.shape[0], None if rest[-1] is None else rest[-1].flatten().tolist(),
                         [r.shape[0] for r in rest[:-1]]))
            return torch.zeros_like(x)
        return f
    return {k: net(k) for k in ("surfpos", "surfz", "edgepos", "edgez")}


@pytest.mark.parametrize("schedule", ["reference", "ddpm", "ddim", "dpm", "unipc", "repaint"])
def test_forward_rows_and_combines_of_a_mixed_batch(fake_lib, schedule):
    rows = []
    cfg = _cfg(schedule=schedule, ddim_steps=3, dpm_steps=3, unipc_steps=3, repaint_steps=3, repaint_jump_length=1,
               repaint_jump_n_sample=1, class_label=[6, 9, 10, 1], guidance_w=[0.5, 0.0, 1.0, 0.0],
               negative_label=[2, 0, 0, 0], dense_masks=schedule != "repaint")
    Cascade(_recording_models(rows), device="cpu").run(cfg)
    assert rows and all(n == 6 and lab == [6, 9, 10, 1, 2, 0] for _, n, lab, _ in rows)
    assert all(set(cond) <= {6} for *_, cond in rows)                    # conditioning doubled as x is
    comb = fake_lib.named("bg_cfg_combine")
    assert len(comb) == len(rows)
    assert all(a[4:6] == (4, 2) and a[0] == a[7] for a in comb)        # in place, n = 4 samples, G = 2 guided
    for name, args in fake_lib.calls:                                    # every step runs without an uncond input
        if name.endswith("_step") or name.endswith("_step_tab"):
            if name not in ("bg_pndm_step",):
                assert args[1] is None, name
    assert not fake_lib.named("bg_axpby")


def test_scalar_cascade_issues_no_combine(fake_lib):
    rows = []
    Cascade(_recording_models(rows), device="cpu").run(_cfg(schedule="ddim", ddim_steps=2, dense_masks=True))
    assert all(n == 8 and lab == [6] * 4 + [0] * 4 for _, n, lab, _ in rows)
    assert not fake_lib.named("bg_cfg_combine")
    assert all(a[1] is not None for a in fake_lib.named("bg_ddim_step"))


def test_all_unguided_cascade_runs_at_half_the_rows(fake_lib):
    rows = []
    Cascade(_recording_models(rows), device="cpu").run(_cfg(guidance_w=[0.0] * 4, dense_masks=True))
    assert rows and all(n == 4 and lab == [6] * 4 for _, n, lab, _ in rows)
    assert not fake_lib.named("bg_cfg_combine")


# ------------------------------------------------------------------------------------------------ oracle composition
def test_stacked_oracle_with_uniform_fields_equals_one_batched_run():
    from brepgen_b200.spec import denoiser_spec
    from brepgen_b200.synth import synth_state_dict
    from oracle.ddim import run_cascade_ddim
    from oracle.guidance import run_stacked, take
    sds = {k: synth_state_dict(denoiser_spec(k, True), seed=11) for k in ("surfpos", "surfz", "edgepos", "edgez")}
    B, S, E = 2, 3, 2
    cfg = _cfg(batch_size=B, num_surfaces=S, num_edges=E, schedule="ddim", ddim_steps=2, ddim_eta=1.0, dense_masks=True,
               guidance_w=0.7)
    g = torch.Generator().manual_seed(5)
    init = {"surfPos": torch.randn(B, S, 6, generator=g), "surfZ": torch.randn(B, S, 48, generator=g),
            "edgePos": torch.randn(B, S, E, 6, generator=g), "edgeZV": torch.randn(B, S, E, 18, generator=g)}
    bank = {}

    def step_noise(name, k, shape):
        if (name, k) not in bank:
            bank[(name, k)] = torch.randn((B,) + tuple(shape[1:]), generator=g)
        return bank[(name, k)]
    ref = run_cascade_ddim(sds, cfg, init, step_noise)
    got = run_stacked(run_cascade_ddim, sds, cfg, [6] * B, [0] * B, [0.7] * B,
                      lambda b: ((take(init, b, B), lambda n, k, s, b=b: step_noise(n, k, s)[b:b + 1]), {}))
    for k in ref:
        if ref[k].dtype == torch.bool:
            assert torch.equal(got[k], ref[k]), k
        else:
            err = float((got[k].double() - ref[k].double()).norm() / ref[k].double().norm())
            assert err < 1e-5, (k, err)


def test_negative_forwards_relabel_the_unconditional_half():
    from oracle.guidance import negative_forwards
    seen = []
    f = negative_forwards({"surfpos": lambda x, t, lab: seen.append(lab.flatten().tolist())}, 4)
    f["surfpos"](None, None, torch.tensor([[6], [0]]))
    assert seen == [[6, 4]]
    base = {"surfpos": object()}
    assert negative_forwards(base, 0) is base
