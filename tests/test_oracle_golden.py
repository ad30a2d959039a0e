"""Oracle (oracle/denoisers.py) vs golden vectors produced by the reference's own classes.

The fixtures in tests/golden/denoisers_golden.npz were written by tests/golden/make_golden.py, which
imports network.py (diffusers stubbed) and runs SurfPosNet/SurfZNet/EdgePosNet/EdgeZNet
(network.py:1066-1393) on synthetic weights.  Tolerance: fp32 re-association only (1e-5 of max|ref|).
"""
import os

import numpy as np
import pytest
import torch

from brepgen_b200.spec import denoiser_spec
from brepgen_b200.synth import synth_state_dict
from make_golden import case_inputs
from oracle import denoisers as O

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "denoisers_golden.npz"))


@pytest.mark.parametrize("kind", ["surfpos", "surfz", "edgepos", "edgez"])
@pytest.mark.parametrize("use_cf", [False, True])
def test_denoiser_matches_reference(kind, use_cf):
    sd = synth_state_dict(denoiser_spec(kind, use_cf), seed=7)
    for seed in (0, 1, 2):
        inp = case_inputs(kind, use_cf, seed)
        with torch.no_grad():
            y = O.FORWARDS[kind](sd, *inp.values()).numpy()
        ref = GOLD[f"{kind}|cf{int(use_cf)}|s{seed}"]
        assert y.shape == ref.shape
        err = np.abs(y - ref).max() / np.abs(ref).max()
        assert err < 1e-5, (kind, use_cf, seed, err)


def test_sincos_matches_reference():
    y = O.sincos_embedding(torch.tensor([0, 1, 249, 999])).numpy()
    assert np.abs(y - GOLD["sincos|surfpos"]).max() < 1e-6
    # cos block first, then sin (network.py:1060)
    assert np.allclose(y[0, :384], 1.0) and np.allclose(y[0, 384:], 0.0)


def test_dedup_oracle_matches_reference_statements():
    """oracle/cascade.py dedup loops vs the outputs of the reference's own statements (sample.py:159-183, :242-261),
    executed verbatim by tests/golden/make_golden_dedup.py: packed boxes and both masks must be IDENTICAL."""
    from oracle.cascade import dedup_edges_np, dedup_surfaces_np
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "dedup_golden.npz"))
    n = len([k for k in gold.files if k.endswith("_surfPos_in")])
    assert n >= 5
    for i in range(n):
        sp = gold[f"c{i}_surfPos_in"]
        pos, mask = dedup_surfaces_np(sp, 0.08)
        assert np.array_equal(mask, gold[f"c{i}_surfMask"]), i
        assert np.array_equal(pos, gold[f"c{i}_surfPos_out"]), i
        em = dedup_edges_np(gold[f"c{i}_edgePos_in"], mask, 0.08)
        assert np.array_equal(em, gold[f"c{i}_edgeM"]), i
        assert mask.shape == sp.shape[:2] and em.shape == gold[f"c{i}_edgePos_in"].shape[:3]


@pytest.mark.parametrize("case", ["abc_like", "furniture_like"])
def test_cascade_driver_matches_reference_statements(case):
    """oracle/cascade.py:run_cascade (the restated driver) vs the reference's own sampling block, sample.py:122-299,
    executed verbatim around stand-in networks by tests/golden/make_golden_driver.py: the shipped PNDM/DDPM hybrid, the
    classifier-free batching and combine, the late increase, both de-duplications, the zeroing of removed edges and
    the decoder input preparation.  Masks must be identical, tensors equal to fp32 round-off."""
    import make_golden_driver as G
    from brepgen_b200.sampler import CascadeConfig
    from oracle.cascade import run_cascade
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "driver_golden.npz"))
    use_cf, B, S0, E, seed = G.CASES[case]
    S = S0 if use_cf else 2 * S0
    src = G.NoiseSource(seed)
    init = {"surfPos": src.init((B, S0, 6)), "surfZ": src.init((B, S, 48)), "edgePos": src.init((B, S, E, 6)),
            "edgeZV": src.init((B, S, E, 18))}
    cfg = CascadeConfig(batch_size=B, num_surfaces=S0, num_edges=E, use_cf=use_cf, class_label=G.LABEL, guidance_w=G.W,
                        schedule="reference", dense_masks=False, bbox_threshold=0.08)
    out = run_cascade(None, cfg, init, lambda stage, k, shape: src.step(shape), forwards=G.STANDINS,
                      surf_vae=G.surf_vae, edge_vae=G.edge_vae)
    for k in ("surfMask", "edgeM"):
        assert np.array_equal(out[k].numpy(), gold[f"{case}|{k}"]), k
    for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV", "surf_ncs", "edge_ncs"):
        ref = gold[f"{case}|{k}"]
        got = out[k].numpy()
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        assert np.allclose(got, ref, rtol=1e-5, atol=1e-6), (k, float(np.abs(got - ref).max()))


def test_oracle_matches_reference_at_benchmark_shape():
    """the restatement against the reference's own EdgeZNet at S = 100, E = 40 (L = 4000), B = 3, ragged face masks plus
    30 % random edge masks (tests/golden/make_golden_l4000.py): the L > 128, masked path at the benchmark's own shape"""
    from make_golden_l4000 import CASES, case_inputs_l4000
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "denoisers_l4000_golden.npz"))
    name = "edgez_ragged_b3"
    spec = CASES[name]
    inp, valid = case_inputs_l4000(spec)
    sd = synth_state_dict(denoiser_spec(spec[0], spec[1]), seed=7)
    with torch.no_grad():
        y = O.FORWARDS[spec[0]](sd, *inp.values())
    ref = torch.from_numpy(gold[name])
    err = float((y[valid] - ref[valid]).abs().max() / ref[valid].abs().max())
    assert err < 2e-5, err
