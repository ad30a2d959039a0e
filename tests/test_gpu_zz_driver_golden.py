"""GPU: the PRODUCT cascade driver (brepgen_b200/sampler.py: Cascade.run with the shipped PNDM/DDPM hybrid, the fused
scheduler kernels, the CFG combine and both de-duplication kernels) against the outputs of the reference's OWN sampling
block, sample.py:122-299, executed verbatim around stand-in networks (tests/golden/driver_golden.npz, written by
tests/golden/make_golden_driver.py).  The same stand-ins (plain torch functions with the reference's forward signatures)
are plugged into Cascade here, so everything between the network calls is the code under test.

Strict: no expected failures.
"""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))


@pytest.mark.parametrize("case", ["abc_like", "furniture_like"])
def test_product_driver_matches_reference_statements(case):
    import make_golden_driver as G
    from brepgen_b200.sampler import Cascade, CascadeConfig
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "driver_golden.npz"))
    use_cf, B, S0, E, seed = G.CASES[case]
    S = S0 if use_cf else 2 * S0
    src = G.NoiseSource(seed)
    init = {"surfPos": src.init((B, S0, 6)), "surfZ": src.init((B, S, 48)), "edgePos": src.init((B, S, E, 6)),
            "edgeZV": src.init((B, S, E, 18))}
    cfg = CascadeConfig(batch_size=B, num_surfaces=S0, num_edges=E, use_cf=use_cf, class_label=G.LABEL, guidance_w=G.W,
                        schedule="reference", dense_masks=False, bbox_threshold=0.08, decode=True)
    casc = Cascade(G.STANDINS, G.surf_vae, G.edge_vae, device=torch.device("cuda:0"))
    out = casc.run(cfg, init_noise=init, step_noise=lambda stage, k, shape: src.step(shape))
    for k in ("surfMask", "edgeM"):
        assert np.array_equal(out[k].cpu().numpy(), gold[f"{case}|{k}"]), k
    for k in ("surfPos", "surfZ", "edgePos", "edge_z", "edgeV", "surf_ncs", "edge_ncs"):
        ref, got = gold[f"{case}|{k}"], out[k].float().cpu().numpy()
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        err = float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30))
        assert err < 1e-4, (k, err)
