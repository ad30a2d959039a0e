"""GPU: the de-duplication kernels against the outputs of the reference's OWN statements (tests/golden/dedup_golden.npz,
written by tests/golden/make_golden_dedup.py from sample.py:159-183 and :242-261): packed boxes and masks bit-exact.

Strict: no expected failures."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "dedup_golden.npz"))
CASES = sorted(k[:-len("_surfPos_in")] for k in GOLD.files if k.endswith("_surfPos_in"))


@pytest.mark.parametrize("case", CASES)
def test_dedup_kernels_match_reference_statements(case):
    from brepgen_b200.sampler import dedup_edges, dedup_surfaces
    pos, mask = dedup_surfaces(torch.from_numpy(GOLD[f"{case}_surfPos_in"]).cuda(), 0.08)
    assert np.array_equal(mask.cpu().numpy(), GOLD[f"{case}_surfMask"])
    assert np.array_equal(pos.cpu().numpy(), GOLD[f"{case}_surfPos_out"])
    em = dedup_edges(torch.from_numpy(GOLD[f"{case}_edgePos_in"]).cuda(), mask, 0.08)
    assert np.array_equal(em.cpu().numpy(), GOLD[f"{case}_edgeM"])
