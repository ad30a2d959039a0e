"""Golden vectors AT THE BENCHMARK'S OWN SHAPES from the reference's OWN classes (run in the build container only).

    python tests/golden/make_golden_l4000.py        # writes tests/golden/denoisers_l4000_golden.npz

BASELINE.json configs[2] runs the edge stages at S = 100 faces x E = 40 edges = ONE sequence of L = 4000 tokens per sample
(network.py:1257-1286, 1357-1393).  The small goldens of make_golden.py (L = 5 / 15) only reach the
single-key-block attention path; these cases pin the exact kernel instantiation the headline number is measured on
(flash attention over 32 key blocks, block lists with fully padded 128-key blocks, ragged masks, B >= 2 so the
per-sample batch pitch of every buffer is exercised):

  edgepos_dense_b2      EdgePosNet, cf off, B = 2, nothing masked, scalar timestep
  edgepos_ragged_b3_cf  EdgePosNet, cf on,  B = 3, face masks leaving whole key blocks padded, per-sample timesteps
  edgez_ragged_b3       EdgeZNet,   cf off, B = 3, ragged faces + 30 % random edge masks, scalar timestep
  edgez_dense_b2_cf     EdgeZNet,   cf on,  B = 2, nothing masked, per-sample timesteps
  edgepos_chain4_b2     4 DDPM steps (t = 999..996, injected noise) of EdgePosNet, B = 2, one sample ragged:
                        x after the 4th step (reference class forward + oracle/schedulers.py DDPM step)

Only outputs are stored; inputs and weights are regenerated from seeds (`case_inputs_l4000`, synth_state_dict(seed=7)).
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

S, E = 100, 40
CASES = {
    # name: (kind, use_cf, B, valid faces per sample, random edge-mask probability, timesteps, seed)
    "edgepos_dense_b2": ("edgepos", False, 2, [100, 100], 0.0, [500], 11),
    "edgepos_ragged_b3_cf": ("edgepos", True, 3, [100, 37, 61], 0.0, [999, 249, 3], 12),
    "edgez_ragged_b3": ("edgez", False, 3, [100, 23, 64], 0.3, [10], 13),
    "edgez_dense_b2_cf": ("edgez", True, 2, [100, 100], 0.0, [750, 0], 14),
}
CHAIN = ("edgepos", False, 2, [100, 50], 0.0, [999, 998, 997, 996], 15)


def case_inputs_l4000(spec):
    """ordered dict of forward arguments (reference signature order) + the per-token validity mask (B, S, E)"""
    kind, use_cf, B, nvalid, p_edge, ts, seed = spec
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    surf_mask = torch.arange(S)[None, :] >= torch.tensor(nvalid)[:, None]            # True = padded face
    edge_mask = surf_mask[..., None].repeat(1, 1, E)
    if p_edge > 0:
        edge_mask = edge_mask | (torch.rand(B, S, E, generator=g) < p_edge)
        edge_mask[:, 0, 0] = False
    label = torch.tensor([[6], [0], [10]][:B]) if use_cf else None
    t = torch.tensor(ts)
    if kind == "edgepos":
        inp = dict(edgePos=r(B, S, E, 6), timesteps=t, surfPos=r(B, S, 6), surfZ=r(B, S, 48), mask=surf_mask,
                   class_label=label)
        valid = ~surf_mask[..., None].expand(B, S, E)
    else:
        inp = dict(edge=r(B, S, E, 18), timesteps=t, edgePos=r(B, S, E, 6), surfPos=r(B, S, 6), surfZ=r(B, S, 48),
                   mask=edge_mask, class_label=label)
        valid = ~edge_mask
    return inp, valid


def chain_noise(k, shape):
    return torch.randn(shape, generator=torch.Generator().manual_seed(1000 + k))


def main():
    from brepgen_b200.spec import denoiser_spec
    from brepgen_b200.synth import synth_state_dict
    from oracle.reference_loader import load_reference_network
    from oracle.schedulers import DDPMOracle

    network = load_reference_network()
    classes = {"edgepos": network.EdgePosNet, "edgez": network.EdgeZNet}
    torch.set_num_threads(os.cpu_count() or 1)
    out = {}

    def model(kind, use_cf):
        m = classes[kind](use_cf)
        m.load_state_dict(synth_state_dict(denoiser_spec(kind, use_cf), seed=7))
        return m.eval()

    for name, spec in CASES.items():
        inp, _ = case_inputs_l4000(spec)
        m = model(spec[0], spec[1])
        t0 = time.time()
        with torch.no_grad():
            y = m(*[v.clone() if torch.is_tensor(v) else v for v in inp.values()])
        out[name] = y.numpy().astype(np.float32)
        print(f"{name}: {tuple(y.shape)} in {time.time() - t0:.1f} s", flush=True)

    # 4-step DDPM chain: the reference's loop body (sample.py:145-153) with explicit step noise
    inp, _ = case_inputs_l4000(CHAIN)
    m = model(CHAIN[0], CHAIN[1])
    orc = DDPMOracle()
    x = inp["edgePos"].clone()
    with torch.no_grad():
        for k, t in enumerate(CHAIN[5]):
            pred = m(x, torch.tensor([t]), inp["surfPos"], inp["surfZ"], inp["mask"], None)
            x = orc.step(pred, t, x, chain_noise(k, x.shape))
    out["edgepos_chain4_b2"] = x.numpy().astype(np.float32)

    path = os.path.join(ROOT, "tests", "golden", "denoisers_l4000_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()}, os.path.getsize(path))


if __name__ == "__main__":
    main()
