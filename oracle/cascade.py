"""ORACLE (test infrastructure): CPU restatement of the cascade driver sample.py:120-299.

sample.py itself cannot be imported here (it imports OpenCASCADE at :9 and hard-codes .cuda() at :48,130,...), so the
loop is restated device-agnostically around the oracle denoisers (oracle/denoisers.py, pinned to the reference's own
classes) and the oracle schedulers (oracle/schedulers.py, parity unpinned).  The de-duplication loops follow
sample.py:159-183 and :242-261 statement by statement (numpy, fp32).

Pinned: tests/golden/dedup_golden.npz and tests/golden/driver_golden.npz hold outputs of the reference's OWN statements
(sample.py:159-183, :242-261 and the whole sampling block :122-299), which tests/golden/make_golden_dedup.py and
make_golden_driver.py read from the reference file and exec() verbatim (the driver around stand-in networks and the
oracle schedulers); tests/test_oracle_golden.py requires identical masks and matching tensors from this restatement.
"""
from __future__ import annotations

import numpy as np
import torch

from . import denoisers as O
from .schedulers import DDPMOracle, PNDMOracle


def dedup_surfaces_np(surfPos: np.ndarray, thr: float):
    """surfPos (B,S,6) fp32 -> (packed (B,S,6), mask (B,S) bool True = padded); sample.py:159-183"""
    B, S, _ = surfPos.shape
    out = np.zeros_like(surfPos)
    mask = np.ones((B, S), dtype=bool)
    for ii in range(B):
        bboxes = np.round(surfPos[ii].reshape(S, 2, 3), 4)
        non_repeat = bboxes[:1]
        for bbox in bboxes:
            diff = np.max(np.max(np.abs(non_repeat - bbox), -1), -1)
            same = diff < thr
            diff_rev = np.max(np.max(np.abs(non_repeat - bbox[::-1]), -1), -1)
            same_rev = diff_rev < thr
            if same.sum() >= 1 or same_rev.sum() >= 1:
                continue
            non_repeat = np.concatenate([non_repeat, bbox[np.newaxis]], 0)
        n = len(non_repeat)
        out[ii, :n] = non_repeat.reshape(n, -1)
        mask[ii, :n] = False
    return out, mask


def dedup_edges_np(edgePos: np.ndarray, surfMask: np.ndarray, thr: float):
    """edgePos (B,S,E,6), surfMask (B,S) -> edgeM (B,S,E) bool; sample.py:242-261"""
    B, S, E, _ = edgePos.shape
    edgeM = np.repeat(surfMask[:, :, None], E, axis=2).copy()
    for ii in range(B):
        edge_bboxs = edgePos[ii][~surfMask[ii]]
        for surf_idx, bboxes in enumerate(edge_bboxs):
            bboxes = bboxes.reshape(len(bboxes), 2, 3)
            valid = bboxes[0:1]
            for bbox_idx, bbox in enumerate(bboxes):
                diff = np.max(np.max(np.abs(valid - bbox), -1), -1)
                diff_rev = np.max(np.max(np.abs(valid - bbox[::-1]), -1), -1)
                if (diff < thr).sum() >= 1 or (diff_rev < thr).sum() >= 1:
                    edgeM[ii, surf_idx, bbox_idx] = True
                    continue
                valid = np.concatenate([valid, bbox[np.newaxis]], 0)
            edgeM[ii, surf_idx, 0] = False
    return edgeM


def run_cascade(sds, cfg, init_noise, step_noise, forwards=None, surf_vae=None, edge_vae=None):
    """sds: {'surfpos','surfz','edgepos','edgez'} state dicts; cfg: brepgen_b200.sampler.CascadeConfig-like object;
    init_noise: dict name -> tensor; step_noise(stage, i, shape) -> tensor (DDPM noise injected at step i).
    Only the 'ddpm' schedule and the 'reference' hybrid for non-CFG / CFG are restated.
    forwards: optional {'surfpos','surfz','edgepos','edgez'} callables with the reference's forward signatures, used
    instead of the oracle denoisers (the driver itself is pinned this way against the reference's own statements executed
    around cheap stand-in networks, tests/golden/make_golden_driver.py).  surf_vae / edge_vae: optional decoders; when
    given, the decode input preparation of sample.py:289-293 is restated too (outputs 'surf_ncs', 'edge_ncs')."""
    B, S0, E = cfg.batch_size, cfg.num_surfaces, cfg.num_edges
    w = cfg.guidance_w
    label2 = None
    if cfg.use_cf:
        label2 = torch.tensor([cfg.class_label] * B + [0] * B).reshape(-1, 1)
    rep2 = (lambda t: torch.cat([t, t], 0)) if cfg.use_cf else (lambda t: t)
    pndm, ddpm = PNDMOracle(), DDPMOracle(clip_sample=True, clip_sample_range=3.0)

    def predict(fwd, x, t):
        tt = torch.tensor([int(t)])
        if cfg.use_cf:
            p = fwd(torch.cat([x, x], 0), tt)
            return p[:B] * (1 + w) - p[B:] * w
        return fwd(x, tt)

    def stage(name, x, fwd, hybrid_tail, late=None):
        k = 0
        if cfg.schedule == "ddpm":
            ddpm.set_timesteps(cfg.ddpm_steps)
            for t in ddpm.timesteps:
                if late is not None:
                    x = late(int(t), x)
                x = ddpm.step(predict(fwd, x, t), int(t), x, step_noise(name, k, x.shape) if int(t) > 0 else None)
                k += 1
            return x
        pndm.set_timesteps(200)
        ts = pndm.timesteps[:158] if hybrid_tail else pndm.timesteps
        for t in ts:
            x = pndm.step(predict(fwd, x, t), int(t), x)
        if hybrid_tail:
            if late is not None:
                x = late(-1, x)
            ddpm.set_timesteps(1000)
            for t in ddpm.timesteps[-250:]:
                x = ddpm.step(predict(fwd, x, t), int(t), x, step_noise(name, k, x.shape) if int(t) > 0 else None)
                k += 1
        return x

    state = {"late": cfg.use_cf}

    def late_increase(t, x):
        if not state["late"] and (t < 0 or t <= 249):
            state["late"] = True
            return x.repeat(1, 2, 1)
        return x

    if forwards is None:
        forwards = {"surfpos": lambda *a: O.surfpos_forward(sds["surfpos"], *a),
                    "surfz": lambda *a: O.surfz_forward(sds["surfz"], *a),
                    "edgepos": lambda *a: O.edgepos_forward(sds["edgepos"], *a),
                    "edgez": lambda *a: O.edgez_forward(sds["edgez"], *a)}
    F = forwards

    with torch.no_grad():
        surfPos = stage("surfPos", init_noise["surfPos"].clone(),
                        lambda x, t: F["surfpos"](x, t, label2), True, late_increase)
        if not state["late"]:
            surfPos = surfPos.repeat(1, 2, 1)
        S = surfPos.shape[1]
        if cfg.dense_masks:
            surfMask = torch.zeros(B, S, dtype=torch.bool)
        else:
            p, m = dedup_surfaces_np(surfPos.numpy(), np.float32(cfg.bbox_threshold))
            surfPos, surfMask = torch.from_numpy(p), torch.from_numpy(m)
        sP, sM = rep2(surfPos), rep2(surfMask)
        surfZ = stage("surfZ", init_noise["surfZ"].clone(),
                      lambda x, t: F["surfz"](x, t, sP, sM, label2), False)
        sZ = rep2(surfZ)
        edgePos = stage("edgePos", init_noise["edgePos"].clone(),
                        lambda x, t: F["edgepos"](x, t, sP, sZ, sM, label2), True)
        if cfg.dense_masks:
            edgeM = torch.zeros(B, S, E, dtype=torch.bool)
        else:
            edgeM = torch.from_numpy(dedup_edges_np(edgePos.numpy(), surfMask.numpy(), np.float32(cfg.bbox_threshold)))
        eP, eM = rep2(edgePos), rep2(edgeM)
        edgeZV = stage("edgeZV", init_noise["edgeZV"].clone(),
                       lambda x, t: F["edgez"](x, t, eP, sP, sZ, eM, label2), False)
        edgeZV = edgeZV.masked_fill(edgeM.unsqueeze(-1), 0.0)
        out = {"surfPos": surfPos / 3.0, "surfMask": surfMask, "surfZ": surfZ, "edgePos": edgePos / 3.0, "edgeM": edgeM,
               "edge_z": edgeZV[..., :12], "edgeV": edgeZV[..., 12:]}
        # decoder inputs (sample.py:289-293): 48 = 16 positions x 3 channels -> (N,3,4,4); 12 = 4 x 3 -> (N,3,4)
        if surf_vae is not None:
            z = surfZ.unflatten(-1, (16, 3)).flatten(0, 1).permute(0, 2, 1).unflatten(-1, (4, 4))
            out["surf_ncs"] = surf_vae(z).permute(0, 2, 3, 1).unflatten(0, (B, S))
        if edge_vae is not None:
            z = out["edge_z"].unflatten(-1, (4, 3)).reshape(-1, 4, 3).permute(0, 2, 1)
            out["edge_ncs"] = edge_vae(z).permute(0, 2, 1).reshape(B, S, E, 32, 3)
    return out
