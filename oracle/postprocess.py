"""ORACLE (test infrastructure, not product code): CPU restatement of the reference's per-CAD post-processing between the
VAE decoders and OpenCASCADE -- SURVEY.md 8(f) row 3.

Only tests/ and tests/golden/make_golden_post.py import this module; brepgen_b200/ never does.

Restated (numpy, statement order of the reference so that vertex / edge numbering comes out identical):
  edge_endpoints          sample.py:316-329  (+ utils.py:48-59 compute_bbox_center_and_size)
  edge2loop               utils.py:403-421
  keep_largelist          utils.py:424-460
  detect_shared_vertex    utils.py:463-586
  detect_shared_edge      utils.py:588-646
  joint_optimize          utils.py:672-776 (torch CPU; `chamfer_reverse_sum` stands in for chamferdist.ChamferDistance)

Pinned: tests/golden/post_golden.npz holds the outputs of the reference's OWN function texts, exec()'d from
utils.py and sample.py by tests/golden/make_golden_post.py on synthetic closed B-reps;
tests/test_oracle_post.py checks this restatement against them (ids exact, coordinates to fp32 round-off).
PARITY UNPINNED for one dependency: `chamferdist` (requirements.txt, absent offline).  Its published semantics are
restated here -- ChamferDistance()(source, target, bidirectional=False, reverse=True) = sum over TARGET points of the
squared distance to the nearest SOURCE point, batch mean -- and the golden run of joint_optimize uses this stand-in.
"""
from __future__ import annotations

import numpy as np
import torch


def bbox_center_and_size(lo, hi):
    c = np.array([(lo[0] + hi[0]) / 2, (lo[1] + hi[1]) / 2, (lo[2] + hi[2]) / 2])
    return c, max(hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2])


def edge_endpoints(edge_pos_cad, edge_ncs_cad, edge_mask_cad):
    """sample.py:316-329: per face, the (n_valid, 2, 3) start / end points of its valid edges in model coordinates"""
    out = []
    for bbox, ncs, mask in zip(edge_pos_cad, edge_ncs_cad, edge_mask_cad):
        rows = []
        for bb, ee in zip(bbox[~mask], ncs[~mask]):
            c, size = bbox_center_and_size(bb[0:3], bb[3:])
            wcs = ee * (size / 2) + c
            rows.append(wcs[[0, -1]].reshape(1, 2, 3))
        out.append(np.vstack(rows))
    return out


def edge2loop(face_edges):
    flat = face_edges.reshape(-1, 3)
    pairs = []
    for e, se in enumerate(face_edges):
        own = [2 * e, 2 * e + 1]
        for k in (0, 1):
            order = list(np.argsort(np.linalg.norm(flat - se[k], axis=1)))
            other = [x for x in order if x not in own]
            pairs.append(sorted([2 * e + k, other[0]]))
    return np.unique(np.array(pairs), axis=0)


def keep_largelist(int_lists):
    sets = [set(l) for l in int_lists]
    largest = []
    for i, s1 in enumerate(sets):
        if not any(i != j and s1.issubset(s2) and s1 != s2 for j, s2 in enumerate(sets)):
            largest.append(list(s1))
    seen, uniq = set(), []
    for l in largest:
        t = tuple(sorted(l))
        if t not in seen:
            seen.add(t)
            uniq.append(l)
    return uniq


def detect_shared_vertex(edgeV_cad, edge_mask_cad, edgeV_bbox):
    offs = 2 * np.concatenate([np.array([0]), np.cumsum((edge_mask_cad == False).sum(1))])[:-1]
    used, merges = [], []
    for f, (fe, fm, be) in enumerate(zip(edgeV_cad, edge_mask_cad, edgeV_bbox)):
        fe = fe[~fm]
        fe = fe.reshape(len(fe), 2, 3)
        ids = edge2loop(be)
        if len(ids) == len(fe):
            merges.append(offs[f] + ids)
            used.append(be * 3)
            continue
        ids = edge2loop(fe)
        if len(ids) == len(fe):
            merges.append(offs[f] + ids)
            used.append(fe)
            continue
        raise AssertionError("face loop could not be closed")
    pts = np.vstack(used)
    flat = pts.reshape(len(pts), 2, 3).reshape(-1, 3)

    total = []
    for f, fm in enumerate(merges):
        others = np.vstack([merges[x] for x in sorted(set(range(len(merges))) - {f})])
        centers = flat[others].mean(1)
        for mid in fm:
            c = flat[mid].mean(0)
            hit = others[np.argsort(np.linalg.norm(centers - c, axis=1))[0]]
            total.append(list(hit) + list(mid))

    while True:
        changed, nxt = False, []
        for i in range(len(total)):
            merged = False
            for j in range(i + 1, len(total)):
                a, b = set(total[i]), set(total[j])
                if len(a | b) > max(len(total[i]), len(total[j])) and len(a & b) > 0:
                    nxt.append(list(a | b))
                    merged = changed = True
                    break
            if not merged:
                nxt.append(total[i])
        total = nxt
        if not changed:
            break
    total = keep_largelist(total)

    centers = np.array([flat[x].mean(0) for x in total])
    close = np.linalg.norm(centers[:, np.newaxis, :] - centers, axis=2) < 0.1
    rows, cols = np.where(close & np.tril(np.ones_like(close, dtype=bool), k=-1))
    upd = [total[r] + total[c] for r, c in zip(rows, cols)]
    upd += [ids for k, ids in enumerate(total) if k not in list(rows) and k not in list(cols)]
    total = upd

    verts = np.vstack([flat[ids].mean(0) / 3.0 for ids in total])
    return [verts, {k: ids for k, ids in enumerate(total)}]


def detect_shared_edge(unique_vertices, new_vertex_dict, edge_z_cad, surf_z_cad, z_threshold, edge_mask_cad):
    new_ids = []
    for old in np.arange(2 * len(edge_z_cad)):
        hit = [k for k, v in new_vertex_dict.items() if old in v]
        assert len(hit) == 1
        new_ids.append(hit[0])
    eva = np.array(new_ids).reshape(-1, 2)
    similar = []
    for i, s1 in enumerate(eva):
        for j, s2 in enumerate(eva):
            if i != j and set(s1) == set(s2) and np.abs(edge_z_cad[i] - edge_z_cad[j]).mean() < z_threshold:
                similar.append(sorted([i, j]))
    similar = np.unique(np.array(similar), axis=0)
    assert 2 * len(similar) == len(eva), "edge not reduced by 2"
    keep = similar[:, 0]
    ranges = np.concatenate([np.array([0]), np.cumsum((edge_mask_cad == False).sum(1))])
    fea = []
    for k in range(len(ranges) - 1):
        row = []
        for e in np.arange(ranges[k], ranges[k + 1]):
            w = np.where(similar == e)[0]
            assert len(w) == 1
            row.append(w[0])
        fea.append(row)
    return [surf_z_cad, edge_z_cad[keep], fea, eva[keep]]


def chamfer_reverse_sum(source: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """chamferdist.ChamferDistance()(source, target, bidirectional=False, reverse=True) for batch size 1: for every TARGET
    point the squared distance to its nearest SOURCE point, summed (point_reduction='sum', batch_reduction='mean')."""
    d = ((target[0][:, None, :] - source[0][None, :, :]) ** 2).sum(-1)       # (n_target, n_source)
    return d.min(dim=1).values.sum()


def fit_edges(edge_ncs, unique_vertices, EdgeVertexAdj):
    """utils.py:688-728"""
    ncs_se = edge_ncs[:, [0, -1]]
    vse = unique_vertices[EdgeVertexAdj]
    out = []
    for wcs, se, v in zip(edge_ncs, ncs_se, vse):
        sc = np.linalg.norm(v[0] - v[1]) / np.linalg.norm(se[0] - se[1])
        upd, e2 = wcs * sc, se * sc
        off, off_r = v - e2, v - e2[::-1]
        if np.abs(off_r[0] - off_r[1]).mean() < np.abs(off[0] - off[1]).mean():
            upd, off = upd[::-1], off_r
        out.append(upd + off.mean(0)[np.newaxis, np.newaxis, :])
    edge_wcs = np.vstack(out)
    for k in range(len(edge_wcs)):
        sv, ev = vse[k, 0] - edge_wcs[k, 0], vse[k, 1] - edge_wcs[k, -1]
        w = np.tile((np.arange(32) / 31)[:, np.newaxis], (1, 3))
        edge_wcs[k] += np.tile(sv[np.newaxis, :], (32, 1)) * (1 - w) + np.tile(ev, (32, 1)) * w
    return edge_wcs, vse


def init_surfaces(surf_ncs, surfPos, edge_wcs, FaceEdgeAdj):
    """utils.py:730-752"""
    out = []
    for adj, ncs, bbox in zip(FaceEdgeAdj, surf_ncs, surfPos):
        c, sscale = bbox_center_and_size(bbox[0:3], bbox[3:])
        flat = edge_wcs[adj].reshape(-1, 3)
        _, escale = bbox_center_and_size(flat.min(0), flat.max(0))
        if sscale < escale:
            sscale = 1.05 * escale
        out.append(ncs * (sscale / 2) + c)
    return np.stack(out)


def joint_optimize(surf_ncs, edge_ncs, surfPos, unique_vertices, EdgeVertexAdj, FaceEdgeAdj, num_edge, num_surf, iters=200):
    edge_wcs, _ = fit_edges(edge_ncs, unique_vertices, EdgeVertexAdj)
    face_edges = [torch.FloatTensor(edge_wcs[adj]) for adj in FaceEdgeAdj]
    surf = torch.FloatTensor(init_surfaces(surf_ncs, surfPos, edge_wcs, FaceEdgeAdj))
    edge_t = torch.nn.Parameter(torch.zeros((num_edge, 3)))
    surf_st = torch.nn.Parameter(torch.FloatTensor([1, 0, 0, 0]).unsqueeze(0).repeat(num_surf, 1))
    opt = torch.optim.AdamW([edge_t, surf_st], lr=1e-3, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-08)
    for _ in range(iters):
        upd = surf + surf_st[:, 1:].reshape(-1, 1, 1, 3)
        loss = 0
        for sp, ep in zip(upd, face_edges):
            loss = loss + chamfer_reverse_sum(sp.reshape(-1, 3).unsqueeze(0), ep.reshape(-1, 3).detach().unsqueeze(0))
        loss = loss / len(upd)
        opt.zero_grad()
        loss.backward()
        opt.step()
    return upd.detach().numpy(), edge_wcs
