"""Post-decode geometry glue with the reference's function surface (SURVEY.md 8(f) row 3).

Drop-in for the per-CAD post-processing of sample.py:303-355 up to (not including) `construct_brep`:

    edge_endpoints(edge_pos_cad, edge_ncs_cad, edge_mask_cad)                    sample.py:316-329
    detect_shared_vertex(edgeV_cad, edge_mask_cad, edgeV_bbox)                   utils.py:463-586
    detect_shared_edge(unique_vertices, new_vertex_dict, edge_z_cad, surf_z_cad, z_threshold, edge_mask_cad)
                                                                                  utils.py:588-646
    joint_optimize(surf_ncs, edge_ncs, surfPos, unique_vertices, EdgeVertexAdj, FaceEdgeAdj, num_edge, num_surf)
                                                                                  utils.py:672-776

Same arguments (numpy arrays as the reference passes them), same return values and the same vertex / edge numbering.  The
numeric cores run on the GPU through the C ABI (csrc/geom.cu): nearest-other-end-point searches, the close-centre and
same-end-points / latent-distance matrices, the closed-form edge fit, the surface initialisation and -- the expensive part --
the 200-step AdamW fit of one translation per face against the one-directional Chamfer distance, which the reference runs as
one chamferdist call per face and iteration and which here is ONE kernel launch for all faces and iterations.  What stays on
the host is the bookkeeping over python lists and sets (loop closing, T-junction merging), a few dozen items per CAD.
No CPU fallback: the library must be present and the device an sm_90 (H100) GPU.
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from . import _ffi


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _f32(a) -> torch.Tensor:
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(_dev())


def _i32(a) -> torch.Tensor:
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32)).to(_dev())


def _valid_counts(edge_mask_cad) -> np.ndarray:
    return (np.asarray(edge_mask_cad) == False).sum(1)


# ------------------------------------------------------------------------------------------------ sample.py:316-329
def edge_endpoints(edge_pos_cad, edge_ncs_cad, edge_mask_cad) -> List[np.ndarray]:
    """per face the (n_valid, 2, 3) start / end points of its valid edges: decoded curve end points mapped from the edge's
    normalised frame into its bounding box (centre, largest extent)"""
    mask = np.asarray(edge_mask_cad, dtype=bool)
    pos = _f32(np.asarray(edge_pos_cad)[~mask])
    ncs = _f32(np.asarray(edge_ncs_cad)[~mask])
    n = pos.shape[0]
    out = torch.empty(n, 2, 3, device=pos.device)
    _ffi.check(_ffi.lib().bg_edge_endpoints(ncs.data_ptr(), pos.data_ptr(), 1.0, n, out.data_ptr(), _ffi.current_stream()),
               "bg_edge_endpoints")
    flat = out.cpu().numpy()
    cuts = np.cumsum(_valid_counts(mask))[:-1]
    return np.split(flat, cuts)


# ------------------------------------------------------------------------------------------------ utils.py:403-421
def _nearest_other(points: np.ndarray, group: np.ndarray, seg_off: np.ndarray) -> np.ndarray:
    """nn[i] = nearest point of another group within i's segment (device kernel bg_nn_exclude)"""
    p, g, s = _f32(points), _i32(group), _i32(seg_off)
    nn = torch.empty(len(points), dtype=torch.int32, device=p.device)
    _ffi.check(_ffi.lib().bg_nn_exclude(p.data_ptr(), g.data_ptr(), s.data_ptr(), len(seg_off) - 1, nn.data_ptr(),
                                       _ffi.current_stream()), "bg_nn_exclude")
    return nn.cpu().numpy().astype(np.int64)


def _loops(ends_per_face: List[np.ndarray]) -> List[np.ndarray]:
    """edge2loop for every face at once: each end point is paired with the nearest end point of ANOTHER edge of its face;
    the distinct (sorted) pairs of a face, as local ids 2 * edge + {0, 1}"""
    counts = [len(e) for e in ends_per_face]
    seg = np.concatenate([[0], np.cumsum([2 * c for c in counts])])
    pts = np.concatenate([e.reshape(-1, 3) for e in ends_per_face])
    grp = np.concatenate([np.repeat(np.arange(c), 2) for c in counts])
    nn = _nearest_other(pts, grp, seg)
    out = []
    for f, c in enumerate(counts):
        lo = seg[f]
        own = np.arange(2 * c)
        pairs = np.sort(np.stack([own, nn[lo:lo + 2 * c] - lo], 1), axis=1)
        out.append(np.unique(pairs, axis=0))
    return out


def edge2loop(face_edges) -> np.ndarray:
    return _loops([np.asarray(face_edges, dtype=np.float32)])[0]


# ------------------------------------------------------------------------------------------------ utils.py:463-586
def _absorb_overlaps(groups: List[List[int]]) -> List[List[int]]:
    """repeat until stable: a group is replaced by its union with the first LATER group it overlaps without containing or
    being contained in it (the union is strictly larger than both); untouched groups are carried over.  Order matters for
    the final numbering, so this follows the reference's sweep exactly."""
    while True:
        nxt, grew = [], False
        for i, gi in enumerate(groups):
            si = set(gi)
            repl = None
            for gj in groups[i + 1:]:
                sj = set(gj)
                if si & sj and len(si | sj) > max(len(gi), len(gj)):
                    repl = list(si | sj)
                    break
            grew |= repl is not None
            nxt.append(repl if repl is not None else gi)
        groups = nxt
        if not grew:
            return groups


def _maximal_distinct(groups: List[List[int]]) -> List[List[int]]:
    """drop groups that are proper subsets of another one, then duplicates (first occurrence wins)"""
    sets = [set(g) for g in groups]
    out, seen = [], set()
    for i, s in enumerate(sets):
        if any(i != j and s < t for j, t in enumerate(sets)):
            continue
        key = tuple(sorted(s))
        if key not in seen:
            seen.add(key)
            out.append(list(s))
    return out


def detect_shared_vertex(edgeV_cad, edge_mask_cad, edgeV_bbox):
    """Find the shared vertices: returns [unique_vertices (V, 3), {new vertex id: [old end-point ids]}]"""
    mask = np.asarray(edge_mask_cad, dtype=bool)
    counts = _valid_counts(mask)
    base = 2 * np.concatenate([[0], np.cumsum(counts)])[:-1]
    pred = [np.asarray(fe)[~fm].reshape(-1, 2, 3).astype(np.float32) for fe, fm in zip(edgeV_cad, mask)]
    bbox = [np.asarray(b, dtype=np.float32) for b in edgeV_bbox]
    loops_bbox = _loops(bbox)
    loops_pred = None
    merges, used = [], []
    for f in range(len(pred)):
        # a face wire is closed when pairing the end points gives exactly one pair per edge: first try the decoded curve end
        # points (scaled to the x3 frame of the predicted vertices), then the predicted vertex positions themselves
        if len(loops_bbox[f]) == counts[f]:
            merges.append(base[f] + loops_bbox[f])
            used.append(bbox[f] * 3)
            continue
        if loops_pred is None:
            loops_pred = _loops(pred)
        if len(loops_pred[f]) == counts[f]:
            merges.append(base[f] + loops_pred[f])
            used.append(pred[f])
            continue
        raise AssertionError("face loop could not be closed")
    flat = np.vstack(used).reshape(-1, 3)

    # across faces: every merged pair of a face joins the nearest merged pair of any OTHER face
    pairs = np.vstack(merges)
    centres = flat[pairs].mean(1)
    face_of = np.concatenate([np.full(len(m), f) for f, m in enumerate(merges)])
    hit = _nearest_other(centres, face_of, np.array([0, len(pairs)]))
    groups = [list(pairs[hit[k]]) + list(pairs[k]) for k in range(len(pairs))]

    groups = _maximal_distinct(_absorb_overlaps(groups))

    # groups whose centres are closer than 0.1 are concatenated (T-junctions of more than three edges)
    c = np.array([flat[g].mean(0) for g in groups], dtype=np.float32)
    cd = _f32(c)
    close = torch.empty(len(c), len(c), dtype=torch.uint8, device=cd.device)
    _ffi.check(_ffi.lib().bg_pairs_within(cd.data_ptr(), len(c), 0.1, close.data_ptr(), _ffi.current_stream()), "bg_pairs_within")
    rows, cols = np.where(np.tril(close.cpu().numpy().astype(bool), k=-1))
    touched = set(rows.tolist()) | set(cols.tolist())
    groups = [groups[r] + groups[q] for r, q in zip(rows, cols)] + [g for k, g in enumerate(groups) if k not in touched]

    verts = np.vstack([flat[g].mean(0) / 3.0 for g in groups])
    return [verts, {k: g for k, g in enumerate(groups)}]


# ------------------------------------------------------------------------------------------------ utils.py:588-646
def detect_shared_edge(unique_vertices, new_vertex_dict: Dict[int, List[int]], edge_z_cad, surf_z_cad, z_threshold, edge_mask_cad):
    """Find the shared edges: returns [unique_faces, unique_edges, FaceEdgeAdj, EdgeVertexAdj]"""
    z = np.asarray(edge_z_cad, dtype=np.float32)
    n = len(z)
    owner = {}
    for new_id, old_ids in new_vertex_dict.items():
        for o in old_ids:
            owner.setdefault(int(o), []).append(new_id)
    assert all(len(owner.get(o, [])) == 1 for o in range(2 * n))          # every end point belongs to exactly one vertex
    eva = np.array([owner[o][0] for o in range(2 * n)]).reshape(-1, 2)

    adj, zd = _i32(eva), _f32(z)
    match = torch.empty(n, n, dtype=torch.uint8, device=zd.device)
    _ffi.check(_ffi.lib().bg_edge_pair_match(adj.data_ptr(), zd.data_ptr(), z.shape[1], n, float(z_threshold), match.data_ptr(),
                                            _ffi.current_stream()), "bg_edge_pair_match")
    similar = np.argwhere(np.triu(match.cpu().numpy().astype(bool), k=1))     # sorted, distinct (i < j) pairs
    if not 2 * len(similar) == n:
        assert False, 'edge not reduced by 2'
    keep = similar[:, 0]
    ranges = np.concatenate([[0], np.cumsum(_valid_counts(edge_mask_cad))])
    fea = []
    for k in range(len(ranges) - 1):
        row = []
        for e in range(ranges[k], ranges[k + 1]):
            where = np.where(similar == e)[0]
            assert len(where) == 1
            row.append(where[0])
        fea.append(row)
    return [surf_z_cad, z[keep], fea, eva[keep]]


# ------------------------------------------------------------------------------------------------ utils.py:672-776
def joint_optimize(surf_ncs, edge_ncs, surfPos, unique_vertices, EdgeVertexAdj, FaceEdgeAdj, num_edge, num_surf, iters: int = 200):
    """Jointly fit faces / edges / vertices: returns (surf_wcs (F, 32, 32, 3), edge_wcs (E, 32, 3)) as numpy arrays"""
    lib, st = _ffi.lib(), _ffi.current_stream()
    e_ncs = _f32(edge_ncs)
    vse = _f32(np.asarray(unique_vertices, dtype=np.float32)[np.asarray(EdgeVertexAdj)])
    ne, nf = e_ncs.shape[0], len(FaceEdgeAdj)
    edge_wcs = torch.empty(ne, 32, 3, device=e_ncs.device)
    _ffi.check(lib.bg_edge_fit(e_ncs.data_ptr(), vse.data_ptr(), ne, edge_wcs.data_ptr(), st), "bg_edge_fit")

    off = _i32(np.concatenate([[0], np.cumsum([len(a) for a in FaceEdgeAdj])]))
    adj = _i32(np.concatenate([np.asarray(a, dtype=np.int64) for a in FaceEdgeAdj]))
    s_ncs, s_pos = _f32(np.asarray(surf_ncs).reshape(nf, -1, 3)), _f32(surfPos)
    init = torch.empty(nf, 1024, 3, device=e_ncs.device)
    _ffi.check(lib.bg_surf_init(s_ncs.data_ptr(), s_pos.data_ptr(), edge_wcs.data_ptr(), off.data_ptr(), adj.data_ptr(), nf,
                                init.data_ptr(), st), "bg_surf_init")
    inv = torch.full((nf,), 1.0 / nf, device=e_ncs.device)
    out = torch.empty_like(init)
    _ffi.check(lib.bg_surf_offset_opt(init.data_ptr(), edge_wcs.data_ptr(), off.data_ptr(), adj.data_ptr(), inv.data_ptr(), nf,
                                      max(len(a) for a in FaceEdgeAdj), int(iters), 1e-3, 0.95, 0.999, 1e-8, 1e-6, out.data_ptr(),
                                      None, st), "bg_surf_offset_opt")
    return out.reshape(nf, 32, 32, 3).cpu().numpy(), edge_wcs.cpu().numpy()


# ------------------------------------------------------------------------------------------------ sample.py:303-355
def postprocess_cad(surf_vae, edge_vae, surfPos_cad, surfZ_cad, surfMask_cad, edge_pos_cad, edge_ncs_cad, edgeV_cad, edge_z_cad,
                    edge_mask_cad, z_threshold: float = 0.2, iters: int = 200):
    """One CAD through the reference's post-processing loop body (sample.py:303-355) up to, not including, construct_brep.

    Inputs are the per-CAD slices of the cascade outputs exactly as sample.py:305-312 forms them from the batch arrays
    (numpy; S face slots, E edge slots per face): surfPos (S,6) in model units, surfZ (S,48), surfMask (S,) True = padded,
    edge_pos (S,E,6) in model units, edge_ncs (S,E,32,3) decoded edge curves, edgeV (S,E,6) predicted vertices (x3 frame),
    edge_z (S,E,12), edge_mask (S,E) True = padded / duplicate.  surf_vae / edge_vae: the drop-in decoders (brepgen_b200.vae).
    Returns (surf_wcs (F,32,32,3), edge_wcs (Eu,32,3), FaceEdgeAdj, EdgeVertexAdj, unique_vertices): the arguments of
    construct_brep(surf_wcs, edge_wcs, FaceEdgeAdj, EdgeVertexAdj) (utils.py:819).  Raises AssertionError where the reference
    prints '... failed' and skips the CAD."""
    keep = ~np.asarray(surfMask_cad, dtype=bool)
    emask = np.asarray(edge_mask_cad, dtype=bool)[keep]
    epos, encs, ev = np.asarray(edge_pos_cad)[keep], np.asarray(edge_ncs_cad)[keep], np.asarray(edgeV_cad)[keep]
    ez = np.asarray(edge_z_cad)[keep][~emask]
    sz, spos = np.asarray(surfZ_cad)[keep], np.asarray(surfPos_cad)[keep]

    ends = edge_endpoints(epos, encs, emask)                                           # sample.py:316-329
    unique_vertices, vertex_dict = detect_shared_vertex(ev, emask, ends)               # 3-1
    unique_faces, unique_edges, fea, eva = detect_shared_edge(unique_vertices, vertex_dict, ez, sz, z_threshold, emask)   # 3-2
    with torch.no_grad():                                                              # sample.py:346-351
        zf = torch.as_tensor(np.asarray(unique_faces, dtype=np.float32)).to(_dev())
        surf_ncs = surf_vae(zf.unflatten(-1, (16, 3)).permute(0, 2, 1).unflatten(-1, (4, 4)).contiguous())
        surf_ncs = surf_ncs.permute(0, 2, 3, 1).cpu().numpy()
        ze = torch.as_tensor(np.asarray(unique_edges, dtype=np.float32)).to(_dev())
        edge_ncs = edge_vae(ze.unflatten(-1, (4, 3)).permute(0, 2, 1).contiguous()).permute(0, 2, 1).cpu().numpy()
    surf_wcs, edge_wcs = joint_optimize(surf_ncs, edge_ncs, spos, unique_vertices, eva, fea, len(edge_ncs), len(surf_ncs),
                                        iters=iters)                                    # 3-3
    return surf_wcs, edge_wcs, fea, eva, unique_vertices
