"""Golden vectors for the post-decode geometry glue from the reference's OWN function texts (build container only).

    python tests/golden/make_golden_post.py          # writes tests/golden/post_golden.npz

utils.py cannot be imported (OpenCASCADE / chamferdist at module import).  The functions of this path are
plain numpy / torch, so their source text is cut out of the file with `ast` and exec()'d VERBATIM:
    compute_bbox_center_and_size  utils.py:48-59      edge2loop             utils.py:403-421
    keep_largelist                utils.py:424-460    detect_shared_vertex  utils.py:463-586
    detect_shared_edge            utils.py:588-646    STModel / get_bbox_minmax / joint_optimize  utils.py:648-776
and the end-point block of sample.py:316-329 is exec()'d as statements.  Stand-ins needed to run them here:
`ChamferDistance` (chamferdist is absent: oracle.postprocess.chamfer_reverse_sum restates its published semantics --
that part stays "parity unpinned") and `.cuda()` as the identity (no GPU in the build container).
Inputs are synthetic closed B-reps (`synth_cad`: boxes with jittered decoded end points, padded face / edge slots);
they are regenerated from seeds by the tests, only outputs are stored.  Nothing from the reference is copied into the repo.
"""
from __future__ import annotations

import ast
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = os.environ.get("BREPGEN_REFERENCE", "/root/reference")
CASES = {"box_a": (1, 8, 6), "box_b": (2, 7, 5), "box_c": (3, 10, 8)}       # seed, padded face slots, padded edge slots
Z_THRESHOLD = 0.2                                                          # eval_config.yaml:10


def synth_cad(seed: int, S: int, E: int):
    """one CAD at the interface of sample.py:303-312: a box (6 quad faces x 4 half-edges, 12 unique edges, 8 vertices) in
    padded (S, E) slot arrays; decoded edge curves and predicted vertices carry small jitter so the merges are not trivial"""
    rng = np.random.default_rng(seed)
    lo, hi = rng.uniform(-0.8, -0.3, 3), rng.uniform(0.3, 0.8, 3)
    corner = lambda i, j, k: np.array([[lo, hi][i][0], [lo, hi][j][1], [lo, hi][k][2]])
    V = {(i, j, k): corner(i, j, k) for i in (0, 1) for j in (0, 1) for k in (0, 1)}
    quads = [[(0, 0, 0), (0, 1, 0), (0, 1, 1), (0, 0, 1)], [(1, 0, 0), (1, 1, 0), (1, 1, 1), (1, 0, 1)],
             [(0, 0, 0), (1, 0, 0), (1, 0, 1), (0, 0, 1)], [(0, 1, 0), (1, 1, 0), (1, 1, 1), (0, 1, 1)],
             [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0)], [(0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]]
    ez_base = {}
    f32 = np.float32
    surfPos = np.zeros((S, 6), f32)
    surfZ = rng.normal(size=(S, 48)).astype(f32)
    surf_ncs = np.zeros((S, 32, 32, 3), f32)
    surfMask = np.ones(S, bool)
    edge_pos = np.zeros((S, E, 6), f32)
    edge_ncs = np.zeros((S, E, 32, 3), f32)
    edgeV = np.zeros((S, E, 6), f32)
    edge_z = np.zeros((S, E, 12), f32)
    edge_mask = np.ones((S, E), bool)
    t = np.linspace(0, 1, 32)[:, None]
    for f, q in enumerate(quads):
        surfMask[f] = False
        P = np.array([V[c] for c in q])
        u, v = np.meshgrid(np.linspace(0, 1, 32), np.linspace(0, 1, 32), indexing="ij")
        grid = ((1 - u) * (1 - v))[..., None] * P[0] + (u * (1 - v))[..., None] * P[1] + (u * v)[..., None] * P[2] \
            + ((1 - u) * v)[..., None] * P[3]
        mn, mx = P.min(0), P.max(0)
        shrink = rng.uniform(0.9, 1.02)                 # some face boxes are smaller than their wire (the 1.05 rule)
        c, size = (mn + mx) / 2, (mx - mn).max() * shrink
        surfPos[f] = np.concatenate([c - (mx - mn) / 2 * shrink, c + (mx - mn) / 2 * shrink])
        surf_ncs[f] = (grid - c) / (size / 2) + rng.normal(scale=2e-3, size=grid.shape)
        for e in range(4):
            a, b = q[e], q[(e + 1) % 4]
            if rng.random() < 0.5:
                a, b = b, a
            pa, pb = V[a], V[b]
            curve = pa * (1 - t) + pb * t + rng.normal(scale=1.5e-3, size=(32, 3))
            bmn, bmx = curve.min(0), curve.max(0)
            bc, bs = (bmn + bmx) / 2, (bmx - bmn).max()
            edge_pos[f, e] = np.concatenate([bmn, bmx])
            edge_ncs[f, e] = (curve - bc) / (bs / 2)
            edgeV[f, e] = np.concatenate([pa, pb]) * 3 + rng.normal(scale=6e-3, size=6)
            key = tuple(sorted([a, b]))
            if key not in ez_base:
                ez_base[key] = rng.normal(size=12)
            edge_z[f, e] = ez_base[key] + rng.normal(scale=0.02, size=12)
            edge_mask[f, e] = False
    return dict(surfPos=surfPos, surfZ=surfZ, surf_ncs=surf_ncs, surfMask=surfMask, edge_pos=edge_pos, edge_ncs=edge_ncs,
                edgeV=edgeV, edge_z=edge_z, edge_mask=edge_mask)


def select_cad(d):
    """the per-CAD selections of sample.py:305-312"""
    keep = ~d["surfMask"]
    edge_mask_cad = d["edge_mask"][keep]
    return dict(edge_mask_cad=edge_mask_cad, edge_pos_cad=d["edge_pos"][keep], edge_ncs_cad=d["edge_ncs"][keep],
                edgeV_cad=d["edgeV"][keep], edge_z_cad=d["edge_z"][keep][~edge_mask_cad], surf_z_cad=d["surfZ"][keep],
                surf_pos_cad=d["surfPos"][keep], surf_ncs_cad=d["surf_ncs"][keep])


def reference_namespace():
    """functions of the path, exec()'d verbatim from the reference's files"""
    from oracle.postprocess import chamfer_reverse_sum

    class ChamferDistance:                      # stand-in for chamferdist (absent offline)
        def __call__(self, source, target, bidirectional=False, reverse=False):
            assert reverse and not bidirectional
            return chamfer_reverse_sum(source, target)

    src = open(os.path.join(REF, "utils.py")).read()
    tree = ast.parse(src)
    ns = {"np": np, "torch": torch, "nn": torch.nn, "ChamferDistance": ChamferDistance, "print": lambda *a, **k: None}
    want = {"compute_bbox_center_and_size", "edge2loop", "keep_largelist", "detect_shared_vertex", "detect_shared_edge",
            "STModel", "get_bbox_minmax", "joint_optimize"}
    for node in tree.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in want:
            exec(compile(ast.get_source_segment(src, node), f"utils.py:{node.name}", "exec"), ns)
    lines = open(os.path.join(REF, "sample.py")).read().split("\n")
    block = "\n".join(l[8:] for l in lines[315:329])                # sample.py:316-329, de-indented
    assert block.lstrip().startswith("# Retrieve vertices") and "edgeV_bbox.append(bbox_startends)" in block
    ns["_endpoint_block"] = compile(block, "sample.py:316-329", "exec")
    return ns


def run_reference(ns, d, decode_identity=True):
    c = select_cad(d)
    loc = dict(ns, edge_pos_cad=c["edge_pos_cad"], edge_ncs_cad=c["edge_ncs_cad"], edge_mask_cad=c["edge_mask_cad"])
    exec(ns["_endpoint_block"], loc)
    edgeV_bbox = loc["edgeV_bbox"]
    uv, vd = ns["detect_shared_vertex"](c["edgeV_cad"], c["edge_mask_cad"], edgeV_bbox)
    uf, ue, fea, eva = ns["detect_shared_edge"](uv, vd, c["edge_z_cad"], c["surf_z_cad"], Z_THRESHOLD, c["edge_mask_cad"])
    # the reference decodes unique faces / edges with the VAEs here (sample.py:346-351); the geometry test takes the decoded
    # grids of the corresponding slots instead (unique edge k = first half-edge of its pair)
    flat_ncs = c["edge_ncs_cad"][~c["edge_mask_cad"]]
    similar_first = unique_edge_ids(eva, vd, c)
    edge_ncs_u = flat_ncs[similar_first]
    cuda_t, cuda_m = torch.Tensor.cuda, torch.nn.Module.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    try:
        torch.manual_seed(0)
        surf_wcs, edge_wcs = ns["joint_optimize"](c["surf_ncs_cad"], edge_ncs_u, c["surf_pos_cad"], uv, eva, fea, len(edge_ncs_u),
                                                  len(c["surf_ncs_cad"]))
    finally:
        torch.Tensor.cuda, torch.nn.Module.cuda = cuda_t, cuda_m
    return dict(edgeV_bbox=edgeV_bbox, unique_vertices=uv, vertex_dict=vd, unique_edges=ue, FaceEdgeAdj=fea, EdgeVertexAdj=eva,
                unique_edge_ids=similar_first, surf_wcs=surf_wcs, edge_wcs=edge_wcs)


def unique_edge_ids(eva_unique, vertex_dict, c):
    """ids (into the flattened valid half-edges) of the half-edges the reference keeps as unique edges: recomputed from the
    full EdgeVertexAdj the way utils.py:592-624 does, because detect_shared_edge does not return them"""
    n = len(c["edge_z_cad"])
    old2new = {}
    for k, ids in vertex_dict.items():
        for i in ids:
            old2new[i] = k
    full = np.array([old2new[i] for i in range(2 * n)]).reshape(-1, 2)
    pairs = set()
    for i in range(n):
        for j in range(n):
            if i != j and set(full[i]) == set(full[j]) and np.abs(c["edge_z_cad"][i] - c["edge_z_cad"][j]).mean() < Z_THRESHOLD:
                pairs.add(tuple(sorted([i, j])))
    first = np.array(sorted(pairs))[:, 0]
    assert np.array_equal(full[first], eva_unique)
    return first


def pack_ragged(lists):
    off = np.cumsum([0] + [len(l) for l in lists]).astype(np.int64)
    return off, np.concatenate([np.asarray(l, dtype=np.int64) for l in lists]) if lists else np.zeros(0, np.int64)


def main():
    ns = reference_namespace()
    out = {}
    for name, (seed, S, E) in CASES.items():
        r = run_reference(ns, synth_cad(seed, S, E))
        out[f"{name}|edgeV_bbox"] = np.concatenate(r["edgeV_bbox"]).astype(np.float32)
        out[f"{name}|unique_vertices"] = np.asarray(r["unique_vertices"], np.float32)
        off, flat = pack_ragged([r["vertex_dict"][k] for k in range(len(r["vertex_dict"]))])
        out[f"{name}|vertex_dict_off"], out[f"{name}|vertex_dict"] = off, flat
        out[f"{name}|unique_edges"] = np.asarray(r["unique_edges"], np.float32)
        off, flat = pack_ragged(r["FaceEdgeAdj"])
        out[f"{name}|FaceEdgeAdj_off"], out[f"{name}|FaceEdgeAdj"] = off, flat
        out[f"{name}|EdgeVertexAdj"] = np.asarray(r["EdgeVertexAdj"], np.int64)
        out[f"{name}|unique_edge_ids"] = np.asarray(r["unique_edge_ids"], np.int64)
        out[f"{name}|surf_wcs"] = np.asarray(r["surf_wcs"], np.float32)
        out[f"{name}|edge_wcs"] = np.asarray(r["edge_wcs"], np.float32)
        print(name, "V", len(r["unique_vertices"]), "E", len(r["unique_edges"]), "F", len(r["FaceEdgeAdj"]))
    path = os.path.join(ROOT, "tests", "golden", "post_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
