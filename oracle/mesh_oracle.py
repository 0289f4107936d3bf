"""CPU oracle (TEST INFRASTRUCTURE -- never imported by the product path) for mesh extraction:
InstantNeuS.extract_fields / extract_geometry / extract_color (src/InstantNeuS.py:402-492).

* field(...)            extract_fields: u = -sdf on the linspace lattice, -100 outside the strict
                        realtime_bound test; the sdf is neus_oracle's restatement (normalised by `bound`).
* marching_cubes(...)   vectorised marching cubes on the tables in go-slam_b200/csrc/mc_tables.cuh
                        (built by tools/gen_mc_tables.py), with the device's orders and fp64 formulas:
                        one vertex per crossing lattice edge in ascending edge id (3 * linear(a) + axis,
                        x-major), t = (iso - ua) / (ub - ua); faces by cell (x-major, z fastest), then
                        table order.  Returns index-space vertices.
* to_world(...)         the numpy line of :473 with its dtypes.
* cull(...)             the tail of :486-492 (bound mask in float32 thresholds, update_faces,
                        remove_unreferenced_vertices), stable orders.
* vertex_colors(...)    extract_color: sdf, feature and analytic gradient at fp32 vertices, sin
                        embedding, the fp16 MLP, sigmoid, uint8(clip(c, 0, 1) * 255).
"""
import os
import re

import numpy as np

from oracle import neus_oracle as no

F32, F16 = np.float32, np.float16
HERE = os.path.dirname(os.path.abspath(__file__))
TABLES = os.path.join(os.path.dirname(HERE), "go-slam_b200", "csrc", "mc_tables.cuh")


def load_tables(path=TABLES):
    """(ntri [256] int64, tris [256, 3 * max_tris] int64) parsed from the committed header"""
    src = open(path).read()
    body_n = re.search(r"c_mc_ntri\[256\] = \{(.*?)\};", src, re.S).group(1)
    body_t = re.search(r"c_mc_tris\[256\]\[(\d+)\] = \{(.*?)\};", src, re.S)
    ntri = np.array([int(v) for v in re.findall(r"-?\d+", body_n)], np.int64)
    tris = np.array([int(v) for v in re.findall(r"-?\d+", body_t.group(2))], np.int64).reshape(256, int(body_t.group(1)))
    return ntri, tris


def _params(w):
    return (np.asarray(w["grid"], F32).astype(F16).reshape(-1, 2), np.asarray(w["sdf_w"], F32),
            np.asarray(w["sdf_b"], F32), np.asarray(w["color_B"], F32), np.asarray(w["mlp"], F32).astype(F16))


def _normalise(P, bound):
    raw = ((P - bound[:, 0]) / (bound[:, 1] - bound[:, 0]) * F32(2.0) - F32(1.0)).astype(F32)
    xn = np.clip(raw, F32(-1), F32(1))
    return raw, xn, ((xn + F32(1)) / F32(2)).astype(F32)


def sdf_points(w, P, bound):
    """SDFNetwork.sdf(P, bound): returns (sdf [n], feat [n,31], xn, raw, x01)"""
    table, sdf_w, sdf_b, _, _ = _params(w)
    raw, xn, x01 = _normalise(np.asarray(P, F32), np.asarray(bound, F32))
    enc = no.hashgrid_encode(x01, table)
    out = (np.concatenate([xn, enc.astype(F32)], 1).astype(np.float64) @ sdf_w.astype(np.float64).T + sdf_b).astype(F32)
    return out[:, 0], out[:, 1:], xn, raw, x01


def field(w, xs, ys, zs, bound, rt_bound):
    """u [nx,ny,nz] float32 (extract_fields on the given linspace tables)."""
    xs, ys, zs = (np.asarray(t, F32) for t in (xs, ys, zs))
    rt = np.asarray(rt_bound, F32)
    P = np.stack(np.meshgrid(xs, ys, zs, indexing="ij"), -1).reshape(-1, 3)
    mask = np.all((P < rt[:, 1]) & (P > rt[:, 0]), axis=1)
    u = np.full(P.shape[0], -100.0, F32)
    if mask.any():
        u[mask] = -sdf_points(w, P[mask], bound)[0]
    return u.reshape(len(xs), len(ys), len(zs))


def marching_cubes(u, iso, tables=None):
    """(vertices [V,3] float64 in index space, faces [F,3] int64)"""
    ntri_t, tris_t = tables if tables is not None else load_tables()
    u = np.asarray(u, F32)
    nx, ny, nz = u.shape
    iso = float(iso)
    ins = u.astype(np.float64) > iso
    # crossing lattice edges, ascending id
    ids, pos = [], []
    for a in range(3):
        sl0 = [slice(None)] * 3
        sl1 = [slice(None)] * 3
        sl0[a] = slice(0, u.shape[a] - 1)
        sl1[a] = slice(1, u.shape[a])
        cr = ins[tuple(sl0)] != ins[tuple(sl1)]
        x, y, z = np.nonzero(cr)
        ua = u[tuple(sl0)][cr].astype(np.float64)
        ub = u[tuple(sl1)][cr].astype(np.float64)
        t = (iso - ua) / (ub - ua)
        p = np.stack([x, y, z], 1).astype(np.float64)
        p[:, a] = p[:, a] + t
        ids.append(3 * ((x * ny + y) * nz + z).astype(np.int64) + a)
        pos.append(p)
    ids = np.concatenate(ids)
    pos = np.concatenate(pos)
    order = np.argsort(ids, kind="stable")
    ids, verts = ids[order], pos[order]
    # cells: case index, x-major / z fastest
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= ins[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz].astype(np.int64) << c
    case = case.reshape(-1)
    nt = ntri_t[case]
    cells = np.nonzero(nt)[0]
    if cells.size == 0:
        return verts.reshape(-1, 3), np.zeros((0, 3), np.int64)
    rep = np.repeat(cells, nt[cells])
    start = np.repeat(np.cumsum(nt[cells]) - nt[cells], nt[cells])
    k = np.arange(rep.size) - start
    cx = rep // ((ny - 1) * (nz - 1))
    cy = (rep // (nz - 1)) % (ny - 1)
    cz = rep % (nz - 1)
    faces = np.empty((rep.size, 3), np.int64)
    for j in range(3):
        e = tris_t[case[rep], 3 * k + j]
        a = e // 4
        o1 = np.where(a == 0, 1, 0)
        o2 = np.where(a == 2, 1, 2)
        off = np.zeros((rep.size, 3), np.int64)
        off[np.arange(rep.size), o1] = e & 1
        off[np.arange(rep.size), o2] = (e >> 1) & 1
        lin = ((cx + off[:, 0]) * ny + (cy + off[:, 1])) * nz + (cz + off[:, 2])
        eid = 3 * lin + a
        idx = np.searchsorted(ids, eid)
        assert np.all(ids[idx] == eid)
        faces[:, j] = idx
    return verts, faces


def to_world(verts, bound_min, bound_max, shape):
    """vertices / (resolution - 1.0) * (b_max_np - b_min_np)[None, :] + b_min_np[None, :]  (per-axis resolution)"""
    bmin, bmax = np.asarray(bound_min, F32), np.asarray(bound_max, F32)
    res = np.asarray(shape, np.float64)
    return verts / (res - 1.0)[None, :] * (bmax - bmin)[None, :] + bmin[None, :]


def cull(verts, faces, rt_bound, eps=0.01):
    """:486-492 on (vertices float64, faces int64): returns (vertices, faces, kept original vertex ids)"""
    bound = np.asarray(rt_bound, F32)
    bound_mask = np.all(verts >= (bound[:, 0] - eps), axis=1) & np.all(verts <= (bound[:, 1] + eps), axis=1)
    face_mask = bound_mask[faces].all(axis=1) if faces.size else np.zeros(0, bool)
    f = faces[face_mask]
    ref = np.zeros(verts.shape[0], bool)
    ref[f.reshape(-1)] = True
    new = np.cumsum(ref) - 1
    return verts[ref], new[f].reshape(-1, 3).astype(np.int64), np.nonzero(ref)[0]


def vertex_colors(w, vertices, bound):
    """extract_color(bound, vertices) -> uint8 [V,3]"""
    table, sdf_w, sdf_b, color_B, mlp = _params(w)
    P = np.asarray(vertices, np.float64).astype(F32)
    bound = np.asarray(bound, F32)
    if P.shape[0] == 0:
        return np.zeros((0, 3), np.uint8)
    sdf, feat, xn, raw, x01 = sdf_points(w, P, bound)
    genc = no.hashgrid_input_grad(x01, table, sdf_w[0, 3:])
    passthru = ((raw >= -1) & (raw <= 1)).astype(F32)
    grad = ((sdf_w[0, :3][None] + F32(0.5) * genc) * passthru * (F32(2.0) / (bound[:, 1] - bound[:, 0]))[None]).astype(F32)
    emb = np.sin((P.astype(np.float64) @ color_B.astype(np.float64)).astype(F32)).astype(F32)
    x = no.mlp_forward(np.concatenate([emb, grad, feat], 1), mlp)
    c = no._sigmoid(x.astype(F32)).astype(F16).astype(F32)
    return (np.clip(c, 0, 1) * F32(255)).astype(np.uint8)


def extract_mesh(w, bound, rt_bound, resolution, iso, color=True):
    """the whole extract_geometry(resolution, iso, None, save_path=None, color) pipeline in this project's order
    (field, marching cubes, world scaling, cull, colours of the kept vertices)."""
    import torch
    bound = np.asarray(bound, F32)
    xs, ys, zs = (torch.linspace(float(bound[a, 0]), float(bound[a, 1]), resolution).numpy() for a in range(3))
    u = field(w, xs, ys, zs, bound, rt_bound)
    v, f = marching_cubes(u, iso)
    v = to_world(v, bound[:, 0], bound[:, 1], u.shape)
    v, f, _ = cull(v, f, rt_bound)
    return u, v, f, (vertex_colors(w, v, bound) if color else None)
