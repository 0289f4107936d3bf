"""Mesh extraction on the CPU: the generated marching-cubes tables, the oracle's marching cubes on analytic and random
fields, the oracle against the reference's own extract_fields / extract_color (tests/golden/mesh.npz), and argument
validation of the new C-ABI entries (no GPU)."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from oracle import neus_oracle as no

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mesh.npz")


def _gen():
    spec = importlib.util.spec_from_file_location("gen_mc_tables", os.path.join(ROOT, "tools", "gen_mc_tables.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_committed_header_is_the_generators_output():
    g = _gen()
    assert open(g.OUT).read() == g.render_header(), "run tools/gen_mc_tables.py"
    ntri, tris = mo.load_tables()
    ntri_g, tris_g = g.build_tables()
    assert np.array_equal(ntri, ntri_g) and np.array_equal(tris, tris_g)


def test_tables_all_cases():
    """for all 256 cases: triangle vertices sit on crossing edges, each crossing edge is used, the loops close on the
    cube faces and follow the face rule, and every loop segment has the inside corners on the stated side"""
    g = _gen()
    ntri, tris = mo.load_tables()
    assert ntri[0] == 0 and ntri[255] == 0
    for case in range(256):
        ins = [bool((case >> c) & 1) for c in range(8)]
        crossing = {e for e in range(12) if ins[g.edge_corners(e)[0]] != ins[g.edge_corners(e)[1]]}
        used = set(int(e) for e in tris[case, :3 * ntri[case]])
        assert used == crossing, case
        assert np.all(tris[case, 3 * ntri[case]:] == -1)
        loops = g.case_loops(case)
        assert sum(len(lp) for lp in loops) == len(crossing)
        assert ntri[case] == sum(len(lp) - 2 for lp in loops)
        segs = {(lp[k], lp[(k + 1) % len(lp)]) for lp in loops for k in range(len(lp))}
        for n, ring in g.faces():
            face_edges = {g.edge_between(ring[k], ring[(k + 1) % 4]) for k in range(4)}
            on_face = [s for s in segs if s[0] in face_edges and s[1] in face_edges]
            fin = [ins[c] for c in ring]
            n_cross = sum(fin[k] != fin[(k + 1) % 4] for k in range(4))
            amb = sum(fin) == 2 and fin[0] == fin[2]
            assert len(on_face) == (2 if amb else n_cross // 2), (case, ring)
            for s0, s1 in on_face:
                p0, p1 = g.edge_mid(s0), g.edge_mid(s1)
                # the corners adjacent to this segment's two edges that are inside: the segment cuts them off
                ends = set(g.edge_corners(s0)) | set(g.edge_corners(s1))
                for c in ring:
                    if c in ends and ins[c]:
                        if amb and not ({c} <= set(g.edge_corners(s0)) and {c} <= set(g.edge_corners(s1))):
                            continue      # on an ambiguous face each segment cuts off one corner only
                        side = np.dot(n, np.cross(p1 - p0, g.corner_pos(c) - p0))
                        assert side < 0, (case, s0, s1, c)
        # each loop's vector area (the sum of its fan triangles' (v1 - v0) x (v2 - v0) / 2) points from the inside ends
        # of its edges towards the outside ends
        for lp in loops:
            p = [g.edge_mid(e) for e in lp]
            area = sum(np.cross(p[k], p[(k + 1) % len(p)]) for k in range(len(p))) / 2.0
            fan = sum(np.cross(p[k] - p[0], p[k + 1] - p[0]) for k in range(1, len(p) - 1)) / 2.0
            assert np.allclose(area, fan)
            out = 0.0
            for e in lp:
                a, b = g.edge_corners(e)
                cin, cout = (a, b) if ins[a] else (b, a)
                out += np.dot(area, g.corner_pos(cout) - g.corner_pos(cin))
            assert out > 0, (case, lp)


def _euler(v, f):
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    return len(v) - len(np.unique(e, axis=0)) + len(f)


def _volume(v, f):
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0


def _closed_and_oriented(f):
    """every directed edge appears once and its reverse once: each edge shared by exactly two faces, opposite directions"""
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = d[:, 0] * (f.max() + 1) + d[:, 1]
    rev = d[:, 1] * (f.max() + 1) + d[:, 0]
    return len(np.unique(key)) == len(key) and np.array_equal(np.sort(key), np.sort(rev))


def _grid(n, c):
    return np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64)] * 3, indexing="ij"), -1) - c


def test_oracle_sphere():
    r = 30.0
    u = (r - np.linalg.norm(_grid(96, 47.3), axis=-1)).astype(np.float32)
    v, f = mo.marching_cubes(u, 0.0)
    assert _euler(v, f) == 2 and _closed_and_oriented(f)
    vol = _volume(v, f)
    assert vol > 0 and abs(vol / (4.0 / 3.0 * np.pi * r ** 3) - 1.0) < 0.01


def test_oracle_torus():
    g = _grid(64, 31.6)
    u = (8.0 - np.sqrt((np.sqrt(g[..., 0] ** 2 + g[..., 1] ** 2) - 20.0) ** 2 + g[..., 2] ** 2)).astype(np.float32)
    v, f = mo.marching_cubes(u, 0.0)
    assert _euler(v, f) == 0 and _closed_and_oriented(f) and _volume(v, f) > 0


@pytest.mark.parametrize("n", [8, 11, 16])
@pytest.mark.parametrize("iso", [0.0, 0.05, -0.05])
def test_oracle_random_fields_are_closed(n, iso):
    """random values inside, outside on the lattice's boundary: a closed surface, every edge on two faces"""
    rng = np.random.default_rng(n)
    u = rng.standard_normal((n, n, n)).astype(np.float32)
    u[[0, -1]], u[:, [0, -1]], u[:, :, [0, -1]] = -1.0, -1.0, -1.0
    v, f = mo.marching_cubes(u, iso)
    assert len(f) > 0 and _closed_and_oriented(f)
    assert np.array_equal(np.unique(f), np.arange(len(v)))
    # every vertex lies on its lattice edge
    frac = v - np.floor(v)
    assert np.all((frac > 0).sum(1) <= 1)


def test_oracle_edge_cases():
    # values exactly at iso are outside (u > iso is inside): the vertex lands on the inside end when ua == iso... never;
    # t == 1 when ub == iso
    u = np.full((5, 5, 5), -1.0, np.float32)
    u[2, 2, 2] = 1.0
    u[2, 2, 3] = 0.0
    v, f = mo.marching_cubes(u, 0.0)
    assert _closed_and_oriented(f) and np.any(np.all(v == [2.0, 2.0, 3.0], axis=1))
    for val in (5.0, -5.0):                                   # all inside, all outside
        v, f = mo.marching_cubes(np.full((6, 7, 8), val, np.float32), 0.0)
        assert v.shape == (0, 3) and f.shape == (0, 3)
    for n in (2, 3):
        rng = np.random.default_rng(n)
        for _ in range(20):
            u = rng.standard_normal((n, n, n)).astype(np.float32)
            v, f = mo.marching_cubes(u, 0.0)
            assert f.size == 0 or (f.min() >= 0 and f.max() < len(v))


def test_oracle_cull_keeps_orders():
    rng = np.random.default_rng(3)
    u = rng.standard_normal((12, 12, 12)).astype(np.float32)
    v, f = mo.marching_cubes(u, 0.0)
    vw = mo.to_world(v, np.float32([-1, -1, -1]), np.float32([1, 1, 1]), u.shape)
    cv, cf, kept = mo.cull(vw, f, np.float32([[-0.5, 0.6], [-0.7, 0.4], [-1, 1]]))
    assert 0 < len(cf) < len(f)
    assert np.array_equal(cv[cf], vw[kept][cf]) and np.all(np.diff(kept) > 0)
    assert np.array_equal(np.unique(cf), np.arange(len(cv)))


def _golden_weights(g):
    from goslam_b200 import synthetic
    metas, tot = no.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [tot * 2]
    return synthetic.make_neus_weights(seed=int(g["weights_seed"]), total_grid_params=tot * 2,
                                       layout=(offs, [m["res"] for m in metas]))


def test_oracle_matches_reference_golden():
    """the oracle's field and colours against the reference's own extract_fields / extract_color"""
    g = np.load(GOLDEN)
    w = _golden_weights(g)
    b, rt = g["bound"], g["rt_bound"]
    for res, sel, want in ((33, None, g["u33"]), (70, g["idx70"], g["u70"])):
        tabs = [torch.linspace(float(b[a, 0]), float(b[a, 1]), res).numpy() for a in range(3)]
        u = mo.field(w, *tabs, b, rt)
        got = u if sel is None else u.reshape(-1)[sel]
        assert np.array_equal(got == -100.0, want == -100.0)
        assert np.abs(got - want).max() < 1e-6
    c = mo.vertex_colors(w, g["vertices"], b)
    d = np.abs(c.astype(np.int64) - g["colors"].astype(np.int64))
    assert d.max() <= 1 and (d == 0).mean() >= 0.99


def test_mesh_abi_validation_without_gpu(lib):
    from goslam_b200 import _lib
    null = ctypes.c_void_p(None)
    one = ctypes.c_void_p(16)
    f3 = (ctypes.c_float * 3)(0.0, 0.0, 0.0)
    assert lib.goslam_mc_workspace_bytes(1, 4, 4) == 0
    assert lib.goslam_mc_workspace_bytes(2, 2, 2) > 0
    # 1.125 bytes per lattice point (crossing bits + per-word prefix) plus the per-block tables
    n = 1024 ** 3
    assert 1.125 * n <= lib.goslam_mc_workspace_bytes(1024, 1024, 1024) < 1.2 * n
    assert lib.goslam_mc_count(null, 4, 4, 4, 0.0, null, 0, one, null) == -1                 # no field
    assert lib.goslam_mc_count(one, 1, 4, 4, 0.0, one, 1 << 20, one, null) == -1             # nx < 2
    assert lib.goslam_mc_count(one, 4, 4, 4, float("nan"), one, 1 << 20, one, null) == -1    # iso NaN
    assert lib.goslam_mc_count(one, 4, 4, 4, 0.0, null, 0, one, null) == -3                  # no workspace
    assert lib.goslam_mc_emit(one, 4, 4, 4, 0.0, f3, null, one, 1 << 20, null, 0, null, 0, null) == -1
    assert lib.goslam_mc_emit(one, 4, 4, 4, 0.0, f3, f3, one, 1 << 20, null, 5, null, 0, null) == -1   # rows, no buffer
    assert lib.goslam_mc_emit(one, 4, 4, 4, 0.0, f3, f3, one, 16, null, 0, null, 0, null) == -3
    assert lib.goslam_mesh_cull_workspace_bytes(-1, 0) == 0 < lib.goslam_mesh_cull_workspace_bytes(0, 0)
    assert lib.goslam_mesh_cull_count(null, 4, null, 0, f3, f3, one, 1 << 20, one, null) == -1
    assert lib.goslam_mesh_cull_count(null, 0, null, 0, f3, f3, null, 0, one, null) == -3
    assert lib.goslam_mesh_cull_emit(one, 4, null, 2, one, 1 << 20, one, 4, null, 0, null) == -1      # faces missing
    assert lib.goslam_mesh_cull_emit(one, 4, one, 2, one, 1 << 20, one, 4, null, 2, null) == -1       # output missing
    p = _lib.NeusParams()
    assert lib.goslam_neus_sdf_grid(None, one, one, one, 4, 4, 4, one, null) == -1
    assert lib.goslam_neus_sdf_grid(ctypes.byref(p), one, one, one, 0, 4, 4, one, null) == -1
    assert lib.goslam_neus_vertex_color(ctypes.byref(p), null, 5, null, null) == -1
    assert lib.goslam_neus_vertex_color(ctypes.byref(p), null, 0, null, null) == 0            # nothing to colour


def test_extraction_needs_a_cuda_network():
    from goslam_b200 import neus, synthetic
    net = neus.InstantNeuS(synthetic.NEUS_CFG, [[-1.0, 1.0]] * 3, device="cpu")
    pts = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.5, -0.99, 0.2]])
    assert net.in_bound(pts, net.bound).tolist() == [True, False, True]
    with pytest.raises(RuntimeError, match="CUDA"):
        net.extract_fields(net.bound[:, 0], net.bound[:, 1], 8)
