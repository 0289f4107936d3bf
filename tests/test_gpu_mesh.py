"""Mesh extraction on the device (InstantNeuS.extract_fields / extract_geometry / extract_color) against the reference's
own methods (tests/golden/mesh.npz) and the numpy restatement (oracle/mesh_oracle.py).

Marching cubes and the cull are compared bit for bit: the field is copied to the host first, so both sides see the same
lattice values.  The field itself is compared to 1e-5 absolute (hash-grid gathers agree exactly; the SDF head's fp32
dot product differs from the fp64 restatement in the last bits), colours to 1 unit with at least 99 % exact (fp16 MLP
accumulation order)."""
import copy
import sys
import types

import numpy as np
import pytest
import torch

from goslam_b200 import neus, synthetic
from oracle import mesh_oracle as mo
from oracle import neus_oracle as no

pytestmark = pytest.mark.gpu
GOLDEN = "tests/golden/mesh.npz"


def _weights(seed):
    metas, tot = no.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [tot * 2]
    return synthetic.make_neus_weights(seed=seed, total_grid_params=tot * 2, layout=(offs, [m["res"] for m in metas]))


@pytest.fixture(scope="module")
def golden():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), GOLDEN))


@pytest.fixture(scope="module")
def scene(golden):
    w = _weights(int(golden["weights_seed"]))
    net = neus.InstantNeuS(synthetic.NEUS_CFG, golden["bound"].tolist())
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to("cuda:0")
    net.update_bound(torch.from_numpy(golden["rt_bound"]))
    return net, w, golden["bound"], golden["rt_bound"]


def _tables(bound, res):
    return [torch.linspace(float(bound[a, 0]), float(bound[a, 1]), res).numpy() for a in range(3)]


def _check_field(u, want, what):
    assert np.array_equal(u == -100.0, want == -100.0), what
    inb = want != -100.0
    err = float(np.abs(u[inb] - want[inb]).max()) if inb.any() else 0.0
    print("%s: %d in-bound points, max |sdf error| %.3g" % (what, int(inb.sum()), err))
    assert err <= 1e-5, what


def test_field_vs_golden_and_oracle(scene, golden):
    net, w, bound, rt = scene
    bt = net.bound
    _check_field(net.extract_fields(bt[:, 0], bt[:, 1], 33), golden["u33"], "res 33 vs reference")
    u70 = net.extract_fields(bt[:, 0].cpu(), bt[:, 1].cpu(), 70)
    _check_field(u70.reshape(-1)[golden["idx70"]], golden["u70"], "res 70 sample vs reference")
    u = net.extract_fields(bt[:, 0], bt[:, 1], 128)
    assert u.dtype == np.float32 and u.shape == (128, 128, 128)
    _check_field(u, mo.field(w, *_tables(bound, 128), bound, rt), "res 128 vs oracle")
    # a lattice over another box than the normalisation bound of the net
    lo, hi = np.float32([-1.0, -0.5, 0.0]), np.float32([0.5, 1.0, 1.5])
    u = net.extract_fields(torch.from_numpy(lo), torch.from_numpy(hi), 40)
    tabs = [torch.linspace(float(lo[a]), float(hi[a]), 40).numpy() for a in range(3)]
    _check_field(u, mo.field(w, *tabs, np.stack([lo, hi], 1), rt), "res 40 sub-box vs oracle")


def _field(kind, shape, seed=0):
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij"), -1)
    c = (np.array(shape, np.float64) - 1) / 2 + 0.137
    if kind == "sphere":
        return (0.35 * min(shape) - np.linalg.norm(g - c, axis=-1)).astype(np.float32) / 10
    if kind == "torus":
        d = g - c
        R, r = 0.3 * min(shape), 0.1 * min(shape)
        return ((r - np.sqrt((np.sqrt(d[..., 0] ** 2 + d[..., 1] ** 2) - R) ** 2 + d[..., 2] ** 2)) / 10).astype(np.float32)
    if kind == "random":
        return rng.standard_normal(shape).astype(np.float32) * 0.2
    if kind == "exact_iso":                                   # many values exactly at 0 and at +-0.05
        return (rng.integers(-2, 3, shape) * 0.05).astype(np.float32)
    if kind == "all_in":
        return np.full(shape, 1.0, np.float32)
    if kind == "all_out":
        return np.full(shape, -100.0, np.float32)
    raise ValueError(kind)


def _mc_compare(u, iso, bmin, bmax):
    verts, faces = neus.marching_cubes(torch.from_numpy(u).cuda(), iso, bmin, bmax)
    v, f = mo.marching_cubes(u, iso)
    vw = mo.to_world(v, bmin, bmax, u.shape)
    got_v, got_f = verts.cpu().numpy(), faces.cpu().numpy()
    assert got_v.dtype == np.float64 and got_f.dtype == np.int64
    assert got_v.shape == vw.shape and got_f.shape == f.shape
    assert np.array_equal(got_v.view(np.int64), vw.view(np.int64)), "vertices differ bitwise"
    assert np.array_equal(got_f, f)
    return got_v, got_f


MC_CASES = [("sphere", (17, 17, 17), 0.0), ("sphere", (64, 64, 64), 0.05), ("torus", (129, 129, 129), -0.05),
            ("torus", (256, 256, 256), 0.0), ("random", (2, 2, 2), 0.0), ("random", (3, 3, 3), 0.0),
            ("random", (17, 17, 17), 0.05), ("random", (64, 64, 64), -0.05), ("random", (5, 9, 13), 0.0),
            ("exact_iso", (17, 17, 17), 0.0), ("exact_iso", (33, 20, 9), 0.05), ("exact_iso", (16, 16, 16), -0.05),
            ("all_in", (9, 9, 9), 0.0), ("all_out", (9, 9, 9), 0.0), ("random", (2, 2, 2), 5.0)]


@pytest.mark.parametrize("kind,shape,iso", MC_CASES, ids=["%s-%s-%g" % (k, "x".join(map(str, s)), i) for k, s, i in MC_CASES])
def test_marching_cubes_vs_oracle(kind, shape, iso):
    u = _field(kind, shape, seed=sum(shape))
    v, f = _mc_compare(u, iso, np.float32([-1.5, -1.0, 0.25]), np.float32([2.0, 1.0, 3.5]))
    if kind in ("all_in", "all_out") or iso == 5.0:
        assert v.shape == (0, 3) and f.shape == (0, 3)
    else:
        assert len(f) > 0


@pytest.mark.parametrize("res,iso", [(17, 0.0), (64, 0.05), (129, -0.05), (256, 0.0)])
def test_marching_cubes_on_network_field(scene, res, iso):
    net, w, bound, rt = scene
    u = net.extract_fields(net.bound[:, 0], net.bound[:, 1], res)
    v, f = _mc_compare(u, iso, bound[:, 0], bound[:, 1])
    assert len(f) > 0


def test_cull_vs_oracle(scene):
    net, w, bound, rt = scene
    u = net.extract_fields(net.bound[:, 0], net.bound[:, 1], 96)
    v, f = mo.marching_cubes(u, 0.0)
    vw = mo.to_world(v, bound[:, 0], bound[:, 1], u.shape)
    box = np.float32([[-1.0, 0.9], [-0.6, 1.1], [-0.2, 1.4]])      # cuts through the surface
    for b in (box, rt, np.float32([[5, 6], [5, 6], [5, 6]])):
        cv, cf, _ = mo.cull(vw, f, b)
        lo, hi = (b[:, 0] - 0.01).tolist(), (b[:, 1] + 0.01).tolist()
        gv, gf = neus.cull_mesh(torch.from_numpy(vw).cuda(), torch.from_numpy(f).cuda(), lo, hi)
        gv, gf = gv.cpu().numpy(), gf.cpu().numpy()
        assert np.array_equal(gv.view(np.int64), cv.view(np.int64)) and np.array_equal(gf, cf)
    assert 0 < len(mo.cull(vw, f, box)[1]) < len(f)


def _colors_close(got, want, what):
    d = np.abs(got.astype(np.int64) - want.astype(np.int64))
    print("%s: %d vertices, max |diff| %d, exact %.4f" % (what, len(d), d.max() if d.size else 0, (d == 0).mean() if d.size else 1))
    assert got.dtype == np.uint8 and got.shape == want.shape
    assert d.size == 0 or (d.max() <= 1 and (d == 0).mean() >= 0.99), what


def test_colors_vs_golden_and_oracle(scene, golden):
    net, w, bound, rt = scene
    got = net.extract_color(net.bound.clone(), golden["vertices"])
    _colors_close(got, golden["colors"], "golden vertices vs reference")
    _colors_close(got, mo.vertex_colors(w, golden["vertices"], bound), "golden vertices vs oracle")
    u = net.extract_fields(net.bound[:, 0], net.bound[:, 1], 64)
    v, f = mo.marching_cubes(u, 0.0)
    vw = mo.to_world(v, bound[:, 0], bound[:, 1], u.shape)
    _colors_close(net.extract_color(net.bound, vw), mo.vertex_colors(w, vw, bound), "mesh vertices vs oracle")
    assert net.extract_color(net.bound, np.zeros((0, 3))).shape == (0, 3)


class _FakeTrimesh:
    calls = []

    def __init__(self, vertices, faces, vertex_colors=None):
        _FakeTrimesh.calls.append(dict(vertices=vertices, faces=faces, vertex_colors=vertex_colors))
        self.vertices, self.faces = vertices, faces
        self.exported = []

    def export(self, path):
        self.exported.append(path)


def test_extract_geometry_end_to_end(scene, monkeypatch):
    net, w, bound, rt = scene
    fake = types.ModuleType("trimesh")
    fake.Trimesh = _FakeTrimesh
    monkeypatch.setitem(sys.modules, "trimesh", fake)
    _FakeTrimesh.calls.clear()
    res = 256
    u = net.extract_fields(net.bound[:, 0], net.bound[:, 1], res)
    # the field against the oracle on a seeded sample of lattice points (the whole 256^3 restatement is slow)
    sel = np.random.default_rng(0).choice(res ** 3, 20000, replace=False)
    tabs = _tables(bound, res)
    idx = np.unravel_index(sel, u.shape)
    P = np.stack([tabs[0][idx[0]], tabs[1][idx[1]], tabs[2][idx[2]]], 1)
    inb = np.all((P < rt[:, 1]) & (P > rt[:, 0]), axis=1)
    want = np.full(len(sel), -100.0, np.float32)
    want[inb] = -mo.sdf_points(w, P[inb], bound)[0]
    _check_field(u.reshape(-1)[sel], want, "res 256 sample vs oracle")
    # the oracle pipeline on this field
    v, f = mo.marching_cubes(u, 0.0)
    v, f, _ = mo.cull(mo.to_world(v, bound[:, 0], bound[:, 1], u.shape), f, rt)
    want_rgb = mo.vertex_colors(w, v, bound)
    outs = []
    for model in (net, copy.deepcopy(net)):
        mesh = model.extract_geometry(res, 0.0, None, save_path=None, color=True)
        call = _FakeTrimesh.calls[-1]
        assert mesh.exported == []
        assert np.array_equal(call["vertices"].view(np.int64), v.view(np.int64))
        assert np.array_equal(call["faces"], f) and len(f) > 0
        _colors_close(call["vertex_colors"], want_rgb, "extract_geometry colours vs oracle")
        outs.append(call)
    assert all(np.array_equal(outs[0][k], outs[1][k]) for k in ("vertices", "faces", "vertex_colors"))
    mesh = net.extract_geometry(64, 0.0, None, save_path="somewhere.ply", color=False)
    assert mesh.exported == ["somewhere.ply"] and _FakeTrimesh.calls[-1]["vertex_colors"] is None


def test_extract_mesh_c2w_ref(scene):
    net, w, bound, rt = scene
    ang = 0.3
    c2w = torch.tensor([[np.cos(ang), -np.sin(ang), 0.0, 0.2], [np.sin(ang), np.cos(ang), 0.0, -0.1],
                        [0.0, 0.0, 1.0, 0.05], [0.0, 0.0, 0.0, 1.0]], dtype=torch.float32)
    verts, faces, rgb = net.extract_mesh(96, 0.0, c2w_ref=c2w.cuda(), color=True)
    u = net.extract_fields(net.bound[:, 0], net.bound[:, 1], 96)
    v, f = mo.marching_cubes(u, 0.0)
    v = mo.to_world(v, bound[:, 0], bound[:, 1], u.shape)
    c = c2w.numpy()                                         # src/InstantNeuS.py:475-479
    homo = np.concatenate([v, np.ones_like(v[:, :1])], axis=1)
    v = np.matmul(c[None, :, :], homo[:, :, None])[:, :3, 0]
    v, f, _ = mo.cull(v, f, rt)
    got = verts.cpu().numpy()
    assert got.shape == v.shape and np.array_equal(faces.cpu().numpy(), f)
    assert np.abs(got - v).max() <= 1e-12
    _colors_close(rgb.cpu().numpy(), mo.vertex_colors(w, got, bound), "c2w_ref colours vs oracle")


def test_extract_mesh_1024(scene):
    """one run at 1024^3: peak memory within u + 2 bytes per lattice point + the mesh arrays, mesh invariants on the
    device, and a 64^3 block of the field through the oracle"""
    net, w, bound, rt = scene
    res = 1024
    n = res ** 3
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    verts, faces, rgb = net.extract_mesh(res, 0.0, color=True)
    peak = torch.cuda.max_memory_allocated() - base
    kept = (verts.numel() + faces.numel()) * 8 + rgb.numel()
    del verts, faces, rgb
    u = net._sdf_grid(net.bound[:, 0].tolist(), net.bound[:, 1].tolist(), res)
    v, f = neus.marching_cubes(u, 0.0, bound[:, 0], bound[:, 1])
    mesh = (v.numel() + f.numel()) * 8
    print("1024^3: V %d F %d, peak %.2f GB = u %.2f GB + %.3f bytes per lattice point besides u and the mesh arrays"
          % (v.shape[0], f.shape[0], peak / 1e9, 4 * n / 1e9, (peak - 4 * n - mesh - kept) / n))
    assert peak <= 4 * n + 2 * n + mesh + kept
    V = v.shape[0]
    assert f.shape[0] > 0 and int(f.min()) >= 0 and int(f.max()) < V
    assert bool((torch.bincount(f.reshape(-1), minlength=V) > 0).all())
    # realtime_bound lies inside the lattice, so the surface is closed: every edge on exactly two faces, opposite ways
    d = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key, rev = d[:, 0] * V + d[:, 1], d[:, 1] * V + d[:, 0]
    key, _ = torch.sort(key)
    assert bool((key[1:] != key[:-1]).all())
    assert torch.equal(key, torch.sort(rev)[0])
    del v, f, d, key, rev
    # a 64^3 block that the surface crosses, through the oracle
    for x0 in range(0, res - 64, 64):
        sub = u[x0:x0 + 64, 448:512, 448:512]
        if bool((sub > 0).any()) and bool((sub <= 0).any()):
            break
    hu = sub.contiguous().cpu().numpy()
    _mc_compare(hu, 0.0, np.float32([0, 0, 0]), np.float32([1, 1, 1]))
    tabs = _tables(bound, res)
    sl = [tabs[0][x0:x0 + 64], tabs[1][448:512], tabs[2][448:512]]
    _check_field(hu, mo.field(w, *sl, bound, rt), "res 1024 block vs oracle")
