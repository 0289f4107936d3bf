"""The scene bound of Mesher.update_param_from_mapping on the GPU: hull vertices against Qhull and the exact
extreme-point oracle, the oriented box and its in-bound mask against oracle/obb_oracle.py, the mapping point
selection against iproj + the reference's masks, and the drop-ins."""
import time
import types

import numpy as np
import pytest
import torch

from oracle import obb_oracle as oo
from oracle import mvfilter_oracle as mv
from test_gpu_multiview_filter import make_video, seeded_scene

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _hull(p):
    from goslam_b200 import mesher
    return mesher.hull_vertices(torch.from_numpy(np.ascontiguousarray(p)).to(DEV)).cpu().numpy()


def gaussian(n, seed, scale=(1.0, 1.0, 1.0)):
    return np.random.default_rng(seed).normal(size=(n, 3)) * np.asarray(scale)


def noisy_sphere(n, seed):
    g = np.random.default_rng(seed)
    v = g.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True) * (1.0 + 1e-3 * g.random((n, 1)))


def room(ht, wd, seed, half=(2.0, 1.5, 1.2)):
    """a box room seen from inside: depth of every pixel ray to the walls (1e-3 relative noise), back-projected in
    float32 as iproj does, widened to f64"""
    g = np.random.default_rng(seed)
    half = np.asarray(half)
    f = 0.8 * wd
    pts = []
    for k in range(6):
        a = 2 * np.pi * k / 6
        c, s = np.cos(a), np.sin(a)
        R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        v, u = np.mgrid[0:ht, 0:wd]
        d = np.stack([(u - wd / 2) / f, (v - ht / 2) / f, np.ones_like(u, float)], -1).reshape(-1, 3) @ R.T
        o = np.array([0.3 * c, 0.1, 0.2 * s])
        with np.errstate(divide="ignore"):
            t = np.where(d > 0, (half - o) / d, np.where(d < 0, (-half - o) / d, np.inf)).min(1)
        t = t * (1.0 + 1e-3 * g.normal(size=t.shape))
        pts.append((o + d * t[:, None]).astype(np.float32).astype(np.float64))
    return np.concatenate(pts)


@pytest.mark.parametrize("kind,n", [
    ("gauss", 4), ("gauss", 5), ("gauss", 50), ("gauss", 1000), ("gauss", 100000), ("gauss", 10_000_000),
    ("slab", 20000), ("slab", 1_000_000), ("sphere", 2000), ("sphere", 20000), ("room", 0),
])
def test_hull_vertices_equal_qhull(kind, n):
    if kind == "gauss":
        p = gaussian(n, 1 + n)
    elif kind == "slab":
        p = gaussian(n, 2 + n, (3.0, 2.0, 1e-3))
    elif kind == "sphere":
        p = noisy_sphere(n, 3 + n)
    else:
        p = room(60, 80, 4)
    got = _hull(p)
    want = oo.hull_vertices(p)
    assert np.array_equal(got, want), (kind, len(p), len(got), len(want), np.setxor1d(got, want)[:10])
    if kind == "sphere":
        assert len(got) > 0.5 * n


def _degenerate_cases():
    g = np.random.default_rng(7)
    lattice = np.stack(np.meshgrid(*[np.arange(5.0)] * 3, indexing="ij"), -1).reshape(-1, 3)
    corners = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 0, 1], [0, 1, 1], [1, 1, 1]], float)
    face_edge = np.concatenate([
        corners, [[0.5, 0.5, 0], [0.5, 0, 0.5], [0, 0.5, 0.5], [0.5, 0, 0], [0, 0.25, 0], [1, 1, 0.5], [0.5, 0.5, 0.5]],
        corners[[3, 5, 0]]])                                 # duplicates after their originals
    dup_first = np.concatenate([corners[[7, 2]], gaussian(30, 8) * 0.2 + 0.5, corners])     # duplicates before
    octa = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [0, 0, 0],
                     [0.5, 0.5, 0], [0.25, 0.25, 0.5]], float)
    prism = np.concatenate([g.random((40, 2)) * [4, 1], np.zeros((40, 1))], 1)
    prism = np.concatenate([prism, prism + [0, 0, 1]])
    return {"lattice": lattice, "face_edge": face_edge, "dup_first": dup_first, "octahedron": octa, "prism": prism}


@pytest.mark.parametrize("name", sorted(_degenerate_cases()))
def test_hull_vertices_exact_degeneracies(name):
    p = _degenerate_cases()[name]
    got = _hull(p)
    assert np.array_equal(got, oo.extreme_points_lp(p)), (name, got)
    if name == "lattice":
        assert len(got) == 8


@pytest.mark.parametrize("pts", [
    np.zeros((1, 3)), np.zeros((5, 3)), np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.0]]),
    np.concatenate([np.random.default_rng(1).random((100, 2)), np.zeros((100, 1))], 1),                # flat
    np.outer(np.random.default_rng(2).random(50), [1.0, 2.0, -0.5]) + [1, 1, 1],                       # collinear
    np.array([[0, 0, 0], [0, 0, 0], [1, 1, 1], [2, 2, 2.0]]),
    np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [np.nan, 0, 1.0]]),
])
def test_degenerate_input_raises(pts):
    from goslam_b200 import mesher
    with pytest.raises(ValueError):
        mesher.hull_vertices(torch.from_numpy(pts).to(DEV))
    with pytest.raises(ValueError):
        mesher.oriented_box(torch.from_numpy(pts).to(DEV))


def _box_case(seed, n=20000):
    g = np.random.default_rng(seed)
    q, _ = np.linalg.qr(g.normal(size=(3, 3)))
    return gaussian(n, seed, (3.0, 1.5, 0.5)) @ q.T + g.normal(size=3)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_box_matches_oracle(seed):
    from goslam_b200 import mesher
    p = _box_case(seed)
    c, R, e, w = oo.oriented_box(p, 0.1)
    assert (np.diff(-w) / w[0] > 1e-3).all()
    gc, gR, ge = (t.cpu().numpy() for t in mesher.oriented_box(torch.from_numpy(p).to(DEV), 0.1))
    scale = np.abs(p).max()
    assert np.abs(gR - R).max() < 1e-9, (gR, R)
    assert np.abs(gc - c).max() < 1e-9 * scale and np.abs(ge - e).max() < 1e-9 * scale
    assert abs(np.linalg.det(gR) - 1) < 1e-12
    # every input point lies inside the extended box, and the masks agree away from the faces
    inb = mesher.in_oriented_box(torch.from_numpy(p).to(DEV), gc, gR, ge).cpu().numpy()
    assert inb.all()
    x = np.concatenate([p, np.random.default_rng(seed + 9).uniform(-6, 6, size=(200000, 3))])
    got = mesher.in_oriented_box(torch.from_numpy(x).to(DEV), torch.from_numpy(gc), torch.from_numpy(gR),
                                 torch.from_numpy(ge)).cpu().numpy()
    want = oo.in_box(x, gc, gR, ge)
    face = np.abs(np.abs((x - gc) @ gR) - ge / 2).min(1) < 1e-9 * scale
    assert 0 < want.sum() < len(x)
    assert np.array_equal(got[~face], want[~face])


def test_dropin_box_class():
    from goslam_b200 import mesher
    p = _box_case(5)
    box = mesher.OrientedBoundingBox().to(DEV)
    assert [(k, v.dtype, tuple(v.shape)) for k, v in box.named_buffers()] == [
        ("center", torch.float64, (3,)), ("R", torch.float64, (3, 3)), ("extent", torch.float64, (3,))]
    box.compute_from_pointcloud(p.astype(np.float32), extend=0.1)
    c, R, e, _ = oo.oriented_box(p.astype(np.float32), 0.1)
    assert np.abs(box.R.cpu().numpy() - R).max() < 1e-9
    assert np.abs(box.center.cpu().numpy() - c).max() < 1e-8 and np.abs(box.extent.cpu().numpy() - e).max() < 1e-8
    x = np.random.default_rng(3).uniform(-8, 8, size=(50000, 3))
    a = box.in_bound(x)
    assert isinstance(a, np.ndarray) and a.dtype == np.bool_
    b = box.in_bound(torch.from_numpy(x).to(DEV))
    assert b.is_cuda and b.dtype == torch.bool and np.array_equal(b.cpu().numpy(), a)
    assert np.array_equal(a, oo.in_box(x, box.center.cpu().numpy(), box.R.cpu().numpy(), box.extent.cpu().numpy()))
    aabb = box.get_axis_aligned_bounding_box()
    assert aabb.dtype == np.float32 and aabb.shape == (3, 2)
    assert np.array_equal(aabb, oo.axis_aligned_bound(box.center.cpu().numpy(), box.R.cpu().numpy(),
                                                      box.extent.cpu().numpy()))
    other = mesher.OrientedBoundingBox().to(DEV)
    other._clone(box)
    assert all(torch.equal(a, b) for a, b in zip(other.buffers(), box.buffers()))
    gpu = mesher.OrientedBoundingBox().to(DEV)
    gpu.compute_from_pointcloud(torch.from_numpy(p.astype(np.float32)).to(DEV), extend=0.1)
    assert all(torch.equal(a, b) for a, b in zip(gpu.buffers(), box.buffers()))


def _video(T=12, ht=48, wd=64, seed=5):
    intr = [f / 8 for f in mv.full_intrinsics(ht, wd)]
    video = make_video(T + 2, ht, wd, intr)
    seeded_scene(video, T, seed)
    video.timestamp[:T] = torch.arange(T, dtype=torch.float32, device=DEV) * 2.0
    return video, T


def test_mapping_points_equal_iproj_and_reference_masks():
    from goslam_b200 import droid_backends, lietorch, mesher
    video, T = _video()
    got = mesher.mapping_points(video, T).cpu()
    want = oo.mapping_points(video, T, droid_backends.iproj, droid_backends.depth_filter, lietorch.SE3, DEV)
    assert got.dtype == torch.float64 and len(want) > 1000
    assert torch.equal(got, want.double())


def test_update_param_from_mapping_tuple():
    from goslam_b200 import droid_backends, lietorch, mesher
    video, T = _video()
    net = torch.nn.Linear(3, 2)
    self_ = types.SimpleNamespace(shared_mapping_net=net, video=video, device=DEV)
    ts, idx, dnet, box, kf = mesher.update_param_from_mapping(self_, the_end=False)
    assert box is None and idx == T - 1 and float(ts) == 2.0 * (T - 1)
    assert kf.device.type == "cpu" and kf.shape == (T, 4, 4)
    ts, idx, dnet, box, kf = mesher.update_param_from_mapping(self_, the_end=True)
    assert dnet is not net and next(dnet.parameters()).device == DEV
    assert torch.equal(dnet.weight.cpu(), net.weight)
    assert torch.equal(kf, lietorch.SE3(video.poses[:T]).inv().matrix().data.cpu())
    sel = oo.mapping_points(video, T, droid_backends.iproj, droid_backends.depth_filter, lietorch.SE3, DEV)
    c, R, e, _ = oo.oriented_box(sel.double().numpy(), 0.1)
    assert isinstance(box, mesher.OrientedBoundingBox) and box.center.device == DEV
    assert np.abs(box.R.cpu().numpy() - R).max() < 1e-9
    assert np.abs(box.center.cpu().numpy() - c).max() < 1e-8 and np.abs(box.extent.cpu().numpy() - e).max() < 1e-8


class _Trimesh:
    def __init__(self, vertices, faces, vertex_colors=None, process=True):
        self.vertices, self.faces = np.asarray(vertices), np.asarray(faces)
        self.visual = types.SimpleNamespace(vertex_colors=vertex_colors)
        self.process = process

    def export(self, path):
        pass


def test_cull_mesh_device_box_equals_host_path(tmp_path, monkeypatch):
    import sys
    from goslam_b200 import mesher
    fake = types.ModuleType("trimesh")
    fake.Trimesh = _Trimesh
    monkeypatch.setitem(sys.modules, "trimesh", fake)
    g = np.random.default_rng(4)
    V = g.uniform(-1, 1, size=(3000, 3))
    F = g.integers(0, len(V), size=(6000, 3))
    box = mesher.OrientedBoundingBox().to(DEV)
    box.compute_from_pointcloud(V[:1500] * 0.8)

    class HostBox:                       # the same box through cull_mesh's host path
        def in_bound(self, p):
            return box.in_bound(np.asarray(p))

    c2w = np.eye(4, dtype=np.float32)[None].repeat(2, 0)
    c2w[:, 2, 3] = -3.0
    self_ = types.SimpleNamespace(output=str(tmp_path), H=48, W=64, fx=40.0, fy=40.0, cx=32.0, cy=24.0,
                                  forecast_radius=0, remove_small_geometry_threshold=0.0, get_largest_components=False,
                                  device=DEV)
    out = str(tmp_path / "m.ply")
    a = mesher.cull_mesh(self_, _Trimesh(V, F), torch.from_numpy(c2w), box, out)
    b = mesher.cull_mesh(self_, _Trimesh(V, F), torch.from_numpy(c2w), HostBox(), out)
    for x, y in zip(a, b):
        assert np.array_equal(x.vertices, y.vertices) and np.array_equal(x.faces, y.faces)


def test_two_runs_bit_identical():
    from goslam_b200 import mesher
    p = torch.from_numpy(np.concatenate([room(48, 64, 9), noisy_sphere(5000, 9) * 3])).to(DEV)
    a = [mesher.hull_vertices(p), *mesher.oriented_box(p, 0.1)]
    b = [mesher.hull_vertices(p), *mesher.oriented_box(p, 0.1)]
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_replica_shaped_run():
    """250 keyframes at 320 x 640: selection, hull and box, timed; the box against the oracle"""
    from goslam_b200 import _lib, mesher
    video, T = _video(250, 320, 640, seed=11)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sel = mesher.mapping_points(video, T)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    ids = mesher.hull_vertices(sel)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    c, R, e = mesher.oriented_box(sel, 0.1)
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    _, _, _, info = mesher._hull_run(sel, "hull")
    print("\n[replica] points %d  survivors %d  hull %d  selection %.1f ms  hull %.1f ms  hull+box %.1f ms"
          % (sel.shape[0], int(info[2]), ids.numel(), 1e3 * (t1 - t0), 1e3 * (t2 - t1), 1e3 * (t3 - t2)))
    hv = sel[ids].cpu().numpy()
    oc, oR, oe, _ = oo.oriented_box(hv, 0.1)
    assert np.array_equal(oo.hull_vertices(hv), np.arange(len(hv)))
    assert np.abs(R.cpu().numpy() - oR).max() < 1e-9
    assert mesher.in_oriented_box(sel, c, R, e).all()
