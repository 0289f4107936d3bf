"""The projection and component culls of Mesher.cull_mesh on the device (goslam_b200.mesher) against the reference's own
point_masks (tests/golden/mesh_view.npz) and the numpy restatement (oracle/mesh_view_oracle.py).

Depth maps, face-mask culls and the component filter are compared bit for bit.  The masks are the reference's f32
arithmetic on another device: a vertex may differ from the golden only where some view puts it within 1e-5 (relative) of
a decision boundary, and on at most 0.01 % of the vertices."""
import os
import sys
import time
import types

import numpy as np
import pytest
import torch

from goslam_b200 import mesher, neus, synthetic
from oracle import mesh_view_oracle as mvo
from oracle import neus_oracle as no

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


@pytest.fixture(scope="module")
def golden():
    g = np.load(os.path.join(ROOT, "tests", "golden", "mesh_view.npz"))
    H, W, fx, fy, cx, cy = g["intrinsics"].tolist()
    return dict(g), (int(H), int(W), fx, fy, cx, cy)


def _cuda(*a):
    return [torch.from_numpy(np.ascontiguousarray(x)).to(DEV) for x in a]


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_depth_bit_identical_on_golden(golden):
    g, cam = golden
    v, f = _cuda(g["verts"], g["faces"])
    d = mesher.render_depth(v, f, torch.from_numpy(g["c2w"]), *cam).cpu().numpy()
    assert _bits_equal(d, g["depth"])
    # poses as a list of tensors (the reference's estimate_c2w_list), one view at a time
    d1 = mesher.render_depth(v, f, [torch.from_numpy(m) for m in g["c2w"][:3]], *cam).cpu().numpy()
    assert _bits_equal(d1, g["depth"][:3])


def _rot_z(a, t):
    m = np.eye(4, dtype=np.float32)
    m[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    m[:3, 3] = t
    return m


QUAD = [[-100, -100, 0.5], [100, -100, 0.5], [100, 100, 0.5], [-100, 100, 0.5]]
HAND = {
    "plane": (QUAD, [[0, 1, 2], [0, 2, 3]], [np.eye(4, dtype=np.float32)], dict(H=60, W=80, fx=50.0, fy=50.0, cx=39.5, cy=29.5)),
    "centres": ([[0, 0, 1], [4, 0, 1], [0, 4, 1]], [[0, 1, 2]], [np.eye(4, dtype=np.float32)],
                dict(H=8, W=8, fx=1.0, fy=1.0, cx=0.0, cy=0.0)),
    "near_far": ([[-50, 1, -5.0], [50, 1, -5.0], [0, 1, 50.0]], [[0, 1, 2], [0, 2, 1]], [np.eye(4, dtype=np.float32)],
                 dict(H=60, W=80, fx=50.0, fy=48.0, cx=39.5, cy=29.5)),
    "zero_area": ([[-1, -1, 3.0], [0, 0, 3.0], [1, 1, 3.0], [1, 1, 3.0]], [[0, 1, 2], [1, 3, 2]], [np.eye(4, dtype=np.float32)],
                  dict(H=60, W=80, fx=50.0, fy=50.0, cx=39.5, cy=29.5)),
    # a full-screen quad at 320 x 640, seen from two rotated poses: every lane of the warp pass walks the whole image
    "full_screen_quad": (QUAD, [[0, 1, 2], [2, 3, 0]], [_rot_z(0.3, [0, 0, -1.0]), _rot_z(-1.2, [0.2, 0.1, -0.2])],
                         dict(H=320, W=640, fx=320.0, fy=282.0, cx=319.5, cy=159.5)),
}


@pytest.mark.parametrize("case", sorted(HAND))
def test_depth_bit_identical_on_hand_cases(case):
    v, f, c2w, cam = HAND[case]
    v, f = np.asarray(v, np.float64), np.asarray(f, np.int64)
    want = mvo.render_depth(v, f, np.stack(c2w), **cam)
    got = mesher.render_depth(*_cuda(v, f), torch.from_numpy(np.stack(c2w)), **cam).cpu().numpy()
    assert _bits_equal(got, want), case
    if case == "full_screen_quad":
        assert (got > 0).all()
    if case == "zero_area":
        assert not got.any()


def _mask_check(got, want, margin, what):
    bad = got != want
    n = int(bad.sum())
    print("%s: %d of %d vertices differ, all within 1e-5 of a boundary: %s" % (what, n, len(got), bool((margin[bad] < 1e-5).all())))
    assert (margin[bad] < 1e-5).all(), what
    assert n <= 1e-4 * len(got), what


def test_masks_vs_golden(golden):
    g, cam = golden
    v, f = _cuda(g["verts"], g["faces"])
    r = int(g["radius"])
    seen, fore = mesher.view_masks(v, f, torch.from_numpy(g["c2w"]), *cam, r)
    s5, f5 = mesher.view_masks(v, f, torch.from_numpy(g["c2w"]), *cam, r, chunk=5)
    assert torch.equal(seen, s5) and torch.equal(fore, f5)
    margin = mvo.mask_margins(g["verts"], g["depth"], g["c2w"], *cam, r)
    _mask_check(seen.cpu().numpy(), g["seen"], margin, "seen")
    _mask_check(fore.cpu().numpy(), g["forecast"], margin, "forecast")


def _same_mesh(got, want, what):
    gv, gf, gc = [None if t is None else t.cpu().numpy() for t in got]
    wv, wf, wc = want[:3]
    assert _bits_equal(gv, np.asarray(wv, np.float64)), what
    assert np.array_equal(gf, wf), what
    assert (gc is None) == (wc is None) and (gc is None or np.array_equal(gc, wc)), what


def test_keep_faces_and_components_vs_oracle(golden):
    g, cam = golden
    V, F, C = g["verts"], g["faces"], g["colors"]
    v, f, c = _cuda(V, F, C)
    fm = g["seen"][F].all(1)
    _same_mesh(mesher.keep_faces(v, f, torch.from_numpy(fm), colors=c), mvo.keep_faces(V, F, fm, C), "keep_faces")
    _same_mesh(mesher.keep_faces(v, f, colors=c, vert_mask=torch.from_numpy(g["seen"])), mvo.keep_faces(V, F, fm, C),
               "keep_faces by vertex mask")
    hv, hf, hc, _ = mvo.keep_faces(V, F, fm, C)
    dh = _cuda(hv, hf, hc)
    for thr, largest in ((0.0, False), (0.01, False), (0.2, False), (0.0, True), (1.0, False)):
        got = mesher.filter_components(*dh[:2], thr, largest, colors=dh[2])
        want = mvo.components(hv, hf, thr, largest, hc)
        _same_mesh(got, want, "components %g %s" % (thr, largest))
    assert len(mvo.components(hv, hf, 0.0)[1]) > len(mvo.components(hv, hf, 0.2)[1]) > 0
    assert len(mvo.components(hv, hf, 1.0)[1]) == 0
    # hand-built: a vertex touch, an edge on three faces, an isolated face, two equal areas at the threshold
    v3 = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [5, 5, 5], [6, 5, 5], [5, 6, 5], [1, 1, 0]], float)
    f3 = np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [5, 6, 7], [1, 8, 2], [2, 8, 5]])
    for thr, largest in ((0.0, False), (0.1, False), (0.0, True)):
        want = mvo.components(v3, f3, thr, largest, np.arange(9))
        _same_mesh(mesher.filter_components(*_cuda(v3, f3), thr, largest, colors=_cuda(np.arange(9))[0]), want, "hand")
    sq = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [3, 0, 0], [4, 0, 0], [4, 1, 0], [3, 1, 0]], float)
    fs = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]])
    assert mesher.filter_components(*_cuda(sq, fs), 0.5)[1].shape == (0, 3)
    assert mesher.filter_components(*_cuda(sq, fs), 0.49)[1].shape == (4, 3)
    assert mesher.filter_components(*_cuda(sq, fs), 0.0, True)[1].cpu().tolist() == [[0, 1, 2], [0, 2, 3]]
    e = mesher.filter_components(*_cuda(np.zeros((0, 3)), np.zeros((0, 3), np.int64)), 0.2)
    assert e[0].shape == (0, 3) and e[1].shape == (0, 3)


# ---- cull_mesh end to end with stand-ins for trimesh and Open3D ------------------------------------------------------
class _FakeTrimesh:
    exported = {}

    def __init__(self, vertices, faces, vertex_colors=None, process=True):
        self.vertices, self.faces = np.asarray(vertices), np.asarray(faces)
        self.visual = types.SimpleNamespace(vertex_colors=vertex_colors)
        self.process = process

    def export(self, path):
        _FakeTrimesh.exported[os.path.basename(path)] = self


def _aabb_indices(box_pts, pts):
    """the stand-in oriented box: the axis-aligned box of the points"""
    lo, hi = box_pts.min(0), box_pts.max(0)
    return np.nonzero(np.all((pts >= lo) & (pts <= hi), axis=1))[0]


def _fake_open3d():
    o3d = types.ModuleType("open3d")
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a, np.float64))

    class PointCloud:
        def __init__(self, pts):
            self.pts = pts

        def get_oriented_bounding_box(self):
            box = self.pts
            return types.SimpleNamespace(get_point_indices_within_bounding_box=lambda p: list(_aabb_indices(box, p)))
    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud)
    return o3d


def _oracle_cull(V, F, C, bound, self_, c2w):
    """the reference's cull_mesh steps on the oracle, with the device's masks"""
    b = np.all(V >= bound[:, 0] - 0.001, axis=1) & np.all(V <= bound[:, 1] + 0.001, axis=1)
    bv, bf, bc, _ = mvo.keep_faces(V, F, b[F].all(1), C)
    seen, fore = mesher.view_masks(*_cuda(bv, bf), torch.from_numpy(c2w), self_.H, self_.W, self_.fx, self_.fy, self_.cx,
                                   self_.cy, self_.forecast_radius)
    seen, fore = seen.cpu().numpy(), fore.cpu().numpy()
    hole = mvo.keep_faces(bv, bf, seen[bf].all(1), bc)
    cull = mvo.components(hole[0], hole[1], self_.remove_small_geometry_threshold, False, hole[2])
    fv, ff, fc, _ = mvo.keep_faces(bv, bf, fore[bf].all(1), bc)
    inb = np.zeros(len(fv), bool)
    inb[_aabb_indices(cull[0], fv)] = True
    fv, ff, fc, _ = mvo.keep_faces(fv, ff, inb[ff].all(1), fc)
    return (bv, bf, bc), hole, cull, mvo.components(fv, ff, self_.remove_small_geometry_threshold, False, fc)


def _same_trimesh(got, want, what):
    assert _bits_equal(np.asarray(got.vertices, np.float64), np.asarray(want[0], np.float64)), what
    assert np.array_equal(got.faces, want[1]), what
    assert np.array_equal(got.visual.vertex_colors, want[2]), what
    assert got.process is False


def test_cull_mesh_end_to_end(golden, tmp_path, monkeypatch):
    g, (H, W, fx, fy, cx, cy) = golden
    fake = types.ModuleType("trimesh")
    fake.Trimesh = _FakeTrimesh
    monkeypatch.setitem(sys.modules, "trimesh", fake)
    monkeypatch.setitem(sys.modules, "open3d", _fake_open3d())
    V, F = g["verts"], g["faces"]
    C = np.concatenate([g["colors"], np.full((len(V), 1), 255, np.uint8)], 1)           # trimesh keeps RGBA
    self_ = types.SimpleNamespace(output=str(tmp_path), H=H, W=W, fx=fx, fy=fy, cx=cx, cy=cy, forecast_radius=25,
                                  remove_small_geometry_threshold=0.2, get_largest_components=False, device=DEV)
    lo, hi = V.min(0), V.max(0)
    bound = np.stack([lo + 0.1 * (hi - lo), hi], 1).astype(np.float32)                    # cuts off one side
    want = _oracle_cull(V, F, C, bound, self_, g["c2w"])
    assert 0 < len(want[2][1]) < len(want[1][1]) < len(want[0][1]) < len(F)
    outs = []
    for run in range(2):
        _FakeTrimesh.exported = {}
        mesh = _FakeTrimesh(V, F, vertex_colors=C)
        out = str(tmp_path / "mesh" / "final_raw_mesh.ply")
        cull, forecast = mesher.cull_mesh(self_, mesh, [torch.from_numpy(m) for m in g["c2w"]], bound, out)
        ex = _FakeTrimesh.exported
        assert sorted(ex) == ["bound_mesh.ply", "final_raw_mesh.ply", "final_raw_mesh_forecast.ply", "mesh_with_hole.ply"]
        assert ex["final_raw_mesh.ply"] is cull and ex["final_raw_mesh_forecast.ply"] is forecast
        _same_trimesh(ex["bound_mesh.ply"], want[0], "bound")
        _same_trimesh(ex["mesh_with_hole.ply"], want[1], "hole")
        _same_trimesh(cull, want[2], "cull")
        _same_trimesh(forecast, want[3], "forecast")
        outs.append([np.asarray(m.vertices).copy() for m in (cull, forecast)] + [np.asarray(m.faces).copy() for m in (cull, forecast)])
    assert all(np.array_equal(a, b) for a, b in zip(*outs))
    # forecast_radius 0: the forecast mesh is the culled mesh
    self_.forecast_radius = 0
    cull, forecast = mesher.cull_mesh(self_, _FakeTrimesh(V, F, vertex_colors=C), torch.from_numpy(g["c2w"]), None, out)
    assert np.array_equal(cull.faces, forecast.faces) and np.array_equal(cull.vertices, forecast.vertices)


# ---- a Replica-shaped run ---------------------------------------------------------------------------------------------
def _scene_net():
    gm = np.load(os.path.join(ROOT, "tests", "golden", "mesh.npz"))
    metas, tot = no.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [tot * 2]
    w = synthetic.make_neus_weights(seed=int(gm["weights_seed"]), total_grid_params=tot * 2,
                                    layout=(offs, [m["res"] for m in metas]))
    net = neus.InstantNeuS(synthetic.NEUS_CFG, gm["bound"].tolist())
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to(DEV)
    net.update_bound(torch.from_numpy(gm["rt_bound"]))
    return net, gm


def trajectory(centre, n, seed=0):
    """n OpenCV camera-to-world poses on a wobbling loop around `centre`, looking across the scene"""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 4, 4), np.float32)
    for i in range(n):
        t = 2 * np.pi * i / n
        p = centre + np.array([0.8 * np.cos(t), 0.8 * np.sin(t), 0.15 * np.sin(3 * t)]) + rng.normal(0, 0.01, 3)
        tgt = centre + np.array([1.5 * np.cos(t + 2.0), 1.5 * np.sin(t + 2.0), 0.2 * np.cos(2 * t)])
        z = tgt - p
        z /= np.linalg.norm(z)
        x = np.cross(z, [0.0, 0.0, 1.0])
        x /= np.linalg.norm(x)
        out[i, :3, :3] = np.stack([x, np.cross(z, x), z], 1)
        out[i, :3, 3], out[i, 3, 3] = p, 1.0
    return out


def test_replica_shaped_run():
    net, gm = _scene_net()
    verts, faces, rgb = net.extract_mesh(512, 0.0, color=True)
    V, F = verts.shape[0], faces.shape[0]
    rt = gm["rt_bound"].astype(np.float64)
    c2w = torch.from_numpy(trajectory((rt[:, 0] + rt[:, 1]) / 2, 2000)).to(DEV)
    H, W, fx, fy, cx, cy = 320, 640, 320.0, 282.0, 319.5, 159.5
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    seen, fore = mesher.view_masks(verts, faces, c2w, H, W, fx, fy, cx, cy, 25)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    hv, hf, hc = mesher.keep_faces(verts, faces, colors=rgb, vert_mask=seen)
    cv, cf, cc = mesher.filter_components(hv, hf, 0.2, colors=hc)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    peak = torch.cuda.max_memory_allocated() - base
    chunk = max(1, mesher.DEPTH_CHUNK_BYTES // (4 * H * W))
    scratch = chunk * (4 * H * W + 64)
    mesh_bytes = V * (24 + 3) + F * 24
    per = (peak - scratch) / (V + F)
    print("replica-shaped: V %d F %d, 2000 views 320x640: masks %.1f ms, hole + components %.1f ms; seen %d forecast %d, "
          "culled F %d; peak %.2f GB = depth scratch %.2f GB + %.1f B per vertex and face"
          % (V, F, (t1 - t0) * 1e3, (t2 - t1) * 1e3, int(seen.sum()), int(fore.sum()), cf.shape[0], peak / 1e9,
             scratch / 1e9, per))
    assert 0 < int(seen.sum()) < V and cf.shape[0] > 0
    assert peak <= scratch + 2 * mesh_bytes + 200 * (V + F)
