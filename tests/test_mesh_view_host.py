"""CPU checks of the mesh-view oracle (oracle/mesh_view_oracle.py) and of the new C-ABI entries' argument validation:
the rasterizer on analytic scenes, the point_masks restatement against the reference's own method (golden), and the
component rule on hand-built meshes."""
import ctypes
import os

import numpy as np
import pytest

from oracle import mesh_view_oracle as mvo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W, FX, FY, CX, CY = 60, 80, 50.0, 50.0, 39.5, 29.5
EYE = np.eye(4, dtype=np.float32)[None]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "mesh_view.npz"))


def _render(v, f, c2w=EYE, **kw):
    args = dict(H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY)
    args.update(kw)
    return mvo.render_depth(np.asarray(v, np.float64), np.asarray(f, np.int64), c2w, **args)


def test_plane_at_known_depth_and_nearest_wins():
    quad = [[-10, -10, 2.0], [10, -10, 2.0], [10, 10, 2.0], [-10, 10, 2.0]]
    d = _render(quad, [[0, 1, 2], [0, 2, 3]])[0]
    assert d.dtype == np.float32 and np.all(d == 2.0)
    back = [[x, y, 3.0] for x, y, _ in quad]
    d = _render(quad + back, [[4, 5, 6], [4, 6, 7], [0, 1, 2], [0, 2, 3]])[0]
    assert np.all(d == 2.0)


def test_pixel_centre_convention_and_inclusive_edges():
    # at z = 1 with fx = fy = 1, cx = cy = 0 screen coordinates are camera x, y: the triangle x, y >= 0, x + y <= 4
    d = _render([[0, 0, 1], [4, 0, 1], [0, 4, 1]], [[0, 1, 2]], H=8, W=8, fx=1.0, fy=1.0, cx=0.0, cy=0.0)[0]
    r, c = np.nonzero(d)
    # centres (c + 0.5, r + 0.5) with (c + 0.5) + (r + 0.5) <= 4: c + r <= 3, the diagonal ones lie on the edge
    assert set(zip(r.tolist(), c.tolist())) == {(i, j) for i in range(8) for j in range(8) if i + j <= 3}
    assert np.all(d[d > 0] == 1.0)


def test_both_windings_and_zero_area():
    v = [[-1, -1, 3.0], [2, -1, 4.0], [0, 2, 5.0]]
    a = _render(v, [[0, 1, 2]])
    assert (a > 0).sum() > 100
    # the other winding covers the same pixels except where a centre lies on an edge (the edge function is evaluated
    # from its other end and rounds differently); the interpolation sums in another order
    b = _render(v, [[0, 2, 1]])
    both = (a > 0) & (b > 0)
    assert ((a > 0) != (b > 0)).sum() <= 2 and np.allclose(a[both], b[both], rtol=1e-6, atol=0)
    assert not _render([[-1, -1, 3.0], [0, 0, 3.0], [1, 1, 3.0]], [[0, 1, 2]]).any()     # collinear
    assert not _render([[-1, -1, 3.0], [-1, -1, 3.0], [1, 1, 3.0]], [[0, 1, 2]]).any()   # repeated vertex


def test_near_clip_far_discard_and_background():
    # a floor y = 1 from z = -5 (behind the camera) to z = 50: row r sees it at z = fy / (r + 0.5 - cy) = 50 / (r - 29)
    v = [[-50, 1, -5.0], [50, 1, -5.0], [0, 1, 50.0]]
    d = _render(v, [[0, 1, 2]])[0]
    assert not d[:30].any()                                      # above the horizon: background
    assert not d[30:32].any()                                    # z = 50, 25: beyond far = 20
    for r in range(32, H):
        want = 50.0 / (r - 29)
        cols = np.nonzero(d[r])[0]
        assert len(cols) == W                                    # the floor spans the view
        assert np.allclose(d[r], want, rtol=1e-6), r
    # the same floor with far = 100 reaches the rows up to the triangle's tip
    assert d.astype(bool).sum() < _render(v, [[0, 1, 2]], far=100.0)[0].astype(bool).sum()
    # entirely behind the near plane: nothing
    assert not _render([[-1, -1, -1.0], [1, -1, -1.0], [0, 1, 0.0005]], [[0, 1, 2]]).any()


def test_full_screen_quad_and_pose():
    # a camera at (0, 0, -1) looking along +z, rotated 90 degrees about z, sees the quad z = 0.5 at depth 1.5
    c2w = np.eye(4, dtype=np.float32)
    c2w[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]
    c2w[2, 3] = -1.0
    quad = [[-100, -100, 0.5], [100, -100, 0.5], [100, 100, 0.5], [-100, 100, 0.5]]
    d = _render(quad, [[0, 1, 2], [2, 3, 0]], c2w[None])[0]
    assert np.all(d == 1.5)


def test_golden_depth_and_masks_match_the_reference(golden):
    H_, W_, fx, fy, cx, cy = golden["intrinsics"].tolist()
    H_, W_ = int(H_), int(W_)
    d = mvo.render_depth(golden["verts"], golden["faces"], golden["c2w"], H_, W_, fx, fy, cx, cy)
    assert np.array_equal(d.view(np.int32), golden["depth"].view(np.int32))
    seen, fore = mvo.point_masks(golden["verts"], golden["depth"], golden["c2w"], H_, W_, fx, fy, cx, cy,
                                 int(golden["radius"]))
    assert np.array_equal(seen, golden["seen"]) and np.array_equal(fore, golden["forecast"])
    assert 0 < seen.sum() < fore.sum() < len(seen)
    assert np.all(fore[seen])


def _square(x0, y0, base=0):
    v = [[x0, y0, 0.0], [x0 + 1, y0, 0.0], [x0 + 1, y0 + 1, 0.0], [x0, y0 + 1, 0.0]]
    return v, [[base, base + 1, base + 2], [base, base + 2, base + 3]]


def test_components_vertex_touch_three_faces_isolated():
    a, fa = _square(0, 0)
    b, fb = _square(1, 1, 4)                 # touches square a at the vertex (1, 1) only (a duplicate vertex id below)
    v = a + b
    f = fa + fb
    f[2] = [2, 5, 6]                         # b's first face uses a's vertex 2 in place of its own corner
    f[3] = [2, 6, 7]
    lab = mvo.component_labels(np.array(f))
    assert lab.tolist() == [0, 0, 2, 2]
    # an edge shared by three faces joins none of them; a face elsewhere is alone
    v3 = [[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [5, 5, 5], [6, 5, 5], [5, 6, 5]]
    f3 = [[0, 1, 2], [1, 0, 3], [0, 1, 4], [5, 6, 7]]
    assert mvo.component_labels(np.array(f3)).tolist() == [0, 1, 2, 3]
    f3[1] = [1, 0, 3]
    f3 = f3[:2] + f3[3:]                     # two faces on the edge: adjacent
    assert mvo.component_labels(np.array(f3)).tolist() == [0, 0, 2]


def test_components_threshold_is_strict_and_largest_breaks_ties():
    a, fa = _square(0, 0)
    b, fb = _square(3, 0, 4)
    v, f = np.array(a + b, np.float64), np.array(fa + fb)
    assert mvo.face_areas(v, f).tolist() == [0.5] * 4
    # two components of area 1 in a mesh of area 2: threshold 0.5 keeps neither (1 > 1 is false)
    assert not mvo.component_face_mask(v, f, 0.5).any()
    assert mvo.component_face_mask(v, f, 0.49).all()
    assert mvo.component_face_mask(v, f, 0.0, largest=True).tolist() == [True, True, False, False]
    rv, rf, rc = mvo.components(v, f, 0.5, colors=np.arange(8)[:, None])
    assert rv.shape == (0, 3) and rf.shape == (0, 3) and rc.shape == (0, 1)
    # a larger second component wins `largest`
    v[4:, :2] *= 2.0
    assert mvo.component_face_mask(v, f, 0.0, largest=True).tolist() == [False, False, True, True]
    kv, kf, kc = mvo.components(v, f, 0.3, True, colors=np.arange(8)[:, None])
    assert np.array_equal(kv, v[4:]) and kf.tolist() == [[0, 1, 2], [0, 2, 3]] and kc[:, 0].tolist() == [4, 5, 6, 7]


def test_keep_faces_is_stable_and_carries_colours():
    v = np.arange(18, dtype=np.float64).reshape(6, 3)
    f = np.array([[0, 1, 2], [3, 4, 5], [1, 3, 5]])
    kv, kf, kc, ids = mvo.keep_faces(v, f, [False, True, True], colors=np.arange(6) * 10)
    assert ids.tolist() == [1, 3, 4, 5] and kf.tolist() == [[1, 2, 3], [0, 1, 3]] and kc.tolist() == [10, 30, 40, 50]
    assert np.array_equal(kv, v[[1, 3, 4, 5]])


def test_argument_validation_without_gpu(lib):
    null = ctypes.c_void_p(None)
    cnt = (ctypes.c_int64 * 2)()
    # depth: bad sizes, missing pointers, bad near / far; K = 0 is a no-op
    assert lib.goslam_mesh_depth_render(null, 3, null, 1, null, 1, 4, 4, 1.0, 1.0, 0.0, 0.0, 0.001, 20.0, null, null) == -1
    assert lib.goslam_mesh_depth_render(null, 0, null, 0, null, 1, 0, 4, 1.0, 1.0, 0.0, 0.0, 0.001, 20.0, null, null) == -1
    assert lib.goslam_mesh_depth_render(null, 0, null, 0, null, 0, 4, 4, 1.0, 1.0, 0.0, 0.0, 0.0, 20.0, null, null) == -1
    assert lib.goslam_mesh_depth_render(null, 0, null, 0, null, 0, 4, 4, 1.0, 1.0, 0.0, 0.0, 0.1, 0.05, null, null) == -1
    assert lib.goslam_mesh_depth_render(null, 0, null, 0, null, 70000, 4, 4, 1.0, 1.0, 0.0, 0.0, 0.001, 20.0, null, null) == -1
    assert lib.goslam_mesh_depth_render(null, 0, null, 0, null, 0, 4, 4, 1.0, 1.0, 0.0, 0.0, 0.001, 20.0, null, null) == 0
    # masks: H, W >= 2, pointers, radius >= 0; nothing to do is a no-op
    assert lib.goslam_mesh_view_masks(null, 5, null, null, 1, 4, 4, 1, 1, 0, 0, 0, 0.05, null, null, null) == -1
    assert lib.goslam_mesh_view_masks(null, 0, null, null, 1, 1, 4, 1, 1, 0, 0, 0, 0.05, null, null, null) == -1
    assert lib.goslam_mesh_view_masks(null, 0, null, null, 0, 4, 4, 1, 1, 0, 0, -1, 0.05, null, null, null) == -1
    assert lib.goslam_mesh_view_masks(null, 0, null, null, 0, 4, 4, 1, 1, 0, 0, 25, 0.05, null, null, null) == 0
    # components
    assert lib.goslam_mesh_components_workspace_bytes(-1, 4) == 0
    assert lib.goslam_mesh_components_workspace_bytes(4, 1 << 31) == 0
    assert lib.goslam_mesh_components_count(null, 4, null, 2, null, 0, cnt, null) == -1
    assert lib.goslam_mesh_components_count(null, 0, null, 0, null, 0, None, null) == -1
    assert lib.goslam_mesh_components_keep(4, 5, 0.2, 0, null, 0, null, null) == -1          # more components than faces
    assert lib.goslam_mesh_components_keep(4, 0, 0.2, 0, null, 0, null, null) == -1
    assert lib.goslam_mesh_components_keep(4, 2, float("nan"), 0, null, 0, null, null) == -1
    assert lib.goslam_mesh_components_keep(0, 0, 0.2, 0, null, 0, null, null) == -3          # no workspace
    # face-mask cull and vertex ids
    assert lib.goslam_mesh_cull_mask_count(4, null, 2, null, null, null, 0, cnt, null) == -1
    assert lib.goslam_mesh_cull_mask_count(-1, null, 0, null, null, null, 0, cnt, null) == -1
    assert lib.goslam_mesh_cull_mask_count(4, null, 0, null, null, null, 0, cnt, null) == -3
    assert lib.goslam_mesh_cull_vertex_ids(4, 2, null, 0, null, 3, null) == -1
    assert lib.goslam_mesh_cull_vertex_ids(4, 2, null, 0, null, 0, null) == -3
