"""oracle/obb_oracle.py on the CPU: its hull vertices against the linear-programming definition of an extreme point,
the box containing its points, the plane tests against the box's own frame, and the mesher's selection against the
reference-run golden."""
import os

import numpy as np
import pytest
import torch

from oracle import obb_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _clouds():
    g = np.random.default_rng(0)
    corners = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 0, 1], [0, 1, 1], [1, 1, 1]], float)
    return {
        "gauss": g.normal(size=(60, 3)),
        "sphere": (lambda v: v / np.linalg.norm(v, axis=1, keepdims=True))(g.normal(size=(40, 3))),
        "lattice": np.stack(np.meshgrid(*[np.arange(4.0)] * 3, indexing="ij"), -1).reshape(-1, 3),
        "faces_edges_dups": np.concatenate([corners[[6, 1]], corners, [[0.5, 0.5, 0], [0.5, 0, 0], [0.5, 0.5, 0.5]],
                                            corners[[0, 7]]]),
    }


@pytest.mark.parametrize("name", sorted(_clouds()))
def test_hull_vertices_equal_lp_definition(name):
    p = _clouds()[name]
    got = oo.hull_vertices(p)
    assert np.array_equal(got, oo.extreme_points_lp(p)), name
    if name == "lattice":
        assert len(got) == 8
    if name == "faces_edges_dups":
        assert got.tolist() == [0, 1, 2, 4, 5, 6, 7, 9]


def test_box_contains_points_and_plane_tests_agree():
    g = np.random.default_rng(1)
    q, _ = np.linalg.qr(g.normal(size=(3, 3)))
    p = g.normal(size=(3000, 3)) * [3.0, 1.0, 0.3] @ q.T + [1.0, -2.0, 0.5]
    c, R, e, w = oo.oriented_box(p)
    assert abs(np.linalg.det(R) - 1) < 1e-12 and (np.diff(w) < 0).all()
    assert np.abs(R.T @ R - np.eye(3)).max() < 1e-12
    local = (p - c) @ R
    assert (np.abs(local) <= e / 2 * (1 + 1e-12)).all()
    assert oo.in_box(p[np.abs(np.abs(local) - e / 2).min(1) > 1e-9], c, R, e).all()
    x = g.uniform(-8, 8, size=(100000, 3))
    lx = np.abs((x - c) @ R)
    away = np.abs(lx - e / 2).min(1) > 1e-9
    assert np.array_equal(oo.in_box(x, c, R, e)[away], (lx <= e / 2).all(1)[away])
    aabb = oo.axis_aligned_bound(c, R, e)
    assert aabb.dtype == np.float32 and (aabb[:, 0] <= p.min(0) + 1e-6).all() and (aabb[:, 1] >= p.max(0) - 1e-6).all()


def test_golden_selection_reproduced():
    from oracle import geom_oracle
    g = np.load(os.path.join(ROOT, "tests", "golden", "obb.npz"))
    T = int(g["cur_idx"])
    video = _golden_video(g)

    class SE3:
        from goslam_b200 import lietorch as _l
        def __new__(cls, data):
            return SE3._l.SE3(data)

    def iproj(poses, disps, intr):
        return torch.from_numpy(geom_oracle.iproj(poses.numpy(), disps.numpy(), intr.numpy()))

    def depth_filter(poses, disps, intr, ix, thresh):
        return torch.from_numpy(geom_oracle.depth_filter(poses.numpy(), disps.numpy(), intr.numpy(), ix.numpy(),
                                                         thresh.numpy()))

    got = oo.mapping_points(video, T, iproj, depth_filter, SE3, "cpu")
    assert np.array_equal(got.numpy(), g["sel_points"])
    assert float(g["extend"]) == 0.1


def _golden_video(g):
    import types
    return types.SimpleNamespace(poses=torch.from_numpy(g["poses"]), disps_up=torch.from_numpy(g["disps_up"]),
                                 intrinsics=torch.from_numpy(g["intrinsics"]), scale_factor=8,
                                 pose_compensate=torch.from_numpy(g["pose_compensate"]))
