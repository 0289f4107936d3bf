"""The reconstruction evaluation on the device (goslam_b200.mesher: sample_surface, nearest, icp_point_to_point,
mesh_metrics and the drop-ins align_mesh / eval_mesh) against tests/golden/mesh_eval.npz and brute-force fp64
restatements.  Needs neither scipy, Open3D, trimesh nor the reference tree.

Samples and nearest distances are compared bit for bit (distances within 1 ulp, threshold counts equal); the ICP result
within 1e-9 of the oracle's (its sums run in another order)."""
import io
import contextlib
import math
import os

import numpy as np
import pytest
import torch

from goslam_b200 import mesher, neus, synthetic
from oracle import mesh_eval_oracle as meo
from oracle import neus_oracle as no

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "mesh_eval.npz")))


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


class StandIn:
    """what align_mesh / eval_mesh read of a trimesh.Trimesh"""

    def __init__(self, v, f):
        self.vertices, self.faces = np.array(v, np.float64), np.array(f, np.int64)

    def apply_transform(self, M):
        h = np.c_[self.vertices, np.ones(len(self.vertices))] @ np.asarray(M).T
        self.vertices = h[:, :3] / h[:, 3:]
        return self


def brute(q, p, max_dist=math.inf):
    """(dist, idx) by comparing every pair in fp64, (dx^2 + dy^2) + dz^2, the smallest index among equal minima"""
    q, p = q.to(DEV, torch.float64), p.to(DEV, torch.float64)
    dists, idxs = [], []
    for q0 in range(0, q.shape[0], 256):
        c = q[q0:q0 + 256]
        dx, dy, dz = (c[:, None, j] - p[None, :, j] for j in range(3))
        d2 = (dx * dx + dy * dy) + dz * dz
        if not math.isinf(max_dist):
            d2 = torch.where(d2 < max_dist * max_dist, d2, torch.full_like(d2, math.inf))
        m = d2.min(1).values
        i = torch.argmax((d2 == m[:, None]).to(torch.int8), 1)
        dists.append(torch.sqrt(m))
        idxs.append(torch.where(torch.isinf(m), torch.full_like(i, -1), i))
    return torch.cat(dists), torch.cat(idxs)


def _ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a.view(np.int64) - b.view(np.int64)).max()


# ---- sampling -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["est", "gt"])
def test_samples_match_golden(golden, which):
    v, f = golden[which + "_verts"], golden[which + "_faces"]
    got = mesher.sample_surface_from(_cuda(v), _cuda(f), _cuda(golden["u_" + which])).cpu().numpy()
    want, face = golden["s_" + which], golden["f_" + which]
    same = (got == want).all(1)
    if not same.all():
        # a face choice may differ only where u * total lies within 1e-12 * total of a cumulative boundary
        cum = np.cumsum(meo.face_areas(v, f))
        t = golden["u_" + which][~same, 0] * cum[-1]
        near = np.abs(cum[face[~same]] - t) <= 1e-12 * cum[-1]
        near |= np.abs(cum[np.maximum(face[~same] - 1, 0)] - t) <= 1e-12 * cum[-1]
        assert near.all(), "samples differ away from face boundaries"
    assert same.mean() > 0.999


def test_sample_surface_draws_from_the_generator():
    v, f = _cuda(np.eye(3)), _cuda(np.array([[0, 1, 2]]))
    a = mesher.sample_surface(v, f, 1000, torch.Generator(DEV).manual_seed(5))
    b = mesher.sample_surface(v, f, 1000, torch.Generator(DEV).manual_seed(5))
    assert torch.equal(a, b) and a.shape == (1000, 3)
    assert (a.sum(1) - 1).abs().max() < 1e-15 and (a >= 0).all()
    with pytest.raises(ValueError):
        mesher.sample_surface(v, f[:0], 10)
    with pytest.raises(RuntimeError):
        mesher.sample_surface(v.cpu(), f.cpu(), 10)


# ---- nearest neighbours -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", [("s_gt", "s_est", "comp"), ("s_est", "s_gt", "acc")])
def test_nearest_matches_golden(golden, direction):
    q, p, key = direction
    dist, idx = mesher.nearest(_cuda(golden[q]), _cuda(golden[p]))
    dist, idx = dist.cpu().numpy(), idx.cpu().numpy()
    want = golden[key + "_dist"]
    assert _ulps(dist, want) <= 1
    assert (dist == want).mean() == 1.0
    th = float(golden["dist_th"])
    assert (dist < th).sum() == (want < th).sum()
    # the returned index attains the distance (ties may pick another index than cKDTree)
    assert np.array_equal(np.sqrt(meo.sq_dist(golden[q], golden[p][idx])), dist)


def _hand_cases():
    g = torch.Generator().manual_seed(9)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)  # noqa: E731
    pts = r(500, 3)
    dup = torch.cat([pts[:100], pts[:100], pts[50:60]])                       # duplicate points
    cases = {
        "duplicates": (torch.cat([r(300, 3), dup[:40]]), dup),
        "query_on_point": (pts[::7].clone(), pts),                            # distance 0
        "one_point": (r(200, 3) * 4 - 2, r(1, 3)),
        "far_outside": (torch.cat([r(50, 3) * 1e3 + 500, -r(50, 3) * 1e3, torch.tensor([[0.5, 0.5, 1e4],
                                                                                      [-1e5, 0.5, 0.5]])]), pts),
        "two_clusters": (torch.cat([r(200, 3) * 7 - 1, r(50, 3) * 0.01 + 3.5]),
                         torch.cat([r(300, 3) * 0.05, r(300, 3) * 0.05 + torch.tensor([6.0, 5.0, 4.0])])),
        "flat": (r(300, 3), torch.cat([r(400, 2), torch.zeros(400, 1)], 1)),
        "collinear": (r(300, 3), torch.cat([r(400, 1)] * 3, 1)),
    }
    return cases


@pytest.mark.parametrize("case", list(_hand_cases()))
@pytest.mark.parametrize("max_dist", [math.inf, 0.05, 1e-6])
def test_nearest_hand_cases(case, max_dist):
    q, p = _hand_cases()[case]
    dist, idx = mesher.nearest(q.to(DEV), p.to(DEV), max_dist)
    wd, wi = brute(q, p, max_dist)
    assert torch.equal(dist, wd) and torch.equal(idx, wi)
    if max_dist == 1e-6 and case not in ("duplicates", "query_on_point"):
        assert (idx == -1).all() and torch.isinf(dist).all()                 # a radius below every distance


def test_index_reuse_and_workspace_queries():
    from goslam_b200 import _lib
    lib = _lib.load()
    assert lib.goslam_nn_index_workspace_bytes(0) == 0 and lib.goslam_nn_index_workspace_bytes(1 << 29) == 0
    assert lib.goslam_icp_workspace_bytes(0) == 0 and lib.goslam_mesh_sample_workspace_bytes(0) == 0
    assert lib.goslam_nn_index_workspace_bytes(1000) < lib.goslam_nn_index_workspace_bytes(2000)
    g = torch.Generator().manual_seed(3)
    p = torch.rand(5000, 3, generator=g, dtype=torch.float64)
    index = mesher.NNIndex(p.to(DEV), 0.02)
    for k in range(3):
        q = torch.rand(700, 3, generator=g, dtype=torch.float64) * 1.2 - 0.1
        for md in (math.inf, 0.02):
            d, i = index.query(q.to(DEV), md)
            wd, wi = brute(q, p, md)
            assert torch.equal(d, wd) and torch.equal(i, wi)


# ---- ICP ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("init", ["rigid", "scaled"])
def test_icp_matches_golden(golden, init):
    T, fit, rmse, it = mesher.icp_point_to_point(_cuda(golden["est_verts"]), _cuda(golden["gt_verts"]),
                                                 float(golden["threshold"]), golden["icp_init_" + init])
    assert it == int(golden["icp_iterations_" + init])
    assert np.abs(T.numpy() - golden["icp_T_" + init]).max() < 1e-9
    assert abs(fit - float(golden["icp_fitness_" + init])) <= 1e-12 * abs(float(golden["icp_fitness_" + init]))
    assert abs(rmse - float(golden["icp_rmse_" + init])) <= 1e-12 * abs(float(golden["icp_rmse_" + init]))


def test_icp_without_correspondences_returns_init():
    init = meo.rigid([0, 0, 1], 0.1, [5.0, 0, 0])
    src = torch.rand(100, 3, dtype=torch.float64, device=DEV)
    T, fit, rmse, it = mesher.icp_point_to_point(src, src + 100.0, 0.1, init)
    assert np.array_equal(T.numpy(), init) and fit == 0.0 and rmse == 0.0 and it == 1
    T, fit, rmse, it = mesher.icp_point_to_point(src, src, 0.1, init, max_iteration=0)
    assert np.array_equal(T.numpy(), init) and it == 0


# ---- drop-ins -----------------------------------------------------------------------------------------------------
def test_dropins_reproduce_golden(golden, monkeypatch, tmp_path):
    est = StandIn(golden["est_verts"], golden["est_faces"])
    gt = StandIn(golden["gt_verts"], golden["gt_faces"])
    draws = [golden["u_est"], golden["u_gt"]]
    monkeypatch.setattr(mesher, "_uniforms", lambda n, gen, dev: _cuda(draws.pop(0)))
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        m = mesher.eval_mesh(est, gt, N3d=int(golden["n3d"]), dist_th=float(golden["dist_th"]),
                             out_path=str(tmp_path / "metrics_mesh.txt"))
    msg = str(golden["message"])
    assert (tmp_path / "metrics_mesh.txt").read_text() == msg and out.getvalue() == msg + "\n"
    want = golden["metrics"]
    got = [m[k] for k in ("accuracy", "completion", "accuracy_ratio", "completion_ratio", "f_score")]
    assert np.allclose(got, want, rtol=1e-12, atol=0)
    aligned, T = mesher.align_mesh(est, gt, threshold=float(golden["threshold"]), trans_init=golden["icp_init_rigid"],
                                   return_transformation=True)
    assert aligned is est and isinstance(T, np.ndarray) and T.dtype == np.float64 and T.shape == (4, 4)
    assert np.abs(T - golden["icp_T_rigid"]).max() < 1e-9
    want_v = StandIn(golden["est_verts"], golden["est_faces"]).apply_transform(golden["icp_T_rigid"]).vertices
    assert np.abs(aligned.vertices - want_v).max() < 1e-8
    with pytest.raises(ValueError):
        mesher.align_mesh(StandIn(np.zeros((0, 3)), np.zeros((0, 3))), gt)


def test_eval_mesh_same_generator_state_same_metrics(golden):
    est = StandIn(golden["est_verts"], golden["est_faces"])
    gt = StandIn(golden["gt_verts"], golden["gt_faces"])
    with contextlib.redirect_stdout(io.StringIO()):
        torch.cuda.manual_seed(21)
        a = mesher.eval_mesh(est, gt, N3d=20000)
        torch.cuda.manual_seed(21)
        b = mesher.eval_mesh(est, gt, N3d=20000)
        c = mesher.eval_mesh(est, gt, N3d=20000, generator=torch.Generator(DEV).manual_seed(21))
    assert a == b and set(a) == {"accuracy", "completion", "accuracy_ratio", "completion_ratio", "f_score"}
    # another stream of draws: the same estimator, close values
    assert abs(a["accuracy"] - c["accuracy"]) < 0.5 and abs(a["completion"] - c["completion"]) < 0.5


# ---- the size the grid exists for ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def res512():
    metas, tot = no.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [tot * 2]
    g = np.load(os.path.join(ROOT, "tests", "golden", "mesh.npz"))
    w = synthetic.make_neus_weights(seed=int(g["weights_seed"]), total_grid_params=tot * 2,
                                    layout=(offs, [m["res"] for m in metas]))
    net = neus.InstantNeuS(synthetic.NEUS_CFG, g["bound"].tolist())
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to(DEV)
    net.update_bound(torch.from_numpy(g["rt_bound"]))
    out = net.extract_mesh(512, 0.0)
    return out[0], out[1]


def test_res512_icp_and_nearest(res512):
    v, _ = res512
    assert v.shape[0] > 500000
    M = meo.rigid([0.4, -0.7, 0.2], np.deg2rad(0.3), [0.004, -0.003, 0.002])
    dst = _cuda(meo.transform(v.cpu().numpy(), M))
    T, fit, rmse, it = mesher.icp_point_to_point(v, dst, 0.1, max_iteration=60, relative_fitness=1e-12,
                                                 relative_rmse=1e-12)
    assert fit == 1.0 and np.abs(T.numpy() - M).max() < 1e-6, (T, fit, rmse, it)
    sub = torch.randperm(v.shape[0], generator=torch.Generator().manual_seed(1))[:10000].to(DEV)
    q = v[sub]
    for md in (math.inf, 0.1):
        d, i = mesher.nearest(q, dst, md)
        wd, wi = brute(q, dst, md)
        assert torch.equal(d, wd) and torch.equal(i, wi)
