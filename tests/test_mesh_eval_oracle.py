"""CPU checks of the reconstruction-evaluation oracle (oracle/mesh_eval_oracle.py): Umeyama, ICP, surface sampling and
the golden's metrics."""
import os

import numpy as np
from scipy import stats

from oracle import mesh_eval_oracle as meo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sphere_mesh(n=24):
    """a closed UV sphere of radius 1 with uneven face areas"""
    th, ph = np.linspace(0, np.pi, n)[1:-1], np.linspace(0, 2 * np.pi, 2 * n, endpoint=False)
    v = [[0, 0, 1.0], [0, 0, -1.0]]
    for t in th:
        for p in ph:
            v.append([np.sin(t) * np.cos(p), np.sin(t) * np.sin(p), np.cos(t)])
    v = np.array(v)
    m, f = 2 * n, []
    ring = lambda i, j: 2 + i * m + j % m  # noqa: E731
    for j in range(m):
        f.append([0, ring(0, j), ring(0, j + 1)])
        f.append([1, ring(len(th) - 1, j + 1), ring(len(th) - 1, j)])
    for i in range(len(th) - 1):
        for j in range(m):
            f += [[ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)], [ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)]]
    return v, np.array(f, np.int64)


def test_umeyama_recovers_rigid_motion():
    rng = np.random.default_rng(0)
    src = rng.normal(size=(200, 3)) * [1.0, 2.0, 0.5]
    M = meo.rigid([0.2, 1.0, -0.3], 0.7, [0.5, -1.0, 2.0])
    T = meo.umeyama(src, meo.transform(src, M))
    assert np.abs(T - M).max() < 1e-12


def test_umeyama_planar_and_mirrored_sets():
    rng = np.random.default_rng(1)
    src = np.c_[rng.normal(size=(100, 2)), np.zeros(100)]          # rank-2 cross-covariance: det(U) det(V) may be -1
    M = meo.rigid([0.5, -0.2, 1.0], 2.5, [0.1, 0.2, 0.3])
    T = meo.umeyama(src, meo.transform(src, M))
    assert np.abs(T - M).max() < 1e-12
    # a mirrored target: the reflection fix keeps a proper rotation, the best one (flip of the least spread axis)
    src = np.array([[x, y, z] for x in (-3.0, 3.0) for y in (-2.0, 2.0) for z in (-0.1, 0.1)]) + [1.0, 2.0, 3.0]
    T = meo.umeyama(src, src * [1.0, 1.0, -1.0])        # sigma = diag(+, +, -)
    assert abs(np.linalg.det(T[:3, :3]) - 1.0) < 1e-12
    assert np.abs(T[:3, :3] - np.eye(3)).max() < 1e-12


def test_icp_recovers_rigid_motion_of_a_sampled_surface():
    v, f = _sphere_mesh()
    v = v * [1.0, 0.7, 0.5]                                         # an ellipsoid: no rotational symmetry
    rng = np.random.default_rng(2)
    pts, _ = meo.sample_surface(v, f, rng.random((3000, 3)))
    M = meo.rigid([0.1, 0.3, 1.0], np.deg2rad(2.0), [0.02, -0.01, 0.015])
    T, fit, rmse, it = meo.icp(pts, meo.transform(pts, M), 0.1, max_iteration=100, relative_fitness=1e-12,
                               relative_rmse=1e-12)
    assert fit == 1.0 and rmse < 1e-9 and it < 100
    assert np.abs(T - M).max() < 1e-8


def test_icp_without_correspondences_returns_init():
    init = meo.rigid([0, 0, 1], 0.1, [5.0, 0, 0])
    T, fit, rmse, it = meo.icp(np.zeros((3, 3)), np.ones((4, 3)) * 100, 0.1, init)
    assert np.array_equal(T, init) and fit == 0.0 and rmse == 0.0 and it == 1


def test_samples_lie_on_their_triangles():
    v, f = _sphere_mesh(10)
    rng = np.random.default_rng(3)
    s, face = meo.sample_surface(v, f, rng.random((5000, 3)))
    a, b, c = v[f[face, 0]], v[f[face, 1]], v[f[face, 2]]
    n = np.cross(b - a, c - a)
    assert np.abs(np.einsum("ij,ij->i", s - a, n)).max() < 1e-12
    # barycentric coordinates in [0, 1]
    e0, e1, p = b - a, c - a, s - a
    d00, d01, d11 = (e0 * e0).sum(1), (e0 * e1).sum(1), (e1 * e1).sum(1)
    d20, d21 = (p * e0).sum(1), (p * e1).sum(1)
    den = d00 * d11 - d01 * d01
    l1, l2 = (d11 * d20 - d01 * d21) / den, (d00 * d21 - d01 * d20) / den
    assert l1.min() > -1e-9 and l2.min() > -1e-9 and (l1 + l2).max() < 1 + 1e-9


def test_face_frequencies_follow_areas():
    v, f = _sphere_mesh(6)
    area = meo.face_areas(v, f)
    rng = np.random.default_rng(4)
    _, face = meo.sample_surface(v, f, rng.random((200000, 3)))
    counts = np.bincount(face, minlength=len(f))
    _, p = stats.chisquare(counts, area / area.sum() * len(face))
    assert p > 1e-3


def test_face_choice_is_searchsorted_left():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0.0]])
    f = np.array([[0, 1, 2], [0, 0, 1], [1, 3, 2]])                   # the middle face has zero area
    u = np.array([[0.0, 0.2, 0.2], [0.5, 0.2, 0.2], [0.9999, 0.9, 0.9]])
    s, face = meo.sample_surface(v, f, u)
    assert face.tolist() == [0, 0, 2]                                 # u * total == cum[0] picks face 0, never face 1
    assert np.allclose(s[2], [0.9, 0.2, 0.0], atol=1e-15)                # l0 + l1 > 1 folds both to 0.1


def test_golden_metrics_match_the_reference_message():
    g = np.load(os.path.join(ROOT, "tests", "golden", "mesh_eval.npz"))
    m = meo.metrics(g["s_est"], g["s_gt"], float(g["dist_th"]))
    got = np.array([m[k] for k in ("accuracy", "completion", "accuracy_ratio", "completion_ratio", "f_score")])
    assert np.array_equal(got, g["metrics"])
    msg = ('\n\nMetrics of reconstructed mesh are:\n\tAccuracy: {:.2f}cm\n\tCompletion: {:.2f}cm\n\tAccuracy Ratio: '
           '{:.2f}%\n\tCompletion Ratio: {:.2f}%\n\tF-score: {:.2f}%\n\n').format(*got)
    assert msg == str(g["message"])
    s, face = meo.sample_surface(g["est_verts"], g["est_faces"], g["u_est"])
    assert np.array_equal(s, g["s_est"]) and np.array_equal(face, g["f_est"])
