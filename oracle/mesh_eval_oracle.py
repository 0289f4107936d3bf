"""CPU restatement (numpy + scipy) of the reconstruction evaluation, align_mesh and eval_mesh (src/mesher.py:339-421).

Rules, and where they come from:

* Surface sampling (trimesh.sample.sample_surface, from given uniforms u, l0, l1 per sample).  Face weights are the fp64
  areas 0.5 |(v1 - v0) x (v2 - v0)| of mesh_view_oracle.face_areas (the component filter's formula; trimesh's own area
  formula is version-dependent and differs only in the last bits).  cum = np.cumsum(weights); the face is
  np.searchsorted(cum, u * cum[-1]) (side='left': the first face whose cumulative weight is >= u * total).  If
  l0 + l1 > 1 both become |l - 1|; the sample is ((v1 - v0) * l0 + (v2 - v0) * l1) + v0 per component.
* Nearest neighbours: scipy.spatial.cKDTree, whose squared distance for three coordinates is (dx^2 + dy^2) + dz^2, so
  the distance is sqrt of that, correctly rounded.
* Metrics (eval_mesh): completion = mean distance of the gt samples to the est samples * 100, accuracy the other way,
  the ratios np.mean((dist < dist_th).astype(np.float32)) * 100 (float32), F-score 2 a c / (a + c) in float32.
* ICP: Open3D's RegistrationICP (pipelines/registration/Registration.cpp) with TransformationEstimationPointToPoint
  (TransformationEstimation.cpp) and the default ICPConvergenceCriteria (max_iteration 30, relative_fitness and
  relative_rmse 1e-6):
    1. T = init; the working copy of the source is transformed by init as a general 4x4 (PointCloud::Transform):
       x' = ((m00 x + m01 y) + m02 z) + m03, likewise y', z', w'; the point is (x', y', z') / w'.
    2. Correspondences: each source point's nearest target with d2 < threshold^2 (KDTreeFlann::SearchHybrid with one
       neighbour: nanoflann's radius result set keeps dist < radius strictly).  fitness = matches / n_source,
       inlier_rmse = sqrt(sum d2 / matches); both 0 without matches.
    3. Per iteration: update = Eigen::umeyama(src, dst, with_scaling=false) over the correspondences (means as
       sum * (1 / n), sigma = (1 / n) dst_demean src_demean^T, SVD, S = diag(1, 1, det(U) det(V) < 0 ? -1 : 1),
       R = U S V^T, t = dst_mean - R src_mean); the identity without correspondences.  T <- update T, the working copy
       is transformed by update, correspondences are found again, and the loop stops when |d fitness| <
       relative_fitness and |d rmse| < relative_rmse.  `iterations` counts the updates made.
  Open3D is not a dependency; this restatement is what the device is pinned to.
"""
import numpy as np

F64 = np.float64


def face_areas(verts, faces):
    from oracle.mesh_view_oracle import face_areas as fa
    return fa(verts, faces)


def sample_surface(verts, faces, uniforms):
    """(samples [count,3] f64, face index [count]) for uniforms [count,3] (u, l0, l1)"""
    v = np.asarray(verts, F64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    u = np.asarray(uniforms, F64).reshape(-1, 3)
    cum = np.cumsum(face_areas(v, f))
    face = np.searchsorted(cum, u[:, 0] * cum[-1])
    lengths = u[:, 1:3].copy()
    fold = (lengths[:, 0] + lengths[:, 1]) > 1.0
    lengths[fold] -= 1.0
    lengths = np.abs(lengths)
    v0, v1, v2 = v[f[face, 0]], v[f[face, 1]], v[f[face, 2]]
    return ((v1 - v0) * lengths[:, 0:1] + (v2 - v0) * lengths[:, 1:2]) + v0, face


def sq_dist(a, b):
    d = np.asarray(a, F64) - np.asarray(b, F64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def nearest(query, points, max_dist=np.inf):
    """(dist, idx) of the nearest point (cKDTree), -1 / inf where none has d2 < max_dist^2"""
    from scipy.spatial import cKDTree
    dist, idx = cKDTree(np.asarray(points, F64)).query(np.asarray(query, F64))
    idx = np.asarray(idx, np.int64)
    if np.isfinite(max_dist):
        far = ~(sq_dist(query, np.asarray(points, F64)[idx]) < max_dist * max_dist)
        dist, idx = dist.copy(), idx.copy()
        dist[far], idx[far] = np.inf, -1
    return dist, idx


def ratio(count, n):
    return np.float32(np.float32(count) / np.float32(n)) * np.float32(100)


def metrics(est_pts, gt_pts, dist_th):
    comp, _ = nearest(gt_pts, est_pts)
    acc, _ = nearest(est_pts, gt_pts)
    completion, accuracy = np.mean(comp) * 100, np.mean(acc) * 100
    cr = np.mean((comp < dist_th).astype(np.float32)) * 100
    ar = np.mean((acc < dist_th).astype(np.float32)) * 100
    return dict(accuracy=accuracy, completion=completion, accuracy_ratio=ar, completion_ratio=cr,
                f_score=(2.0 * ar * cr) / (ar + cr))


def transform(points, M):
    """PointCloud::Transform with a general 4x4: (((m_a0 x + m_a1 y) + m_a2 z) + m_a3) / w'"""
    p = np.asarray(points, F64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r = [((M[a, 0] * x + M[a, 1] * y) + M[a, 2] * z) + M[a, 3] for a in range(4)]
    return np.stack([r[0] / r[3], r[1] / r[3], r[2] / r[3]], 1)


def umeyama(src, dst):
    """Eigen::umeyama(src^T, dst^T, with_scaling=false) for src, dst [n,3]: the 4x4 rigid transform"""
    src, dst = np.asarray(src, F64), np.asarray(dst, F64)
    inv = 1.0 / len(src)
    ms, md = src.sum(0) * inv, dst.sum(0) * inv
    sigma = inv * ((dst - md).T @ (src - ms))
    U, _, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = U @ np.diag(S) @ Vt
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = md - R @ ms
    return T


def correspondences(pts, tree, target, threshold):
    dist, idx = tree.query(pts)
    idx = np.asarray(idx, np.int64)
    d2 = sq_dist(pts, target[idx])
    ok = d2 < threshold * threshold
    n = int(ok.sum())
    fitness = n / len(pts)
    rmse = float(np.sqrt(d2[ok].sum() / n)) if n else 0.0
    return np.nonzero(ok)[0], idx[ok], (fitness if n else 0.0), rmse


def icp(src, dst, threshold, init=None, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6):
    """(T [4,4], fitness, inlier_rmse, iterations) of point-to-point ICP, the rules in the module docstring"""
    from scipy.spatial import cKDTree
    src, dst = np.asarray(src, F64), np.asarray(dst, F64)
    T = np.eye(4) if init is None else np.asarray(init, F64).copy()
    tree = cKDTree(dst)
    pts = transform(src, T)
    si, di, fit, rmse = correspondences(pts, tree, dst, threshold)
    it = 0
    for i in range(max_iteration):
        upd = umeyama(pts[si], dst[di]) if len(si) else np.eye(4)
        T = upd @ T
        pts = transform(pts, upd)
        prev = (fit, rmse)
        si, di, fit, rmse = correspondences(pts, tree, dst, threshold)
        it = i + 1
        if abs(prev[0] - fit) < relative_fitness and abs(prev[1] - rmse) < relative_rmse:
            break
    return T, fit, rmse, it


def rigid(axis, angle, t, scale=1.0):
    """4x4 [s R | t] with R the rotation by `angle` about `axis`"""
    a = np.asarray(axis, F64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K
    M = np.eye(4)
    M[:3, :3] = scale * R
    M[:3, 3] = t
    return M
