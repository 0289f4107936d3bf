"""The scene bound of Mesher.update_param_from_mapping restated in numpy / torch on the CPU (TEST INFRASTRUCTURE — never
imported by the product path).

Rules and where they come from:
- Hull vertices: `scipy.spatial.ConvexHull(points).vertices` (Qhull, as Open3D 0.13's `ComputeConvexHull` runs it),
  with each vertex replaced by the lowest index holding the same coordinates.  Qhull merges facets within its
  tolerance, so for general-position clouds this is the exact extreme-point set; `extreme_points_lp` is the
  independent definition (p is a vertex iff it is not in the convex hull of the other points) by linear programming.
- Mean and covariance: Open3D's `PointCloud::ComputeMeanAndCovariance`: cumulants (x, y, z, xx, xy, xz, yy, yz, zz)
  summed over the points and divided by n, then `E[ab] - E[a] E[b]`.
- Axes: Open3D's `OrientedBoundingBox::CreateFromPoints` orders the eigenvectors by descending eigenvalue (its three
  swaps).  Eigen's eigenvector signs are not reproducible here; the stated convention is: columns 0 and 1 have their
  largest-magnitude component positive (the first on ties), column 2 = column 0 x column 1, so R is a proper rotation.
- Box: the axis-aligned box of R^T (v - mean) over the hull vertices; center = R (min + max) / 2 + mean,
  extent = max - min, plus `extend` as in `src/oriented_bounding_box.py:compute_from_pointcloud`.
- Corners: `OrientedBoundingBox::GetBoxPoints`; in-bound: `GetPointIndicesWithinBoundingBox`'s six
  `det[b - a, c - a, x - a]` tests on those corners, in Eigen's 3x3 cofactor order; the min bound of
  `get_axis_aligned_bounding_box` is the corners' minimum.

Not checked against Open3D itself (it is not installed): Eigen's eigenvector signs, and whether 0.13 can return an
improper R (det = -1) for some inputs; the convention above never does.
"""
import numpy as np
import torch


# ---- hull ----------------------------------------------------------------------------------------------------------
def _lowest_equal(points, ids):
    """each id replaced by the lowest index whose point equals it"""
    _, first, inv = np.unique(points, axis=0, return_index=True, return_inverse=True)
    return np.unique(first[inv.reshape(-1)[ids]])


def hull_vertices(points):
    from scipy.spatial import ConvexHull
    points = np.asarray(points, np.float64)
    return _lowest_equal(points, ConvexHull(points).vertices)


def extreme_points_lp(points):
    """sorted ids of the exact extreme points: p (the lowest index of its duplicates) with p not in conv(others)"""
    from scipy.optimize import linprog
    points = np.asarray(points, np.float64)
    n = len(points)
    out = []
    for i in range(n):
        same = np.all(points == points[i], axis=1)
        if np.argmax(same) != i:
            continue
        others = points[~same]
        if len(others) == 0:
            out.append(i)
            continue
        A = np.vstack([others.T, np.ones(len(others))])
        b = np.append(points[i], 1.0)
        r = linprog(np.zeros(len(others)), A_eq=A, b_eq=b, bounds=(0, None), method="highs")
        if r.status != 0:          # infeasible: not a convex combination of the others
            out.append(i)
    return np.array(out, np.int64)


# ---- box -----------------------------------------------------------------------------------------------------------
def mean_and_covariance(points):
    p = np.asarray(points, np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    c = np.array([x.sum(), y.sum(), z.sum(), (x * x).sum(), (x * y).sum(), (x * z).sum(), (y * y).sum(),
                  (y * z).sum(), (z * z).sum()]) / len(p)
    cov = np.array([[c[3] - c[0] * c[0], c[4] - c[0] * c[1], c[5] - c[0] * c[2]],
                    [c[4] - c[0] * c[1], c[6] - c[1] * c[1], c[7] - c[1] * c[2]],
                    [c[5] - c[0] * c[2], c[7] - c[1] * c[2], c[8] - c[2] * c[2]]])
    return c[:3], cov


def axes(cov):
    """(R, eigenvalues descending) with the sign convention above"""
    w, V = np.linalg.eigh(cov)
    order = np.argsort(-w, kind="stable")
    w, V = w[order], V[:, order]
    R = np.zeros((3, 3))
    for j in range(2):
        col = V[:, j] / np.linalg.norm(V[:, j])
        if col[np.argmax(np.abs(col))] < 0:
            col = -col
        R[:, j] = col
    R[:, 2] = np.cross(R[:, 0], R[:, 1])
    return R, w


def oriented_box(points, extend=0.0):
    """(center, R, extent, eigenvalues) of CreateFromPoints(points), extent + extend"""
    hull = np.asarray(points, np.float64)[hull_vertices(points)]
    mean, cov = mean_and_covariance(hull)
    R, w = axes(cov)
    q = (hull - mean) @ R
    lo, hi = q.min(0), q.max(0)
    return R @ ((lo + hi) * 0.5) + mean, R, (hi - lo) + extend, w


def box_points(center, R, extent):
    c, R, e = np.asarray(center, np.float64), np.asarray(R, np.float64), np.asarray(extent, np.float64)
    x, y, z = R[:, 0] * (e[0] / 2), R[:, 1] * (e[1] / 2), R[:, 2] * (e[2] / 2)
    return np.array([c - x - y - z, c + x - y - z, c - x + y - z, c - x - y + z,
                     c + x + y + z, c - x + y + z, c + x - y + z, c + x + y - z])


def _det_cols(u, v, w):
    """Eigen's 3x3 determinant of the matrix with columns u, v, w (rows: x, y, z), vectorised over w"""
    return (u[0] * (v[1] * w[..., 2] - v[2] * w[..., 1]) - v[0] * (u[1] * w[..., 2] - u[2] * w[..., 1])
            + w[..., 0] * (u[1] * v[2] - u[2] * v[1]))


def in_box(points, center, R, extent):
    bp = box_points(center, R, extent)
    x = np.asarray(points, np.float64)

    def test(a, b, c):
        A = bp[a]
        return _det_cols(bp[b] - A, bp[c] - A, x - A)

    return ((test(0, 1, 3) <= 0) & (test(0, 5, 3) >= 0) & (test(2, 5, 7) <= 0) & (test(1, 4, 7) >= 0)
            & (test(3, 4, 5) <= 0) & (test(0, 1, 7) >= 0))


def axis_aligned_bound(center, R, extent):
    bp = box_points(center, R, extent)
    return np.stack([bp.min(0).astype(np.float32), bp.max(0).astype(np.float32)], 1)


# ---- the mesher's selection ----------------------------------------------------------------------------------------
def mapping_points(video, cur_idx, iproj, depth_filter, SE3, device):
    """src/mesher.py:256-276 with iproj / depth_filter / SE3 injected: the points handed to compute_from_pointcloud"""
    filter_thresh = 0.01
    filter_visible_num = 3
    dirty_index = torch.arange(0, cur_idx).long().to(device)
    poses = torch.index_select(video.poses.detach(), dim=0, index=dirty_index)
    disps = torch.index_select(video.disps_up.detach(), dim=0, index=dirty_index)
    common_intrinsic_id = 0
    intrinsic = video.intrinsics[common_intrinsic_id].detach() * video.scale_factor
    w2w = SE3(video.pose_compensate[0].clone().unsqueeze(dim=0)).to(device)
    points = iproj((w2w * SE3(poses).inv()).data, disps, intrinsic).cpu()
    thresh = filter_thresh * torch.ones_like(disps.mean(dim=[1, 2]))
    count = depth_filter(poses, disps, intrinsic, dirty_index, thresh)
    count = count.cpu()
    disps = disps.cpu()
    masks = (count >= filter_visible_num)
    masks = masks & (disps > 0.01 * disps.mean(dim=[1, 2], keepdim=True))
    return points.reshape(-1, 3)[masks.reshape(-1)]
