"""CPU restatement (numpy f64) of the trajectory evaluation of SLAM.terminate (src/slam.py:289-370): evo's APE w.r.t.
the translation part with a Sim(3) Umeyama alignment, main_ape.ape(traj_ref, traj_est,
pose_relation=PoseRelation.translation_part, align=True, correct_scale=True).

evo is not a dependency of this project and cannot be run here, so these rules, restated from its source, are the
contract the device is pinned to:

* Row selection (src/slam.py:341-347): row i is kept iff stream.poses[i].sum() is neither NaN nor Inf; the estimate of
  a kept row is traj_est[i].  Kept rows stay in input order.  The sum is numpy's pairwise sum of the 16 entries.
* Umeyama with scale (evo core/geometry.py umeyama_alignment(x = est^T, y = ref^T, with_scale=True)): mean_x, mean_y
  = x.mean(axis=1) (sum / n); sigma_x = 1 / n * |x - mean_x|_F^2; cov_xy = 1 / n * sum_i (y_i - mean_y)(x_i - mean_x)^T;
  u, d, v = svd(cov_xy); fewer than 2 of d > np.finfo(float64).eps raises "Degenerate covariance rank, Umeyama
  alignment is not possible"; s = diag(1, 1, -1 if det(u) det(v) < 0 else 1); r = u s v; c = 1 / sigma_x *
  trace(diag(d) s); t = mean_y - c * (r mean_x).  Fewer than three kept rows are degenerate outright: their centred
  positions span at most a line, so the covariance has rank <= 1 and only rounding could lift a second singular value
  over eps.
* Alignment (evo core/trajectory.py PosePath3D.align, then scale(c) and transform(se3(r, t))): the positions become
  r (c x_i) + t; sim3 = [[c r, t], [0, 1]] (evo core/lie_algebra.py sim3), np_arrays['alignment_transformation_sim3'].
* Errors (evo core/metrics.py APE.process_data, translation_part): e_i = |p_est_i - p_ref_i|.
* Statistics (evo core/metrics.py PE.get_all_statistics): rmse = sqrt(mean(e^2)), mean, median (np.median: the mean
  of the two middle values for even n), std (np.std, population), min, max, sse = sum(e^2).
* Text (evo core/result.py Result.pretty_str; the title from evo main_ape.ape): the title, a blank line, then each
  statistic in sorted name order as "{:>10}\t{:.6f}\n".  Stated from evo's source as remembered.
"""
import numpy as np

F64 = np.float64
EPS = float(np.finfo(np.float64).eps)
TITLE = "APE w.r.t. translation part (m)\n(with Sim(3) Umeyama alignment)"
DEGENERATE = "Degenerate covariance rank, Umeyama alignment is not possible"
NO_ROWS = "APE: no reference pose has finite entries"
NONFINITE = "APE: an estimated position of a kept row is not finite"
STATS = ("rmse", "mean", "median", "std", "min", "max", "sse")


def keep_rows(ref):
    """[n] bool: the reference c2w [n,4,4] rows whose entry sum is finite"""
    ref = np.asarray(ref, F64)
    return np.isfinite(ref.reshape(len(ref), 16).sum(1))


def umeyama(x, y):
    """(r [3,3], t [3], c, d [3]) of evo's umeyama_alignment(x^T, y^T, with_scale=True) for x, y [n,3]"""
    x, y = np.asarray(x, F64), np.asarray(y, F64)
    n = len(x)
    mx, my = x.sum(0) / n, y.sum(0) / n
    xc, yc = x - mx, y - my
    sigma_x = 1.0 / n * float((xc * xc).sum())
    cov = 1.0 / n * (yc.T @ xc)
    u, d, v = np.linalg.svd(cov)
    if n < 3 or np.count_nonzero(d > EPS) < 2:
        raise ValueError(DEGENERATE)
    s = np.eye(3)
    if np.linalg.det(u) * np.linalg.det(v) < 0.0:
        s[2, 2] = -1.0
    r = u @ s @ v
    c = 1.0 / sigma_x * np.trace(np.diag(d) @ s)
    t = my - c * (r @ mx)
    return r, t, c, d


def sim3(r, t, c):
    m = np.eye(4)
    m[:3, :3] = c * r
    m[:3, 3] = t
    return m


def errors(x, y, r, t, c):
    """|(r (c x_i) + t) - y_i| for x, y [n,3]"""
    p = c * np.asarray(x, F64)
    d = (p @ r.T + t) - np.asarray(y, F64)
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def statistics(e):
    e = np.asarray(e, F64)
    return {"rmse": float(np.sqrt(np.mean(np.power(e, 2)))), "mean": float(np.mean(e)),
            "median": float(np.median(e)), "std": float(np.std(e)), "min": float(np.min(e)),
            "max": float(np.max(e)), "sse": float(np.sum(np.power(e, 2)))}


def pretty_str(stats, title=TITLE):
    text = "{}\n\n".format(title)
    for name, val in sorted(stats.items()):
        text += "{:>10}\t{:.6f}\n".format(name, val)
    return text


def ape(ref_poses, est_positions):
    """dict(kept [n] bool, r, t, c, d, sim3 [4,4], errors [m], stats) for reference c2w [n,4,4] and estimates [n,3];
    ValueError as the device raises it"""
    ref = np.asarray(ref_poses, F64)
    est = np.asarray(est_positions, F64)
    kept = keep_rows(ref)
    if not kept.any():
        raise ValueError(NO_ROWS)
    x, y = est[kept], ref[kept][:, :3, 3]
    if not np.isfinite(x).all():
        raise ValueError(NONFINITE)
    r, t, c, d = umeyama(x, y)
    e = errors(x, y, r, t, c)
    return dict(kept=kept, r=r, t=t, c=c, d=d, sim3=sim3(r, t, c), errors=e, stats=statistics(e))


def random_rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, a, b, cc = q
    return np.array([[1 - 2 * (b * b + cc * cc), 2 * (a * b - cc * w), 2 * (a * cc + b * w)],
                     [2 * (a * b + cc * w), 1 - 2 * (a * a + cc * cc), 2 * (b * cc - a * w)],
                     [2 * (a * cc - b * w), 2 * (b * cc + a * w), 1 - 2 * (a * a + b * b)]])


def smooth_trajectory(n, rng, offset=(0.0, 0.0, 0.0), spread=1.0):
    """[n,3] positions along a smooth 3-D curve of size ~spread around offset"""
    s = np.linspace(0.0, 4.0 * np.pi, n)
    ph = rng.uniform(0, 2 * np.pi, size=3)
    p = np.stack([np.cos(s + ph[0]), np.sin(0.7 * s + ph[1]), 0.5 * np.sin(0.3 * s + ph[2])], 1)
    return spread * p + np.asarray(offset, F64)


def poses_from(positions, rng):
    """[n,4,4] c2w with the given translations and random rotations"""
    n = len(positions)
    P = np.tile(np.eye(4), (n, 1, 1))
    for i in range(n):
        P[i, :3, :3] = random_rotation(rng)
    P[:, :3, 3] = positions
    return P
