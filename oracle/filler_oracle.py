"""CPU oracle (TEST INFRASTRUCTURE — never imported by the product path) for PoseTrajectoryFiller's bracketing and
linear SE3 interpolation (src/trajectory_filler.py:45-55), restated in float64:

    t0 = #{ts[0:N] <= t} - 1,  t1 = t0 < N-1 ? t0+1 : t0
    dt = ts[t1] - ts[t0] + 1e-3,  dP = P[t1] * P[t0]^-1,  v = log(dP) / dt,  w = v * (t - ts[t0]),  G = exp(w) * P[t0]

The bracket compares in float32 (the video's timestamps are float32 and the reference compares them with the frame's
timestamp in that type); everything after it is float64.  exp / log are lietorch's closed forms (go-slam_b200/lietorch.py)
with their small-angle switches.  Layout [..., 7] = (tx, ty, tz, qx, qy, qz, qw).
"""
import numpy as np

D = np.float64


def qmul(a, b):
    ax, ay, az, aw = np.moveaxis(a, -1, 0)
    bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx,
                     aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def qrot(q, X):
    qv, qw = q[..., :3], q[..., 3:]
    uv = 2.0 * np.cross(qv, X)
    return X + qw * uv + np.cross(qv, uv)


def inv(P):
    qi = np.concatenate([-P[..., 3:6], P[..., 6:]], axis=-1)
    return np.concatenate([-qrot(qi, P[..., :3]), qi], axis=-1)


def mul(A, B):
    return np.concatenate([A[..., :3] + qrot(A[..., 3:], B[..., :3]), qmul(A[..., 3:], B[..., 3:])], axis=-1)


def exp(xi):
    tau, phi = xi[..., :3], xi[..., 3:]
    th2 = (phi * phi).sum(-1, keepdims=True)
    th = np.sqrt(th2)
    small = th2 < 1e-8
    ths = np.where(small, 1.0, th)
    imag = np.where(small, 0.5 - th2 / 48.0 + th2 * th2 / 3840.0, np.sin(0.5 * ths) / ths)
    real = np.where(small, 1.0 - th2 / 8.0 + th2 * th2 / 384.0, np.cos(0.5 * ths))
    big = th > 1e-4
    th2s, thb = np.where(big, th2, 1.0), np.where(big, th, 1.0)
    a = np.where(big, (1.0 - np.cos(thb)) / th2s, 0.0)
    b = np.where(big, (thb - np.sin(thb)) / (thb * th2s), 0.0)
    c1 = np.cross(phi, tau)
    c2 = np.cross(phi, c1)
    return np.concatenate([tau + a * c1 + b * c2, imag * phi, real], axis=-1)


def log(P):
    t, qv, qw = P[..., :3], P[..., 3:6], P[..., 6:]
    n2 = (qv * qv).sum(-1, keepdims=True)
    n = np.sqrt(n2)
    small = n2 < 1e-12
    ns = np.where(small, 1.0, n)
    sgn = np.where(qw < 0, -1.0, 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        two_atan = np.where(small, 2.0 / qw - (2.0 / 3.0) * n2 / (qw * qw * qw), 2.0 * sgn * np.arctan2(ns, qw * sgn) / ns)
    phi = two_atan * qv
    th = np.sqrt((phi * phi).sum(-1, keepdims=True))
    big = th > 1e-4
    thb = np.where(big, th, 1.0)
    coef = (1.0 - thb * np.cos(0.5 * thb) / (2.0 * np.sin(0.5 * thb))) / (thb * thb)
    c1 = np.cross(phi, t)
    c2 = np.cross(phi, c1)
    return np.concatenate([np.where(big, t - 0.5 * c1 + coef * c2, t), phi], axis=-1)


def bracket(ts, tt):
    """ts [N] keyframe timestamps, tt [M] frame timestamps -> t0, t1 [M] int64 (t0 = -1 before the first keyframe)"""
    ts, tt = np.asarray(ts, np.float32), np.asarray(tt, np.float32)
    t0 = (ts[None, :] <= tt[:, None]).sum(1).astype(np.int64) - 1
    t1 = np.where(t0 < ts.size - 1, t0 + 1, t0)
    return t0, t1


def bound(ts, poses, tt, base):
    """per-frame tolerance of a float32 interpolation against this oracle: `base`, plus, after the last keyframe
    (t0 == t1, dt = 1e-3), two float32 ulps of the keyframe's largest pose component (at least 1) amplified by
    (t - ts[t0]) / dt.  There dP = P * P^-1 is the identity up to the rounding of that composition, and
    v = log(dP) / dt scales the rounding by 1000 per frame of distance (the reference's own float32 result carries it
    too)."""
    t0, t1 = bracket(ts, tt)
    ts64 = np.asarray(ts, np.float32).astype(D)
    amp = (np.asarray(tt, np.float32).astype(D) - ts64[t0]) / 1e-3
    mag = 1.0 + np.abs(np.asarray(poses, np.float32).astype(D)[t0]).max(-1)
    return base + np.where(t0 == t1, 2.0 * amp * mag * 2.0 ** -23, 0.0)


def interpolate(ts, poses, tt):
    """ts [N], poses [N, 7] (the video's rows 0..N-1), tt [M] -> (t0, t1, G [M, 7] float64)"""
    t0, t1 = bracket(ts, tt)
    ts64 = np.asarray(ts, np.float32).astype(D)
    P = np.asarray(poses, np.float32).astype(D)
    dt = ts64[t1] - ts64[t0] + 1e-3
    dP = mul(P[t1], inv(P[t0]))
    v = log(dP) / dt[:, None]
    w = v * (np.asarray(tt, np.float32).astype(D) - ts64[t0])[:, None]
    return t0, t1, mul(exp(w), P[t0])
