"""CPU oracle (TEST INFRASTRUCTURE — never imported by the product path) for the SE3 helpers and
the per-pixel geometry kernels of droid_backends.

Each function restates the reference CUDA line by line in numpy float32:
  se3 helpers      src/lib/droid_kernels.cu:58-175 (actSO3/actSE3/adjSE3/relSE3/expSO3/expSE3),
                   :877-895 (retrSE3)
  frame_distance   src/lib/droid_kernels.cu:518-657 (incl. the 256-thread strided partial sums
                   and the 128/64/32/.../1 tree of :36-55)
  projmap          src/lib/droid_kernels.cu:427-516
  iproj            src/lib/droid_kernels.cu:779-850
  depth_filter     src/lib/droid_kernels.cu:661-775
  reproject        src/geom/projective_ops.py:26-144 as called by src/depth_video.py:207-217
Parity pin: cross-checked in tests against (i) the reference's own Python
(src/geom/projective_ops.py imported with this algebra standing in for the absent lietorch)
and (ii) on the GPU box, the reference's own CUDA kernels compiled into oracle/_ref.
"""
import numpy as np

F = np.float32
MIN_DEPTH = F(0.25)


def _f(x):
    return np.asarray(x, dtype=F)


def fma(a, b, c):
    """round32(a*b + c) — the contraction nvcc applies to `c += a*b` (a*b exact in float64)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F)


# ----------------------------------------------------------------------------- SE3
def act_so3(q, X):
    q0, q1, q2, q3 = [q[..., i] for i in range(4)]
    X0, X1, X2 = [X[..., i] for i in range(3)]
    u0 = F(2.0) * (q1 * X2 - q2 * X1)
    u1 = F(2.0) * (q2 * X0 - q0 * X2)
    u2 = F(2.0) * (q0 * X1 - q1 * X0)
    Y0 = X0 + q3 * u0 + (q1 * u2 - q2 * u1)
    Y1 = X1 + q3 * u1 + (q2 * u0 - q0 * u2)
    Y2 = X2 + q3 * u2 + (q0 * u1 - q1 * u0)
    return np.stack([Y0, Y1, Y2], axis=-1).astype(F)


def act_se3(t, q, X):
    Y = act_so3(q, X[..., :3])
    Y = Y + X[..., 3:4] * t
    return np.concatenate([Y, X[..., 3:4]], axis=-1).astype(F)


def adj_se3(t, q, X):
    """Y = Ad^T X on 6-covectors (adjSE3)."""
    qinv = np.concatenate([-q[..., :3], q[..., 3:]], axis=-1)
    a, b = X[..., :3], X[..., 3:]
    Ya = act_so3(qinv, a)
    Yb = act_so3(qinv, b)
    u = np.stack([t[..., 2] * a[..., 1] - t[..., 1] * a[..., 2],
                  t[..., 0] * a[..., 2] - t[..., 2] * a[..., 0],
                  t[..., 1] * a[..., 0] - t[..., 0] * a[..., 1]], axis=-1).astype(F)
    Yb = Yb + act_so3(qinv, u)
    return np.concatenate([Ya, Yb], axis=-1).astype(F)


def rel_se3(ti, qi, tj, qj):
    q = np.stack([
        -qj[..., 3] * qi[..., 0] + qj[..., 0] * qi[..., 3] - qj[..., 1] * qi[..., 2] + qj[..., 2] * qi[..., 1],
        -qj[..., 3] * qi[..., 1] + qj[..., 1] * qi[..., 3] - qj[..., 2] * qi[..., 0] + qj[..., 0] * qi[..., 2],
        -qj[..., 3] * qi[..., 2] + qj[..., 2] * qi[..., 3] - qj[..., 0] * qi[..., 1] + qj[..., 1] * qi[..., 0],
        qj[..., 3] * qi[..., 3] + qj[..., 0] * qi[..., 0] + qj[..., 1] * qi[..., 1] + qj[..., 2] * qi[..., 2],
    ], axis=-1).astype(F)
    t = (tj - act_so3(q, ti)).astype(F)
    return t, q


def edge_pose(poses, ii, jj, stereo_special=True):
    """relative pose per edge; ii == jj -> fixed stereo baseline (droid_kernels.cu:218-229)."""
    poses = _f(poses)
    ti, qi = poses[ii, :3], poses[ii, 3:]
    tj, qj = poses[jj, :3], poses[jj, 3:]
    t, q = rel_se3(ti, qi, tj, qj)
    if stereo_special:
        s = np.asarray(ii) == np.asarray(jj)
        t[s] = _f([-0.1, 0, 0])
        q[s] = _f([0, 0, 0, 1])
    return t, q


def exp_so3(phi):
    th2 = (phi * phi).sum(-1)
    th4 = th2 * th2
    th = np.sqrt(th2)
    small = th2 < F(1e-8)
    ths = np.where(small, F(1), th)
    imag = np.where(small, F(0.5) - F(1.0 / 48.0) * th2 + F(1.0 / 3840.0) * th4, np.sin(F(0.5) * ths) / ths)
    real = np.where(small, F(1.0) - F(1.0 / 8.0) * th2 + F(1.0 / 384.0) * th4, np.cos(F(0.5) * ths))
    return np.concatenate([imag[..., None] * phi, real[..., None]], axis=-1).astype(F)


def exp_se3(xi):
    xi = _f(xi)
    tau, phi = xi[..., :3], xi[..., 3:]
    q = exp_so3(phi)
    th2 = (phi * phi).sum(-1)
    th = np.sqrt(th2)
    big = th > F(1e-4)
    th2s = np.where(big, th2, F(1))
    ths = np.where(big, th, F(1))
    a = np.where(big, (F(1) - np.cos(ths)) / th2s, F(0))[..., None]
    b = np.where(big, (ths - np.sin(ths)) / (ths * th2s), F(0))[..., None]
    c1 = np.cross(phi, tau).astype(F)
    c2 = np.cross(phi, c1).astype(F)
    t = tau + a * c1 + b * c2
    return t.astype(F), q


def retr_se3(xi, t, q):
    dt, dq = exp_se3(xi)
    q1 = np.stack([
        dq[..., 3] * q[..., 0] + dq[..., 0] * q[..., 3] + dq[..., 1] * q[..., 2] - dq[..., 2] * q[..., 1],
        dq[..., 3] * q[..., 1] + dq[..., 1] * q[..., 3] + dq[..., 2] * q[..., 0] - dq[..., 0] * q[..., 2],
        dq[..., 3] * q[..., 2] + dq[..., 2] * q[..., 3] + dq[..., 0] * q[..., 1] - dq[..., 1] * q[..., 0],
        dq[..., 3] * q[..., 3] - dq[..., 0] * q[..., 0] - dq[..., 1] * q[..., 1] - dq[..., 2] * q[..., 2],
    ], axis=-1)
    t1 = act_so3(dq, t) + dt
    return t1.astype(F), q1.astype(F)


def pixel_grid(ht, wd):
    v, u = np.meshgrid(np.arange(ht, dtype=F), np.arange(wd, dtype=F), indexing="ij")
    return u.reshape(-1), v.reshape(-1)


def backproject(disp_flat, intr, ht, wd):
    """Xi = ((u-cx)/fx, (v-cy)/fy, 1, d) for every pixel; disp_flat [..., hw]."""
    fx, fy, cx, cy = [F(x) for x in intr]
    u, v = pixel_grid(ht, wd)
    X = (u - cx) / fx
    Y = (v - cy) / fy
    shp = disp_flat.shape
    X = np.broadcast_to(X, shp)
    Y = np.broadcast_to(Y, shp)
    return np.stack([X, Y, np.ones(shp, F), disp_flat.astype(F)], axis=-1).astype(F)


# ----------------------------------------------------------------------------- frame distance
def _tree256(part):
    """part [..., 256] -> the reference's blockReduce tree (128, 64, then warpReduce)."""
    s = part.astype(F).copy()
    s[..., :128] = s[..., :128] + s[..., 128:256]
    s[..., :64] = s[..., :64] + s[..., 64:128]
    r = s[..., :32] + s[..., 32:64]
    for off in (16, 8, 4, 2, 1):
        r = r.copy()
        r[..., :off] = r[..., :off] + r[..., off:2 * off]
    return r[..., 0]


def frame_distance(poses, disps, intrinsics, ii, jj, beta):
    poses, disps = _f(poses), _f(disps)
    ii, jj = np.asarray(ii, np.int64), np.asarray(jj, np.int64)
    K = ii.shape[0]
    num, ht, wd = disps.shape
    hw = ht * wd
    fx, fy, cx, cy = [F(x) for x in np.asarray(intrinsics, F)]
    beta = F(beta)
    omb = F(F(1) - beta)
    t, q = edge_pose(poses, ii, jj, stereo_special=False)          # [K,3], [K,4]
    Xi = backproject(disps[ii].reshape(K, hw), (fx, fy, cx, cy), ht, wd)   # [K,hw,4]
    u, v = pixel_grid(ht, wd)
    Xj = act_se3(t[:, None, :], q[:, None, :], Xi)
    du = fx * (Xj[..., 0] / Xj[..., 2]) + cx - u
    dv = fy * (Xj[..., 1] / Xj[..., 2]) + cy - v
    d1 = np.sqrt(du * du + dv * dv).astype(F)
    ok1 = Xj[..., 2] > MIN_DEPTH
    X2 = Xi[..., :3] + Xi[..., 3:4] * t[:, None, :]
    du = fx * (X2[..., 0] / X2[..., 2]) + cx - u
    dv = fy * (X2[..., 1] / X2[..., 2]) + cy - v
    d2 = np.sqrt(du * du + dv * dv).astype(F)
    ok2 = X2[..., 2] > MIN_DEPTH

    nrow = (hw + 255) // 256
    pad = nrow * 256 - hw

    def rows(a, fill):
        return np.concatenate([a, np.full((K, pad), fill, a.dtype)], axis=1).reshape(K, nrow, 256)

    d1r, d2r = rows(d1, F(0)), rows(d2, F(0))
    ok1r, ok2r = rows(ok1, False), rows(ok2, False)
    live = rows(np.ones((K, hw), bool), False)
    accum = np.zeros((K, 256), F)
    valid = np.zeros((K, 256), F)
    total = np.zeros((K, 256), F)
    for r in range(nrow):
        lv = live[:, r]
        total = np.where(lv, total + beta, total)
        m = lv & ok1r[:, r]
        accum = np.where(m, fma(beta, d1r[:, r], accum), accum)
        valid = np.where(m, valid + beta, valid)
        total = np.where(lv, total + omb, total)
        m = lv & ok2r[:, r]
        accum = np.where(m, fma(omb, d2r[:, r], accum), accum)
        valid = np.where(m, valid + omb, valid)
    a, tt, w = _tree256(accum), _tree256(total), _tree256(valid)
    with np.errstate(divide="ignore", invalid="ignore"):
        out = np.where(w / (tt + F(1e-8)) < F(0.75), F(1000.0), a / w)
    return out.astype(F)


# ----------------------------------------------------------------------------- projmap / iproj
def projmap(poses, disps, intrinsics, ii, jj):
    poses, disps = _f(poses), _f(disps)
    ii, jj = np.asarray(ii, np.int64), np.asarray(jj, np.int64)
    K = ii.shape[0]
    num, ht, wd = disps.shape
    hw = ht * wd
    fx, fy, cx, cy = [F(x) for x in np.asarray(intrinsics, F)]
    t, q = edge_pose(poses, ii, jj, stereo_special=False)
    Xi = backproject(disps[ii].reshape(K, hw), (fx, fy, cx, cy), ht, wd)
    Xj = act_se3(t[:, None, :], q[:, None, :], Xi)
    u, v = pixel_grid(ht, wd)
    good = Xj[..., 2] > F(0.01)
    with np.errstate(divide="ignore", invalid="ignore"):
        cu = np.where(good, fx * (Xj[..., 0] / Xj[..., 2]) + cx, u)
        cv = np.where(good, fy * (Xj[..., 1] / Xj[..., 2]) + cy, v)
    coords = np.stack([cu, cv, np.zeros_like(cu)], axis=-1).reshape(K, ht, wd, 3).astype(F)
    valid = (Xj[..., 2] > MIN_DEPTH).astype(F).reshape(K, ht, wd, 1)
    return coords, valid


def iproj(poses, disps, intrinsics):
    poses, disps = _f(poses), _f(disps)
    num, ht, wd = disps.shape
    hw = ht * wd
    Xi = backproject(disps.reshape(num, hw), np.asarray(intrinsics, F), ht, wd)
    Xj = act_se3(poses[:, None, :3], poses[:, None, 3:], Xi)
    with np.errstate(divide="ignore", invalid="ignore"):
        pts = Xj[..., :3] / Xj[..., 3:4]
    return pts.reshape(num, ht, wd, 3).astype(F)


def depth_filter(poses, disps, intrinsics, ix, thresh):
    poses, disps = _f(poses), _f(disps)
    ix = np.asarray(ix, np.int64)
    thresh = _f(thresh)
    num, ht, wd = disps.shape
    hw = ht * wd
    fx, fy, cx, cy = [F(x) for x in np.asarray(intrinsics, F)]
    out = np.zeros((len(ix), ht, wd), F)
    for b, i in enumerate(ix):
        Xi = backproject(disps[i].reshape(1, hw), (fx, fy, cx, cy), ht, wd)[0]
        cnt = np.zeros(hw, F)
        for nb in range(6):
            j = i - nb - 1 if nb < 3 else i + nb
            if j < 0 or j >= num:
                continue
            t, q = edge_pose(poses, np.array([i]), np.array([j]), stereo_special=False)
            Xj = act_se3(t, q, Xi)
            with np.errstate(divide="ignore", invalid="ignore"):
                uj = fx * (Xj[:, 0] / Xj[:, 2]) + cx
                vj = fy * (Xj[:, 1] / Xj[:, 2]) + cy
                dj = Xj[:, 3] / Xj[:, 2]
            with np.errstate(invalid="ignore"):
                u0 = np.floor(uj)
                v0 = np.floor(vj)
            inb = (u0 >= 0) & (v0 >= 0) & (u0 < wd - 1) & (v0 < ht - 1) & np.isfinite(u0) & np.isfinite(v0)
            u0i = np.where(inb, u0, 0).astype(np.int64)
            v0i = np.where(inb, v0, 0).astype(np.int64)
            dm = disps[j]
            d00, d01 = dm[v0i, u0i], dm[v0i, np.minimum(u0i + 1, wd - 1)]
            d10, d11 = dm[np.minimum(v0i + 1, ht - 1), u0i], dm[np.minimum(v0i + 1, ht - 1), np.minimum(u0i + 1, wd - 1)]
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / dj.astype(np.float64)
                hit = np.zeros(hw, bool)
                for dn in (d00, d01, d10, d11):
                    hit |= np.abs(inv - 1.0 / dn.astype(np.float64)) < np.float64(thresh[b])
            cnt += (inb & hit).astype(F)
        out[b] = cnt.reshape(ht, wd)
    return out


# ----------------------------------------------------------------------------- reproject
def reproject(poses, disps, intrinsics_all, ii, jj, dtype=F, return_z=False):
    """pops.projective_transform(jacobian=False): Python-side constants (MIN_DEPTH 0.2).

    dtype=np.float64 evaluates the same formula in float64 from the float32 inputs (relative pose, back-projection,
    action, projection), keeping the float32 thresholds the reference compares against (0.5 * 0.2 and 0.2, both
    rounded to float32 as torch rounds a Python scalar against a float32 tensor).  return_z adds X1z [N, ht, wd];
    with dtype=np.float64, return_z="points" returns X1 [N, ht, wd, 3] alone."""
    poses, disps, Kall = _f(poses), _f(disps), _f(intrinsics_all)
    ii, jj = np.asarray(ii, np.int64), np.asarray(jj, np.int64)
    N = ii.shape[0]
    num, ht, wd = disps.shape
    hw = ht * wd
    u, v = pixel_grid(ht, wd)
    if dtype == np.float64:
        return _reproject64(poses, disps, Kall, ii, jj, u, v, return_z)
    Ki, Kj = Kall[ii], Kall[jj]
    X0 = np.stack([(u[None] - Ki[:, 2:3]) / Ki[:, 0:1], (v[None] - Ki[:, 3:4]) / Ki[:, 1:2],
                   np.ones((N, hw), F), disps[ii].reshape(N, hw)], axis=-1).astype(F)
    t, q = edge_pose(poses, ii, jj, stereo_special=True)
    X1 = act_se3(t[:, None, :], q[:, None, :], X0)
    Z = np.where(X1[..., 2] < F(0.5) * F(0.2), F(1.0), X1[..., 2])
    x = Kj[:, 0:1] * (X1[..., 0] / Z) + Kj[:, 2:3]
    y = Kj[:, 1:2] * (X1[..., 1] / Z) + Kj[:, 3:4]
    coords = np.stack([x, y], axis=-1).reshape(1, N, ht, wd, 2).astype(F)
    valid = ((X1[..., 2] > F(0.2)) & (X0[..., 2] > F(0.2))).astype(F).reshape(1, N, ht, wd, 1)
    if return_z:
        return coords, valid, X1[..., 2].reshape(N, ht, wd)
    return coords, valid


def _rot64(q, X):
    """R(q) X in float64 (the act_so3 formula; q need not be exactly unit, as the stored quaternions are not)."""
    q0, q1, q2, q3 = [q[..., i] for i in range(4)]
    X0, X1, X2 = [X[..., i] for i in range(3)]
    u0 = 2.0 * (q1 * X2 - q2 * X1)
    u1 = 2.0 * (q2 * X0 - q0 * X2)
    u2 = 2.0 * (q0 * X1 - q1 * X0)
    return np.stack([X0 + q3 * u0 + (q1 * u2 - q2 * u1),
                     X1 + q3 * u1 + (q2 * u0 - q0 * u2),
                     X2 + q3 * u2 + (q0 * u1 - q1 * u0)], axis=-1)


def edge_pose64(poses, ii, jj):
    """edge_pose(stereo_special=True) in float64 from float32 poses."""
    P = np.asarray(poses, F).astype(np.float64)
    ti, qi, tj, qj = P[ii, :3], P[ii, 3:], P[jj, :3], P[jj, 3:]
    q = np.stack([
        -qj[..., 3] * qi[..., 0] + qj[..., 0] * qi[..., 3] - qj[..., 1] * qi[..., 2] + qj[..., 2] * qi[..., 1],
        -qj[..., 3] * qi[..., 1] + qj[..., 1] * qi[..., 3] - qj[..., 2] * qi[..., 0] + qj[..., 0] * qi[..., 2],
        -qj[..., 3] * qi[..., 2] + qj[..., 2] * qi[..., 3] - qj[..., 0] * qi[..., 1] + qj[..., 1] * qi[..., 0],
        qj[..., 3] * qi[..., 3] + qj[..., 0] * qi[..., 0] + qj[..., 1] * qi[..., 1] + qj[..., 2] * qi[..., 2],
    ], axis=-1)
    t = tj - _rot64(q, ti)
    s = np.asarray(ii) == np.asarray(jj)
    t[s] = [-0.1, 0.0, 0.0]
    q[s] = [0.0, 0.0, 0.0, 1.0]
    return t, q


def _reproject64(poses, disps, Kall, ii, jj, u, v, return_z):
    N = ii.shape[0]
    num, ht, wd = disps.shape
    K64 = Kall.astype(np.float64)
    Ki, Kj = K64[ii], K64[jj]
    u, v = u.astype(np.float64), v.astype(np.float64)
    d = disps[ii].reshape(N, -1).astype(np.float64)
    X0 = np.stack([(u[None] - Ki[:, 2:3]) / Ki[:, 0:1], (v[None] - Ki[:, 3:4]) / Ki[:, 1:2], np.ones_like(d)], -1)
    t, q = edge_pose64(poses, ii, jj)
    X1 = _rot64(q[:, None, :], X0) + d[..., None] * t[:, None, :]
    if return_z == "points":
        return X1.reshape(N, ht, wd, 3)
    z = X1[..., 2]
    Z = np.where(z < float(F(0.5) * F(0.2)), 1.0, z)
    x = Kj[:, 0:1] * (X1[..., 0] / Z) + Kj[:, 2:3]
    y = Kj[:, 1:2] * (X1[..., 1] / Z) + Kj[:, 3:4]
    coords = np.stack([x, y], axis=-1).reshape(1, N, ht, wd, 2)
    valid = (z > float(F(0.2))).astype(np.float64).reshape(1, N, ht, wd, 1)
    if return_z:
        return coords, valid, z.reshape(N, ht, wd)
    return coords, valid


def reproject_motion(coords1, target):
    """FactorGraph.update's motion features (src/factor_graph.py:202-206), in the inputs' dtype:
    cat([coords1 - coords0, target - coords1], -1).permute(0, 1, 4, 2, 3).clamp(-64, 64) with coords0 the pixel
    grid (x, y).  coords1, target [1, N, ht, wd, 2] -> motion [1, N, 4, ht, wd] = [dx, dy, tx - x, ty - y]."""
    coords1 = np.asarray(coords1)
    target = np.asarray(target, coords1.dtype)
    ht, wd = coords1.shape[2], coords1.shape[3]
    v, u = np.meshgrid(np.arange(ht), np.arange(wd), indexing="ij")
    coords0 = np.stack([u, v], axis=-1).astype(coords1.dtype)
    motion = np.concatenate([coords1 - coords0, target - coords1], axis=-1)
    return np.clip(motion.transpose(0, 1, 4, 2, 3), -64.0, 64.0).astype(coords1.dtype)
