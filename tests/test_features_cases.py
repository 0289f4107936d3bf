"""Crafted inputs for the update's input features (reprojection, motion features, windowed correlation) and CPU
pins of their float64 restatements.

`synthetic.make_scene` windows have small motions, inverse depths in 0.5-0.9, one intrinsics row and no stereo edge,
so they never reach the branches where a reprojection kernel can be silently wrong.  `reproject_case` builds windows
that do:
  * frames rotated by up to 180 degrees (some look away from the others) and translated by about the scene depth;
  * inverse depths that are 0 (points at infinity), negative, tiny or large;
  * different intrinsics per frame, so Ki and Kj of an edge differ;
  * stereo self-edges (ii == jj, the fixed 0.1 baseline), unsorted and repeated edges;
  * planted pixels whose depth X1z in frame j lands exactly on 0.1 and 0.2 (the Z-replacement and `valid` thresholds)
    and a few ulp either side, plus pixels in (0.2, 0.25) so that 0.2 cannot be confused with 0.25;
  * motion features exactly at +-64 and beyond, on both sides, in every channel.
Planted frames: P at the origin and A, B translated along z only, all with the identity rotation.  Then the edge's
X1 is X0 + d * t exactly except for X1z = fma(d, tz, 1) (one rounding), so X1z = 0.1f exactly when d * tz = 0.1f - 1
exactly: 0.1f - 1 = -120795955 * 2^-27 = -(34405 * 2^-15) * (3511 * 2^-12) and 0.2f - 1 = -53687091 * 2^-26 =
-(3741 * 2^-12) * (14351 * 2^-14).  With d = 0 and fx a power of two, coords are exact small numbers, so target
offsets of exactly +-64 survive the float32 arithmetic.
"""
import os

import numpy as np
import torch

from oracle import corr_oracle, geom_oracle

F = np.float32
U = 2.0 ** -24                                   # float32 unit roundoff
T01, T02 = F(0.5) * F(0.2), F(0.2)               # the kernel's thresholds: Z < 0.1 -> 1, valid = X1z > 0.2
D01, TZ01 = F(34405 * 2.0 ** -15), F(-3511 * 2.0 ** -12)       # D01 * TZ01 == 0.1f - 1 exactly
D02, TZ02 = F(3741 * 2.0 ** -12), F(-14351 * 2.0 ** -14)       # D02 * TZ02 == 0.2f - 1 exactly
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "features.npz")


def _quat(axis, angle):
    axis = np.asarray(axis, np.float64)
    axis = axis / np.linalg.norm(axis)
    return np.concatenate([np.sin(angle / 2) * axis, [np.cos(angle / 2)]])


def _ulps(x, k):
    """x moved by k float32 ulps (k may be negative)."""
    x = F(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, F(np.inf) if k > 0 else F(-np.inf), dtype=F)
    return x


def x1z_bound(case):
    """per-pixel bound on |X1z(float32 kernel) - X1z(float64)|, see test_gpu_features.coords_bound."""
    return coords_bound(case)[2]


def coords_bound(case, Z64=None, X1=None):
    """Per-pixel bounds on the float32 errors of X1 = G_ij * X0 and of the projected coords [N, ht, wd] each.

    The kernel computes (all float32, u = 2^-24): the relative pose G = (t, q) from the two stored poses (q: four
    products summed, t = tj - R(q) ti), X0 = ((x - cx) / fx, (y - cy) / fy, 1, d), X1 = R(q) X0 + d t, Z, then
    x' = fx_j * (X1x / Z) + cx_j.  Every quantity on the way is a sum of at most ~8 terms whose absolute values are
    bounded by M = |X0|_1 + |d| (|ti|_1 + |tj|_1) (|q| <= 1 component-wise, the stored quaternions are unit to
    float32 precision), and each path has at most ~12 roundings plus the relative-pose errors it inherits; 64 u M
    covers both with room (the measured worst case is reported as a fraction of this bound).  Division by Z adds
    the 1/Z^2 amplification: |d(X/Z)| <= (eX + |X/Z| eZ) / (|Z| - eZ) + u |X/Z|, and the final multiply-add two
    roundings of its magnitude.  Where Z was replaced by 1 it is exact (eZ = 0)."""
    P = case["poses"].astype(np.float64)
    Kall = case["intrinsics"].astype(np.float64)
    ii, jj = case["ii"], case["jj"]
    N = len(ii)
    ht, wd = case["disps"].shape[1:]
    v, u = np.meshgrid(np.arange(ht), np.arange(wd), indexing="ij")
    Ki, Kj = Kall[ii][:, :, None, None], Kall[jj][:, :, None, None]
    d = case["disps"][ii].astype(np.float64)
    X0 = np.abs((u - Ki[:, 2]) / Ki[:, 0]) + np.abs((v - Ki[:, 3]) / Ki[:, 1]) + 1.0
    tn = (np.abs(P[ii, :3]).sum(-1) + np.abs(P[jj, :3]).sum(-1))[:, None, None]
    M = X0 + np.abs(d) * np.maximum(tn, 0.1)          # self-edges use the fixed 0.1 baseline
    eX = 64 * U * M
    if Z64 is None:
        return None, None, eX
    rep = np.abs(Z64 - 1.0) == 0
    eZ = np.where(rep, 0.0, eX)
    Za = np.abs(Z64) - eZ
    out = []
    for c in (0, 1):
        r = np.abs(X1[..., c]) / np.abs(Z64)
        e = (eX + r * eZ) / Za + U * r
        out.append(np.abs(Kj[:, c]) * e + 2 * U * (np.abs(Kj[:, c]) * r + np.abs(Kj[:, c + 2])) + U)
    return out[0], out[1], eX


def reproject_case(name):
    """crafted window -> dict(poses [num,7], disps [num,ht,wd], intrinsics [num,4], ii, jj [K] int64,
    target [1,K,ht,wd,2], planted [K] bool (edges P->A, P->B, A->P: identity rotation, z translation),
    tz [K] (their translation), ht, wd)."""
    ht, wd, n_rand, K_rand, seed = {"rig_37x45": (37, 45, 6, 0, 1), "strip_7x45": (7, 45, 5, 0, 2),
                                     "pixel_1x1": (1, 1, 4, 0, 3), "many_60x80": (60, 80, 20, 300, 4)}[name]
    rng = np.random.default_rng(seed)
    num = n_rand + 3
    iP, iA, iB = n_rand, n_rand + 1, n_rand + 2
    poses = np.zeros((num, 7))
    for f in range(n_rand):
        ang = np.pi if f == 1 else rng.uniform(0, np.pi)     # frame 1: a half turn, exactly facing away
        poses[f, 3:] = _quat(rng.normal(size=3), ang)
        poses[f, :3] = rng.normal(size=3) * rng.uniform(0.2, 2.0)
    poses[iP, 6] = poses[iA, 6] = poses[iB, 6] = 1.0
    poses[iA, 2], poses[iB, 2] = TZ01, TZ02
    poses = poses.astype(F)
    intr = np.stack([rng.uniform(20, 60, num), rng.uniform(20, 60, num), rng.uniform(0, wd, num),
                     rng.uniform(0, ht, num)], 1).astype(F)
    # planted frames: power-of-two focal lengths and integer / half principal points -> exact d = 0 coords
    intr[iP] = [32, 16, wd // 2, ht // 2]
    intr[iA] = [32, 16, wd // 2 + 64, ht // 2 - 70]                  # x' - x = +64, y' - y = -70 (clamped)
    intr[iB] = [32, 16, wd // 2 - 80, ht // 2 + 64]                  # x' - x = -80 (clamped), y' - y = +64
    disps = rng.uniform(0.2, 2.0, (num, ht, wd))
    kind = rng.integers(0, 10, (num, ht, wd))
    disps = np.where(kind == 0, 0.0, disps)                                       # infinity
    disps = np.where(kind == 1, -rng.uniform(0, 1.5, (num, ht, wd)), disps)       # behind
    disps = np.where(kind == 2, rng.uniform(0, 1e-6, (num, ht, wd)), disps)        # tiny
    disps = np.where(kind == 3, rng.uniform(5, 20, (num, ht, wd)), disps)          # close
    disps = disps.astype(F)
    # frame P: the planted values, row-major from pixel 0, the rest random
    planted_d = [F(0.0)] * 3
    for dd in (D01, D02):
        planted_d += [_ulps(dd, k) for k in range(-3, 4)]
    for tz in (TZ01, TZ02):                                        # X1z in (0.2, 0.25), (0.25, 1), < 0.1, < 0
        planted_d += [F((z - 1) / tz) for z in (0.21, 0.235, 0.249, 0.26, 0.5, 0.05, -0.3)]
    flat = disps[iP].reshape(-1)
    m = min(len(planted_d), flat.size)
    flat[:m] = planted_d[:m]
    if ht >= 2:
        disps[iP, -1, :] = 0.0                                     # a row of exact d = 0 coords
    # edges: all ordered pairs of the random frames, self-edges (stereo), the planted edges, a repeat
    if K_rand:
        ii = rng.integers(0, n_rand, K_rand)
        jj = rng.integers(0, n_rand, K_rand)
        jj[::7] = ii[::7]
    else:
        a, b = np.meshgrid(np.arange(n_rand), np.arange(n_rand), indexing="ij")
        ii, jj = a.reshape(-1), b.reshape(-1)
    pl_i = np.array([iP, iP, iA, iP, iB, iP])
    pl_j = np.array([iA, iB, iP, iA, iB, iP])
    ii = np.concatenate([ii, pl_i, ii[:3]]).astype(np.int64)
    jj = np.concatenate([jj, pl_j, jj[:3]]).astype(np.int64)
    perm = rng.permutation(len(ii))
    ii, jj = ii[perm], jj[perm]
    planted = (ii >= iP) & (ii != jj)
    tz = np.where(planted, poses[jj, 2] - poses[ii, 2], 0).astype(F)
    case = dict(name=name, poses=poses, disps=disps, intrinsics=intr, ii=ii, jj=jj, planted=planted, tz=tz,
                ht=ht, wd=wd, iP=iP)
    # keep the random edges' pixels out of the float32 uncertainty band around the thresholds, so that every band
    # pixel is a planted one, whose float32 depth is known exactly (fma(d, tz, 1))
    for _ in range(20):
        _, _, z = geom_oracle.reproject(poses, disps, intr, ii, jj, dtype=np.float64, return_z=True)
        ez = x1z_bound(case)
        near = ((np.abs(z - float(T01)) <= ez) | (np.abs(z - float(T02)) <= ez)) & ~planted[:, None, None]
        if not near.any():
            break
        e, y, x = np.nonzero(near)
        disps[ii[e], y, x] += F(0.01) * (1 + np.abs(disps[ii[e], y, x]))
    else:
        raise AssertionError("could not clear the threshold band")
    # targets: coords (float32 restatement) plus offsets; on exact pixels offsets of exactly +-64 and beyond
    c32, _ = geom_oracle.reproject(poses, disps, intr, ii, jj)
    off = rng.normal(size=c32.shape) * 60.0
    choice = np.array([64.0, -64.0, 63.0, -65.0, 1000.0, -0.5], F)
    exact = off_mask = (disps[ii] == 0)[None, ..., None] & planted[None, :, None, None, None]
    off = np.where(np.broadcast_to(off_mask, off.shape), choice[rng.integers(0, len(choice), off.shape)], off)
    case["target"] = (c32 + off.astype(F)).astype(F)
    case["exact"] = np.broadcast_to(exact[..., 0], (1,) + ii.shape + (ht, wd))[0]
    return case


CASES = ["rig_37x45", "strip_7x45", "pixel_1x1", "many_60x80"]


def planted_z32(case):
    """float32 X1z of the kernel on planted edges (identity rotation: fma(d, tz, 1), one rounding); NaN elsewhere."""
    d = case["disps"][case["ii"]]
    z = geom_oracle.fma(d, case["tz"][:, None, None], F(1))
    return np.where(case["planted"][:, None, None], z, np.nan)


# ----------------------------------------------------------------------------- case content
def test_reproject_cases_contain_what_they_claim():
    tot = dict(z_exact01=0, z_exact02=0, band01_lo=0, band01_hi=0, band02_lo=0, band02_hi=0, between=0,
               replaced=0, behind=0, valid0=0, valid1=0, stereo=0, m_pos64=0, m_neg64=0, m_beyond_pos=0,
               m_beyond_neg=0, d0=0, dneg=0, facing_away=0)
    for name in CASES:
        c = reproject_case(name)
        _, valid, z = geom_oracle.reproject(c["poses"], c["disps"], c["intrinsics"], c["ii"], c["jj"],
                                            dtype=np.float64, return_z=True)
        z32 = planted_z32(c)
        with np.errstate(invalid="ignore"):
            tot["z_exact01"] += int((z32 == T01).sum())
            tot["z_exact02"] += int((z32 == T02).sum())
            for thr, tag in ((T01, "01"), (T02, "02")):
                near = (np.abs(z32 - thr) <= 32 * np.spacing(thr)) & (z32 != thr)
                tot["band%s_lo" % tag] += int((near & (z32 < thr)).sum())
                tot["band%s_hi" % tag] += int((near & (z32 > thr)).sum())
        tot["between"] += int(((z > 0.2) & (z < 0.25)).sum())
        tot["replaced"] += int((z < float(T01)).sum())
        tot["behind"] += int((z < 0).sum())
        tot["valid0"] += int((valid == 0).sum())
        tot["valid1"] += int((valid == 1).sum())
        tot["stereo"] += int((c["ii"] == c["jj"]).sum())
        Ki, Kj = c["intrinsics"][c["ii"]], c["intrinsics"][c["jj"]]
        assert ((Ki != Kj).any(1) | (c["ii"] == c["jj"])).all(), "every non-stereo edge has Ki != Kj"
        c32, _ = geom_oracle.reproject(c["poses"], c["disps"], c["intrinsics"], c["ii"], c["jj"])
        raw = np.concatenate([c32 - _grid(c), c["target"] - c32], -1)
        ex = c["exact"][None, ..., None]
        tot["m_pos64"] += int(((raw == 64) & ex).sum())
        tot["m_neg64"] += int(((raw == -64) & ex).sum())
        tot["m_beyond_pos"] += int(((raw > 64) & ex).sum())
        tot["m_beyond_neg"] += int(((raw < -64) & ex).sum())
        tot["d0"] += int((c["disps"] == 0).sum())
        tot["dneg"] += int((c["disps"] < 0).sum())
        tot["facing_away"] += int(((c["poses"][:, 6] ** 2) < 0.02).sum())
        assert (c["disps"].shape[1] * c["disps"].shape[2]) % 256 != 0 or name == "many_60x80"
    print(tot)
    for k, v in tot.items():
        assert v > 0, (k, tot)


def _grid(c):
    v, u = np.meshgrid(np.arange(c["ht"]), np.arange(c["wd"]), indexing="ij")
    return np.stack([u, v], -1).astype(F)[None, None]


def test_reproject64_restates_float32_oracle():
    """the float64 restatement agrees with the float32 one away from the thresholds, and classifies the planted
    exact-threshold pixels as the float32 arithmetic does (X1z == 0.1f is not replaced; == 0.2f is not valid)."""
    c = reproject_case("rig_37x45")
    args = (c["poses"], c["disps"], c["intrinsics"], c["ii"], c["jj"])
    c32, v32, z32 = geom_oracle.reproject(*args, return_z=True)
    c64, v64, z64 = geom_oracle.reproject(*args, dtype=np.float64, return_z=True)
    far = (np.abs(z64 - 0.1) > 1e-4) & (np.abs(z64 - 0.2) > 1e-4)
    assert (v32[0, ..., 0] == v64[0, ..., 0])[far].all()
    np.testing.assert_allclose(c32[0][far], c64[0][far], rtol=1e-4, atol=1e-3)
    zp = planted_z32(c)
    on01, on02 = zp == T01, zp == T02
    assert on01.any() and on02.any()
    assert (z64[on01] == float(T01)).all() and (z64[on02] == float(T02)).all()
    assert (v64[0, ..., 0][on02] == 0).all()


def test_reproject_motion_oracle_layout():
    c = reproject_case("rig_37x45")
    c32, _ = geom_oracle.reproject(c["poses"], c["disps"], c["intrinsics"], c["ii"], c["jj"])
    m = geom_oracle.reproject_motion(c32, c["target"])
    g = _grid(c)
    np.testing.assert_array_equal(m[:, :, 0], np.clip(c32[..., 0] - g[..., 0], -64, 64))
    np.testing.assert_array_equal(m[:, :, 3], np.clip(c["target"][..., 1] - c32[..., 1], -64, 64))


def test_features_golden_pins_reproject64_and_motion():
    """the reference's own pops.projective_transform and FactorGraph.update's motion lines on the crafted
    rig case (tests/golden/make_golden.py gen_features): the float32 outputs of the reference equal the float64
    restatement within float32 rounding wherever the depth is clear of the thresholds, classify alike, and the
    motion features equal the restatement applied to the reference's own coords bit for bit."""
    g = np.load(GOLDEN)
    args = (g["poses"], g["disps"], g["intrinsics"], g["ii"], g["jj"])
    c64, v64, z64 = geom_oracle.reproject(*args, dtype=np.float64, return_z=True)
    far = (np.abs(z64 - 0.1) > 1e-4) & (np.abs(z64 - 0.2) > 1e-4)
    assert far.mean() > 0.9
    np.testing.assert_array_equal(g["valid"][0, ..., 0][far], v64[0, ..., 0][far])
    np.testing.assert_allclose(g["coords"][0][far], c64[0][far], rtol=1e-4, atol=1e-3)
    np.testing.assert_array_equal(g["motion"], geom_oracle.reproject_motion(g["coords"], g["target"]))
    # the planted exact-threshold pixels, classified as float32 does
    zp = geom_oracle.fma(g["disps"][g["ii"]], g["tz"][:, None, None], F(1))
    on02 = g["planted"][:, None, None] & (zp == T02)
    assert on02.any() and (g["valid"][0, ..., 0][on02] == 0).all()


# ----------------------------------------------------------------------------- windowed correlation oracle
def test_altcorr_pyramid_oracle_matches_reference_class_golden():
    """the float64 windowed-correlation restatement on the reference AltCorrBlock's own golden outputs
    (tests/golden/altcorr_block.npz: fp32 maps, fp32 kernel): same levels, channel order and edge indexing."""
    from goslam_b200.modules.corr import AltCorrBlock
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "altcorr_block.npz"))
    blk = AltCorrBlock(torch.from_numpy(g["fmaps"]))
    pyr = [p[0] for p in blk.pyramid]
    ii, jj = torch.from_numpy(g["ii"]), torch.from_numpy(g["jj"])
    for coords, want in ((g["coords"][0], g["out5"][0]), (g["coords6"][0, ..., 1, :], g["out6"][0, ..., 1])):
        out, mag = corr_oracle.altcorr_pyramid(pyr, torch.from_numpy(np.ascontiguousarray(coords)), ii, jj,
                                               blk.num_levels)
        got = out.numpy()[:, ::7]
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()
        assert (mag.numpy() >= np.abs(out.numpy())).all()
