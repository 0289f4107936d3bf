"""The update's input features on the device against float64 restatements, on the crafted windows of
test_features_cases.py: reprojection (goslam_reproject), motion features (goslam_reproject_motion), projmap and
frame_distance behind the camera, and the windowed correlation (goslam_altcorr_pyramid, tensor-core and SIMT
paths) at every tile edge, plus the correlation volume against the windowed correlation.  Each bounded comparison
prints its worst error as a fraction of the bound."""
import numpy as np
import pytest
import torch

from oracle import corr_oracle, geom_oracle
from test_features_cases import CASES, T01, T02, U, coords_bound, planted_z32, reproject_case

pytestmark = pytest.mark.gpu
F = np.float32


def dev():
    return torch.device("cuda:0")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def _worst(name, err, bound):
    r = float((err / bound).max()) if err.size else 0.0
    print("%-40s worst error / bound = %.3g" % (name, r))
    assert r <= 1.0, (name, r)


# ----------------------------------------------------------------------------- reprojection + motion
@pytest.mark.parametrize("name", CASES)
def test_reproject_and_motion_vs_float64(name):
    from goslam_b200 import droid_backends
    c = reproject_case(name)
    args = [_t(c[k]) for k in ("poses", "disps", "intrinsics", "ii", "jj")]
    co, va = droid_backends.reproject(*args)
    co_nv, none = droid_backends.reproject(*args, want_valid=False)
    assert none is None and torch.equal(co_nv, co), "coords depend on whether valid is written"
    cm, mo = droid_backends.reproject_motion(*args, _t(c["target"]))
    assert torch.equal(cm, co), "reproject_motion's coords differ from reproject's"
    co, va, mo = co.cpu().numpy(), va.cpu().numpy(), mo.cpu().numpy()
    # motion = the clamp formula on the kernel's own coords, bit for bit: channels [dx, dy, tx - x, ty - y]
    np.testing.assert_array_equal(mo, geom_oracle.reproject_motion(co, c["target"]))

    # classification: float64 everywhere except the planted edges, whose float32 depth fma(d, tz, 1) is exact
    X1 = geom_oracle.reproject(c["poses"], c["disps"], c["intrinsics"], c["ii"], c["jj"], dtype=np.float64,
                               return_z="points")
    z64 = X1[..., 2]
    zp = planted_z32(c)
    pl = np.broadcast_to(c["planted"][:, None, None], z64.shape)
    replaced = np.where(pl, zp < T01, z64 < float(T01))
    valid = np.where(pl, zp > T02, z64 > float(T02))
    np.testing.assert_array_equal(va[0, ..., 0], valid.astype(F))
    assert ((z64 > 0.2) & (z64 < 0.25) & (va[0, ..., 0] == 1)).any() or name == "pixel_1x1"

    # coordinates: float64 with the kernel's branch, per-pixel bound (coords_bound)
    Z = np.where(replaced, 1.0, z64)
    Kj = c["intrinsics"].astype(np.float64)[c["jj"]][:, :, None, None]
    c64 = np.stack([Kj[:, 0] * (X1[..., 0] / Z) + Kj[:, 2], Kj[:, 1] * (X1[..., 1] / Z) + Kj[:, 3]], -1)
    bx, by, _ = coords_bound(c, Z, X1)
    err = np.abs(co[0].astype(np.float64) - c64)
    _worst("reproject coords x [%s]" % name, err[..., 0], bx)
    _worst("reproject coords y [%s]" % name, err[..., 1], by)
    # motion: the float64 features of the float64 coords; the clamp is 1-Lipschitz, the subtraction one rounding
    m64 = geom_oracle.reproject_motion(c64[None], c["target"].astype(np.float64))
    g = np.stack(np.meshgrid(np.arange(c["wd"]), np.arange(c["ht"]), indexing="xy"), -1)[None]
    raw = np.concatenate([c64 - g, c["target"][0] - c64], -1)
    mb = np.stack([bx, by, bx, by], -1) + U * np.abs(raw)
    _worst("motion [%s]" % name, np.abs(mo[0].astype(np.float64) - m64[0]).transpose(0, 2, 3, 1), mb)


def test_projmap_and_frame_distance_behind_the_camera():
    """projmap's Xj_z <= 0.01 pixel-grid fallback and frame_distance's valid < 0.75 -> 1000 branch on the crafted
    rig window (frames facing away), under the existing contracts: valid exact, the >= 999 sets exact."""
    from goslam_b200 import droid_backends
    c = reproject_case("rig_37x45")
    num = c["poses"].shape[0]
    ii, jj = [a.reshape(-1) for a in np.meshgrid(np.arange(num), np.arange(num), indexing="ij")]
    intr0 = c["intrinsics"][0]
    P, D = _t(c["poses"]), _t(c["disps"])
    co, va = droid_backends.projmap(P, D, _t(intr0), _t(ii), _t(jj))
    rc, rv = geom_oracle.projmap(c["poses"], c["disps"], intr0, ii, jj)
    np.testing.assert_array_equal(va.cpu().numpy(), rv)
    t, q = geom_oracle.edge_pose(c["poses"], ii, jj, stereo_special=False)
    Xi = geom_oracle.backproject(c["disps"][ii].reshape(len(ii), -1), intr0, c["ht"], c["wd"])
    zj = geom_oracle.act_se3(t[:, None], q[:, None], Xi)[..., 2].reshape(rv.shape[:3])
    fb = zj <= 0.01
    assert fb.sum() > 1000 and (~fb).sum() > 1000
    got = co.cpu().numpy()
    np.testing.assert_array_equal(got[fb], rc[fb])                       # the pixel grid, exactly
    clear = np.abs(zj - 0.01) > 1e-5
    np.testing.assert_allclose(got[~fb & clear], rc[~fb & clear], rtol=1e-4, atol=1e-3)
    for fn, ref in ((droid_backends.frame_distance, None), (droid_backends.frame_distance_bidirectional, None)):
        d = fn(P, D, _t(intr0), _t(ii), _t(jj), 0.3).cpu().numpy()
        r = geom_oracle.frame_distance(c["poses"], c["disps"], intr0, ii, jj, 0.3)
        if fn is droid_backends.frame_distance_bidirectional:
            r2 = geom_oracle.frame_distance(c["poses"], c["disps"], intr0, jj, ii, 0.3)
            r = (F(0.5) * (r + r2)).astype(F)
        far = r >= 999
        assert far.any() and (~far).any()
        np.testing.assert_array_equal(d >= 999, far)
        np.testing.assert_allclose(d[~far], r[~far], rtol=2e-4, atol=1e-4)


# ----------------------------------------------------------------------------- windowed correlation
def _fmaps(F_, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(1, F_, C, H, W, generator=g).half().to(dev())


def _coords(kind, N, H, W, seed):
    """[1, N, H, W, 2] float32 coordinate fields (level-0 pixels)."""
    rng = np.random.default_rng(seed)
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    grid = np.broadcast_to(np.stack([x, y], -1), (N, H, W, 2)).copy()
    if kind == "smooth":
        c = grid + 2.0 * np.sin(grid[..., ::-1] / 5.0 + rng.normal(size=(N, 1, 1, 2))) + rng.normal(size=(N, 1, 1, 2))
    elif kind == "scattered":                      # a warp's box spans the whole target level
        c = rng.uniform(0, 1, (N, H, W, 2)) * [W + 8, H + 8] - 4
    elif kind == "far":                            # one pixel of every 16 at +-1e6, the rest in the image
        c = grid + rng.normal(size=(N, H, W, 2))
        flat = c.reshape(N, -1, 2)
        flat[:, 5::16] = rng.choice([-1e6, 1e6], size=flat[:, 5::16].shape)
    elif kind == "empty":                          # whole warps outside: empty boxes, and a ragged last warp
        c = grid + rng.normal(size=(N, H, W, 2))
        flat = c.reshape(N, -1, 2)
        k = np.arange(flat.shape[1])
        out = ((k // 16) % 3 == 0) | (k >= flat.shape[1] - 7)
        flat[:, out] = rng.choice([-60.0, 1e4], size=(N, int(out.sum()), 2))
    elif kind == "intfrac":                        # integer and negative fractional coordinates
        c = np.round(grid + 3 * rng.normal(size=(N, H, W, 2)))
        c[..., ::2, :] -= rng.choice([0.25, 0.5, 3.75], size=c[..., ::2, :].shape)
        c = np.where(rng.uniform(size=c.shape) < 0.3, -rng.uniform(0, 3, c.shape), c)
    elif kind == "border":                         # windows hanging over each border at each level
        s = 2.0 ** rng.integers(0, 4, (N, H, W, 1))
        lim = np.array([W, H], np.float64)
        edge = rng.choice([-1, 0, 1], size=(N, H, W, 2))
        off = rng.uniform(-4.5, 4.5, (N, H, W, 2))
        c = np.where(edge < 0, off * s, np.where(edge > 0, lim - 1 + off * s, grid))
    else:
        raise ValueError(kind)
    return torch.from_numpy(c.astype(F))[None].to(dev())


def _edges(N, F_, seed):
    rng = np.random.default_rng(seed)
    ii, jj = rng.integers(0, F_, N), rng.integers(0, F_, N)
    if N > 2:
        ii[1], jj[1] = ii[0], jj[0]                 # a repeated edge
    return torch.from_numpy(ii).to(dev()), torch.from_numpy(jj).to(dev())


def _alt_bound(mag, C):
    """mma.sync f16 x f16 -> f32: products of halves are exact in fp32; the C-term accumulation and the 4-tap blend
    are <= C + 4 further additions plus the weight products, each within one fp32 ulp (2u: the tensor core's
    accumulation may truncate rather than round).  So |out - exact| <= 2 * 2^-24 * (C + 4) * mag, with mag the
    per-output sum_taps |w| sum_c |f1 f2| the oracle returns; zero-magnitude outputs must be exactly zero."""
    return 2.0 * U * (C + 4) * mag


def _check_alt(name, got, fm, coords, ii, jj, L):
    blk_pyr = [p[0] for p in fm]
    want, mag = corr_oracle.altcorr_pyramid(blk_pyr, coords[0], ii, jj, L)
    err = (got[0].double() - want).abs()
    C = blk_pyr[0].shape[-1]
    _worst(name, err.cpu().numpy(), np.maximum(_alt_bound(mag, C).cpu().numpy(), 1e-300))


ALT_SHAPES = [(30, 40, 4, 300), (48, 64, 4, 24), (60, 80, 4, 8), (37, 45, 3, 17), (8, 8, 4, 1), (37, 45, 1, 5),
              (30, 40, 2, 9)]


@pytest.mark.parametrize("field", ["smooth", "scattered", "far", "empty", "intfrac", "border"])
@pytest.mark.parametrize("shape", ALT_SHAPES, ids=lambda s: "%dx%d_L%d_N%d" % s)
def test_altcorr_vs_float64(shape, field):
    from goslam_b200.modules import AltCorrBlock
    H, W, L, N = shape
    F_ = 6
    fm = _fmaps(F_, 128, H, W, seed=H * W + L)
    blk = AltCorrBlock(fm, num_levels=L)
    coords = _coords(field, N, H, W, seed=N + L)
    ii, jj = _edges(N, F_, seed=N)
    got = blk(coords, ii, jj)
    assert got.shape == (1, N, L * 49, H, W)
    _check_alt("altcorr tc %dx%d L%d N%d %s" % (H, W, L, N, field), got, blk.pyramid, coords, ii, jj, L)


def test_altcorr_6d_sliced_and_gathered_coords():
    """S = 2 coordinate sets, and the chunked forms update_lowmem passes (coords1[:, lo:hi] and coords1[:, pos]):
    every row equals the whole-graph call's bit for bit."""
    from goslam_b200.modules import AltCorrBlock
    H, W, N = 30, 40, 23
    fm = _fmaps(5, 128, H, W, seed=3)
    blk = AltCorrBlock(fm)
    coords = _coords("smooth", N, H, W, seed=4)
    ii, jj = _edges(N, 5, seed=5)
    full = blk(coords, ii, jj)
    lo, hi = 7, 19
    assert torch.equal(blk(coords[:, lo:hi], ii[lo:hi], jj[lo:hi]), full[:, lo:hi])
    pos = torch.tensor([22, 3, 3, 0, 17], device=dev())
    assert torch.equal(blk(coords[:, pos], ii[pos], jj[pos]), full[:, pos])
    c6 = torch.stack([coords, _coords("scattered", N, H, W, seed=6)], dim=-2)
    out6 = blk(c6, ii, jj)
    assert out6.shape == (1, N, 196, H, W, 2)
    assert torch.equal(out6[..., 0], full)
    _check_alt("altcorr 6-D set 1", out6[..., 1], blk.pyramid, c6[..., 1, :], ii, jj, 4)


@pytest.mark.parametrize("C", [64, 256])
def test_altcorr_simt_fallback(C):
    from goslam_b200.modules import AltCorrBlock
    H, W, N = 37, 45, 11
    fm = _fmaps(4, C, H, W, seed=C)
    blk = AltCorrBlock(fm, num_levels=3)
    for field in ("smooth", "border", "far"):
        coords = _coords(field, N, H, W, seed=C + 1)
        ii, jj = _edges(N, 4, seed=C + 2)
        _check_alt("altcorr simt C%d %s" % (C, field), blk(coords, ii, jj), blk.pyramid, coords, ii, jj, 3)


def test_altcorr_rejects_bad_shapes():
    """C % 8 != 0 and a level that shrinks to zero are shape errors, returned before any launch."""
    from goslam_b200 import _lib
    from goslam_b200.modules.corr import _ptr_array
    lib = _lib.load()
    H, W, N = 4, 8, 2
    pyr = [torch.zeros(1, H >> l, W >> l, 12, dtype=torch.float16, device=dev()) for l in range(3)]
    c = torch.zeros(N, H, W, 2, device=dev())
    e = torch.zeros(N, dtype=torch.int64, device=dev())
    out = torch.empty(N, 4 * 49, H, W, device=dev())
    assert lib.goslam_altcorr_pyramid(_ptr_array(pyr), 1, _lib.ptr(c), _lib.ptr(e), _lib.ptr(e), _lib.ptr(out),
                                      N, H, W, 12, 3, _lib.stream_ptr()) == -1
    pyr = [torch.zeros(1, H >> l, W >> l, 16, dtype=torch.float16, device=dev()) for l in range(3)] + [pyr[0]]
    assert lib.goslam_altcorr_pyramid(_ptr_array(pyr), 4, _lib.ptr(c), _lib.ptr(e), _lib.ptr(e), _lib.ptr(out),
                                      N, H, W, 16, 3, _lib.stream_ptr()) == -1          # level 3 of H = 4 is empty


def test_altcorr_pyramid_levels_are_rounded_averages():
    """level l = the float64 2x2 average of level l - 1 (level 0 = fmaps / 4, exact), rounded to half: within one
    half ulp of that average (the worst case is printed in half ulps; the assertion allows one ulp)."""
    from goslam_b200.modules import AltCorrBlock
    fm = _fmaps(3, 128, 37, 45, seed=9)
    blk = AltCorrBlock(fm)
    prev = (fm.double() / 4).permute(0, 1, 3, 4, 2)
    for lvl, p in enumerate(blk.pyramid):
        if lvl:
            q = prev[..., : 2 * p.shape[2], : 2 * p.shape[3], :]
            prev = q.unflatten(2, (-1, 2)).unflatten(4, (-1, 2)).mean(dim=(3, 5))
        half_ulp = torch.where(prev.abs() < 2.0 ** -14, torch.full_like(prev, 2.0 ** -25),
                               2.0 ** (torch.floor(torch.log2(prev.abs().clamp_min(2.0 ** -14))) - 11))
        r = float(((p.double() - prev).abs() / half_ulp).max())
        print("pyramid level %d: worst |level - average| = %.3g half ulps" % (lvl, r))
        assert r <= 2.0, (lvl, r)
        prev = p.double()


def test_volume_equals_windowed_correlation_rig2():
    """CorrBlock.from_video (the 4-D volume, pooled in half) and AltCorrBlock (pooled features) compute the same
    quantity on a stereo rig (rig 2, frames rig*i and rig*j + (i == j)).  Bound: the volume level l holds l + 1
    half roundings of averages, the half lookup 4 products + 3 adds + its output and its weights in half, so
    (l + 10) * 2^-11 * a magnitude that dominates every tap (the oracle on |f1| and max-pooled |f2|), plus an
    absolute 2^-20 for half subnormals, plus the windowed correlation's own bound."""
    from goslam_b200.modules import AltCorrBlock
    from goslam_b200.modules.corr import CorrBlock, fmaps_to_kmajor
    buf, rig, H, W = 5, 2, 40, 60
    g = torch.Generator().manual_seed(21)
    fmaps = torch.randn(buf, rig, 128, H, W, generator=g).half().to(dev())
    ii = torch.tensor([0, 1, 2, 2, 4, 3, 0, 1], device=dev())
    jj = torch.tensor([1, 0, 2, 3, 4, 1, 0, 4], device=dev())
    N = ii.numel()
    coords = torch.cat([_coords("smooth", N // 2, H, W, seed=1), _coords("border", N - N // 2, H, W, seed=2)], 1)
    vol = CorrBlock.from_video(fmaps_to_kmajor(fmaps), ii, jj, H, W, rig=rig)(coords).float()
    blk = AltCorrBlock(fmaps.reshape(1, buf * rig, 128, H, W))
    ia, ja = rig * ii, rig * jj + (ii == jj).long()
    alt = blk(coords, ia, ja)
    apyr = [(fmaps.reshape(buf * rig, 128, H, W).float() / 4).abs()]
    for _ in range(3):
        apyr.append(torch.nn.functional.max_pool2d(apyr[-1], 2))
    apyr = [p.permute(0, 2, 3, 1).contiguous() for p in apyr]
    amag, _ = corr_oracle.altcorr_pyramid(apyr, coords[0], ia, ja, 4)
    want, mag = corr_oracle.altcorr_pyramid([p[0] for p in blk.pyramid], coords[0], ia, ja, 4)
    lvl = torch.arange(4, device=dev()).repeat_interleave(49).view(1, -1, 1, 1).double()
    bound = (lvl + 10) * 2.0 ** -11 * amag + 2.0 ** -20 + _alt_bound(mag, 128)
    _worst("volume vs windowed correlation (rig 2)", (vol[0].double() - alt[0].double()).abs().cpu().numpy(),
           bound.cpu().numpy())
    # ...and both against the float64 restatement
    _worst("windowed correlation (rig 2)", (alt[0].double() - want).abs().cpu().numpy(),
           np.maximum(_alt_bound(mag, 128).cpu().numpy(), 1e-300))
