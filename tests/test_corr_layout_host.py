"""CPU checks of the tiled correlation layout and of the lookup oracle's out-of-image rule: the host's plane
sizes against the library's, the de-tiling map of every envelope shape, the envelope shape list's coverage, and
the oracle on NaN, infinite and huge coordinates against a scalar restatement of the reference kernel's loops."""
import math
import os
import types

import numpy as np
import pytest
import torch

import corr_envelope
from corr_envelope import BAD, nonfinite_coords
from oracle import corr_oracle


def test_plane_elems_match_the_library():
    from goslam_b200 import _lib
    from goslam_b200.modules.corr import CorrPool
    if not os.path.exists(_lib.lib_path()):
        pytest.skip("libgoslam_b200.so not built")
    lib = _lib.load(build_if_missing=False)
    for h in range(8, 137):
        for w in range(8, 129):
            host = types.SimpleNamespace(ht=h, wd=w)
            for i in range(4):
                assert CorrPool._plane_elems(host, i) == lib.goslam_corr_level_plane_elems(i, CorrPool.TILED, h, w), (h, w, i)


@pytest.mark.parametrize("hw", corr_envelope.SHAPES)
def test_level_rowmajor_is_one_to_one(hw):
    """every entry of a level has its own element of the plane; the rest of the plane is the padding set the GPU
    test overwrites"""
    from goslam_b200.modules.corr import CorrPool
    h, w = hw
    pool = CorrPool(0, h, w, device="cpu")
    for i in range(4):
        pos = corr_envelope.plane_positions(h, w, i)
        assert pos.shape == (h >> i, w >> i)
        flat = pos.reshape(-1)
        assert flat.min() >= 0 and flat.max() < pool.plane_elems[i]
        assert torch.unique(flat).numel() == flat.numel()
        pad = corr_envelope.padding_mask(h, w, i)
        assert pad.shape == (pool.plane_elems[i],)
        assert int(pad.sum()) == pool.plane_elems[i] - flat.numel()
        assert not pad[flat].any()


def test_envelope_shapes_cover_the_kernels_cases():
    shapes = corr_envelope.SHAPES
    assert len(set(shapes)) == len(shapes)
    assert all(8 <= h and 8 <= w <= 128 for h, w in shapes)                      # 4 levels, tensor-core build
    assert {-(-w // 16) for _, w in shapes} == set(range(1, 9))                  # n_xb: x-tiles per band
    assert {h % 8 for h, _ in shapes} == set(range(8))                           # rows of the last band
    assert {w % 4 for _, w in shapes} == set(range(4))                           # ragged 4x4 tiles
    assert any(w < 16 for _, w in shapes)                                        # target patch wider than the image
    hw = [h * w for h, w in shapes]
    assert any(n < 128 for n in hw)
    assert any(n % 128 == 0 for n in hw)
    assert any(n % 16 != 0 for n in hw)
    assert any(n % 8 != 0 for n in hw)


# ------------------------------------------------------------------ the reference kernel's loops, restated
def _device_int(f):
    """static_cast<int>(float) as the device converts it: toward zero, NaN -> 0, saturating"""
    if math.isnan(f):
        return 0
    if math.isinf(f):
        return 2 ** 31 - 1 if f > 0 else -2 ** 31
    return max(-2 ** 31, min(2 ** 31 - 1, math.trunc(f)))


def _i32(v):
    """int arithmetic wraps (what the reference's `floor(x0) - r + i` does at the saturated ends)"""
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


def _within_bounds(h, w, H, W):
    return h >= 0 and h < H and w >= 0 and w < W


def _reference_loops(volume, coords, r):
    """corr_index_forward_kernel (src/lib/correlation_kernels.cu:19-70), one thread at a time: `corr` starts at 0
    and only taps inside the level are added.  c10::Half arithmetic goes through float (a product of two halves
    is exact there, and float has enough bits that its rounded sum rounds to half correctly); the float
    instantiation's `corr += s * w` is one fused multiply-add."""
    N, h1, w1, h2, w2 = volume.shape
    half = volume.dtype == np.float16
    T = np.float16 if half else np.float32
    rd = 2 * r + 1
    corr = np.zeros((N, rd, rd, h1, w1), T)

    def add(n, i, j, y, x, s, wt):
        if half:
            prod = T(np.float32(s) * np.float32(T(wt)))
            corr[n, i, j, y, x] = T(np.float32(corr[n, i, j, y, x]) + np.float32(prod))
        else:
            corr[n, i, j, y, x] = T(float(s) * float(wt) + float(corr[n, i, j, y, x]))

    with np.errstate(invalid="ignore"):
        for n in range(N):
            for y in range(h1):
                for x in range(w1):
                    x0, y0 = np.float32(coords[n, 0, y, x]), np.float32(coords[n, 1, y, x])
                    dx, dy = x0 - np.floor(x0), y0 - np.floor(y0)
                    one = np.float32(1.0)
                    for i in range(rd + 1):
                        for j in range(rd + 1):
                            x1 = _i32(_device_int(float(np.floor(x0))) - r + i)
                            y1 = _i32(_device_int(float(np.floor(y0))) - r + j)
                            if _within_bounds(y1, x1, h2, w2):
                                s = volume[n, y, x, y1, x1]
                                if i > 0 and j > 0:
                                    add(n, i - 1, j - 1, y, x, s, dx * dy)
                                if i > 0 and j < rd:
                                    add(n, i - 1, j, y, x, s, dx * (one - dy))
                                if i < rd and j > 0:
                                    add(n, i, j - 1, y, x, s, (one - dx) * dy)
                                if i < rd and j < rd:
                                    add(n, i, j, y, x, s, (one - dx) * (one - dy))
    return corr


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
@pytest.mark.parametrize("shape", [(1, 9, 10, 6, 7), (1, 8, 9, 3, 4), (1, 4, 4, 12, 5)])
def test_oracle_matches_reference_loops_on_nonfinite_coordinates(dtype, shape):
    g = torch.Generator().manual_seed(sum(shape))
    vol = torch.randn(*shape, generator=g).numpy().astype(dtype)
    coords = nonfinite_coords(*shape, g).numpy()
    want = _reference_loops(vol, coords, 3)
    got = corr_oracle.corr_index_forward(vol, coords, 3)
    assert got.dtype == want.dtype
    np.testing.assert_array_equal(got, want)          # NaN where the reference has NaN, equal elsewhere
    N, h1, w1, h2, w2 = shape
    out = got.reshape(N, 49, h1 * w1)
    # x = y = NaN: floor -> 0, window origin -3, NaN weights on every tap inside: on a level of at least 5x5 the
    # 25 outputs with a tap in [0, 5) x [0, 5) are NaN, the other 24 are 0
    if h2 >= 5 and w2 >= 5:
        assert np.isnan(out[0, :, 0]).sum() == 25 and (out[0, :, 0] == 0).sum() == 24
    # an infinite coordinate: every tap outside, all 0
    assert (out[0, :, 1] == 0).all()                  # (NaN, +inf)
    assert (out[0, :, len(BAD) + 2] == 0).all()       # (+inf, NaN)


def test_oracle_finite_coordinates_unchanged_by_the_rule():
    """with finite coordinates an outside tap is 0 and its weight finite: the oracle equals the zero-tap sum"""
    g = torch.Generator().manual_seed(5)
    for dtype in (np.float16, np.float32):
        vol = torch.randn(2, 5, 6, 7, 9, generator=g).numpy().astype(dtype)
        coords = torch.stack([torch.rand(2, 5, 6, generator=g) * 17 - 4, torch.rand(2, 5, 6, generator=g) * 15 - 4], 1).numpy()
        np.testing.assert_array_equal(corr_oracle.corr_index_forward(vol, coords, 3), _reference_loops(vol, coords, 3))
