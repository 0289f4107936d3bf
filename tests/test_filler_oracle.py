"""The float64 trajectory-filler oracle (oracle/filler_oracle.py) pinned to what the REFERENCE PoseTrajectoryFiller
computed on the golden scenario (tests/golden/trajectory_filler.npz): bracket indices exactly, interpolated poses
within 1e-6; and its exp / log against the lietorch shim."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import filler_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))
G = np.load(os.path.join(HERE, "golden", "trajectory_filler.npz"))


@pytest.mark.parametrize("kind", ["rgbd", "mono", "stereo"])
def test_oracle_matches_reference_interpolation(kind):
    import filler_scenario as fs
    ts = np.array(fs.KF_T, np.float32)
    poses = fs.keyframe_poses().numpy()
    tt = np.array([s[0] for s in fs.stream(kind)], np.float32)
    n = int(G[kind + "_chunks"])
    assert n == -(-len(tt) // 16)
    for c in range(n):
        t0, t1, P = fo.interpolate(ts, poses, tt[16 * c:16 * (c + 1)])
        np.testing.assert_array_equal(t0, G["%s_c%d_t0" % (kind, c)])
        np.testing.assert_array_equal(t1, G["%s_c%d_t1" % (kind, c)])
        err = np.abs(P - G["%s_c%d_G" % (kind, c)]).max(-1)
        np.testing.assert_array_less(err, fo.bound(ts, poses, tt[16 * c:16 * (c + 1)], 1e-6))
    # the scenario covers frames on, between and after the keyframes
    if kind == "rgbd":
        t0, t1 = fo.bracket(ts, tt)
        assert (t0 == t1).sum() == 3 and np.isin(tt, ts).sum() == len(ts) and (~np.isin(tt, ts)).sum() > 20


def test_exp_log_against_shim():
    from goslam_b200 import lietorch
    g = torch.Generator().manual_seed(3)
    xi = torch.randn(64, 6, generator=g, dtype=torch.float64)
    xi[:8, 3:] *= 1e-5                                         # below both small-angle switches
    xi[8:16, 3:] *= 3.0 / xi[8:16, 3:].norm(dim=-1, keepdim=True)   # near pi
    P = fo.exp(xi.numpy())
    np.testing.assert_allclose(P, lietorch.SE3.exp(xi).data.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(fo.log(P), lietorch.SE3(torch.from_numpy(P)).log().numpy(), rtol=0, atol=1e-9)
    np.testing.assert_allclose(fo.log(P), xi.numpy(), rtol=0, atol=1e-9)
    Q = P.copy()
    Q[:, 3:] *= -1                                             # the same rotations with qw < 0
    np.testing.assert_allclose(fo.log(Q), xi.numpy(), rtol=0, atol=1e-9)


def test_bracket_before_first_keyframe_is_minus_one():
    t0, t1 = fo.bracket([2.0, 5.0], [1.0, 2.0, 6.0])
    assert t0.tolist() == [-1, 0, 1] and t1.tolist() == [0, 1, 1]
