"""Pins the APE oracle (oracle/ape_oracle.py), the restatement of evo's Sim(3)-aligned translation APE that the device
is tested against: exact recovery of a known Sim(3), the reflection case, the rank rule, the statistics, the row
selection and the text written to metrics_traj.txt."""
import numpy as np
import pytest

from oracle import ape_oracle as ao


def _sim3_case(rng, n, scale, offset):
    """x (estimate) and reference poses y = s R x + t exactly, for a random rotation"""
    x = ao.smooth_trajectory(n, rng, spread=2.0)
    R = ao.random_rotation(rng)
    t = np.asarray(offset, np.float64) * rng.uniform(0.5, 1.0, 3)
    y = scale * x @ R.T + t
    return x, ao.poses_from(y, rng), R, t


@pytest.mark.parametrize("scale", [1e-3, 1e-1, 1.0, 10.0, 1e3])
@pytest.mark.parametrize("offset", [0.0, 1.0, 1e3])
def test_recovers_known_sim3(scale, offset):
    rng = np.random.default_rng(int(scale * 1000) % 97 + int(offset))
    x, ref, R, t = _sim3_case(rng, 200, scale, [offset, -offset, 0.5 * offset])
    res = ao.ape(ref, x)
    # 1e-12, plus the rounding of the reference's coordinates relative to the spread they carry (a millimetre-sized
    # trajectory a kilometre away keeps only ~10 significant digits of its shape)
    tol = 1e-12 + 8 * ao.EPS * max(1.0, np.abs(ref[:, :3, 3]).max() / (scale * np.ptp(x, 0).max()))
    assert np.abs(res["r"] - R).max() < tol
    assert abs(res["c"] - scale) <= tol * scale
    assert np.abs(res["t"] - t).max() <= tol * max(1.0, np.abs(t).max())
    want = np.eye(4)
    want[:3, :3], want[:3, 3] = scale * R, t
    assert np.abs(res["sim3"] - want).max() <= tol * max(1.0, np.abs(want).max())
    # the aligned estimate lands on the reference: errors at the rounding level of the reference's coordinates
    assert res["stats"]["max"] <= tol * max(1.0, scale * 2.0 + np.abs(t).max())


def test_reflection_flips_the_last_axis():
    """the estimate is a mirror image of the reference: S33 = -1, and R stays a rotation"""
    rng = np.random.default_rng(5)
    x = ao.smooth_trajectory(100, rng)
    y = x * np.array([1.0, 1.0, -1.0])
    res = ao.ape(ao.poses_from(y, rng), x)
    u, _, v = np.linalg.svd((y - y.mean(0)).T @ (x - x.mean(0)))
    assert np.linalg.det(u) * np.linalg.det(v) < 0
    assert abs(np.linalg.det(res["r"]) - 1.0) < 1e-12
    assert res["stats"]["max"] > 1e-3             # a mirror image cannot be matched by a rotation
    # the scale uses trace(D S) = d1 + d2 - d3
    d = res["d"]
    xc = x - x.mean(0)
    assert abs(res["c"] - (d[0] + d[1] - d[2]) / ((xc * xc).sum() / len(x))) < 1e-12 * res["c"]


def test_planar_input_is_accepted():
    rng = np.random.default_rng(6)
    x = ao.smooth_trajectory(50, rng)
    x[:, 2] = 0.0
    R = ao.random_rotation(rng)
    y = 2.0 * x @ R.T + 1.0
    res = ao.ape(ao.poses_from(y, rng), x)
    assert res["d"][2] <= 1e-15 and np.abs(res["r"] - R).max() < 1e-12 and abs(res["c"] - 2.0) < 1e-12


@pytest.mark.parametrize("n", [1, 2])
def test_two_rows_or_fewer_are_degenerate(n):
    rng = np.random.default_rng(n)
    x = rng.normal(size=(n, 3)) * 100.0
    with pytest.raises(ValueError, match="Degenerate covariance rank, Umeyama alignment is not possible"):
        ao.ape(ao.poses_from(rng.normal(size=(n, 3)) * 100.0, rng), x)


def test_collinear_input_is_degenerate():
    rng = np.random.default_rng(7)
    x = np.zeros((40, 3))
    x[:, 0] = np.linspace(-3.0, 5.0, 40)
    y = ao.smooth_trajectory(40, rng)
    with pytest.raises(ValueError, match="Degenerate covariance rank"):
        ao.ape(ao.poses_from(y, rng), x)


def test_statistics_by_hand():
    odd = ao.statistics([3.0, 1.0, 2.0, 2.0, 7.0])          # odd n, a tie in the middle
    assert odd == {"rmse": np.sqrt(67.0 / 5), "mean": 3.0, "median": 2.0, "std": np.sqrt(22.0 / 5), "min": 1.0,
                   "max": 7.0, "sse": 67.0}
    even = ao.statistics([4.0, 1.0, 3.0, 0.5])              # even n: the mean of the two middle values
    assert even["median"] == 2.0 and even["min"] == 0.5 and even["max"] == 4.0
    assert even["mean"] == 2.125 and even["sse"] == 26.25
    assert even["std"] == np.sqrt(((4 - 2.125) ** 2 + (1 - 2.125) ** 2 + (3 - 2.125) ** 2 + (0.5 - 2.125) ** 2) / 4)
    tied = ao.statistics([1.5, 1.5, 1.5, 1.5])
    assert tied["median"] == 1.5 and tied["std"] == 0.0 and tied["rmse"] == 1.5


def test_nonfinite_reference_rows_are_skipped():
    rng = np.random.default_rng(8)
    x, ref, _, _ = _sim3_case(rng, 30, 2.0, [1.0, 2.0, 3.0])
    x = x + rng.normal(size=x.shape) * 1e-2
    bad = [0, 7, 8, 29]
    ref2 = ref.copy()
    ref2[0, 3, 3] = np.nan
    ref2[7, 0, 1] = np.inf
    ref2[8, 2, 0] = -np.inf
    ref2[29, 1, 3] = np.nan
    x2 = x.copy()
    x2[bad] = np.nan                                          # the estimate of a skipped row is never read
    res = ao.ape(ref2, x2)
    keep = np.ones(30, bool)
    keep[bad] = False
    assert np.array_equal(res["kept"], keep)
    want = ao.ape(ref[keep], x[keep])
    assert np.array_equal(res["errors"], want["errors"]) and res["stats"] == want["stats"]
    # +inf and -inf in one row sum to NaN: skipped as well
    ref3 = ref.copy()
    ref3[3, 0, 0], ref3[3, 1, 1] = np.inf, -np.inf
    assert not ao.keep_rows(ref3)[3]


def test_errors_raise():
    rng = np.random.default_rng(9)
    x, ref, _, _ = _sim3_case(rng, 10, 1.0, [0.0, 0.0, 0.0])
    nan_ref = ref.copy()
    nan_ref[:, 0, 0] = np.nan
    with pytest.raises(ValueError, match="no reference pose"):
        ao.ape(nan_ref, x)
    x[4, 1] = np.inf
    with pytest.raises(ValueError, match="not finite"):
        ao.ape(ref, x)


def test_pretty_str_text():
    stats = {"rmse": 0.25, "mean": 0.2, "median": 0.125, "std": 0.15, "min": 0.0, "max": 1.0 / 3.0, "sse": 12.5}
    assert ao.pretty_str(stats) == (
        "APE w.r.t. translation part (m)\n(with Sim(3) Umeyama alignment)\n\n"
        "       max\t0.333333\n"
        "      mean\t0.200000\n"
        "    median\t0.125000\n"
        "       min\t0.000000\n"
        "      rmse\t0.250000\n"
        "       sse\t12.500000\n"
        "       std\t0.150000\n")
