"""The trajectory evaluation on the device (goslam_b200.slam.ape, goslam_ape_sim3) against the numpy oracle
(oracle/ape_oracle.py), and the drop-in SLAM.terminate on stub objects.

Every returned number is within 1e-9 relative of the oracle's (1e-12 absolute for R), plus 64 ulps of the conditioning
of far-away trajectories: a millimetre-sized trajectory a kilometre from the origin keeps only ~10 significant digits
of its shape in any f64 arithmetic.  Distances also get sqrt(n) ulps of the largest reference coordinate.  The median, min and max equal the oracle's statistics of the device's own errors bit
for bit."""
import types

import numpy as np
import pytest
import torch

from goslam_b200 import lietorch, slam
from oracle import ape_oracle as ao

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _case(kind, n, seed):
    """(ref [n,4,4], est [n,3], conditioning) of a named case"""
    rng = np.random.default_rng(seed)
    spread, offset = 2.0, np.array([0.5, -1.0, 0.3])
    if kind == "far":
        spread, offset = 1e-3, np.array([1e3, -7e2, 4e2])
    y = ao.smooth_trajectory(n, rng, offset=offset, spread=spread)
    if n <= 5:
        y = offset + spread * rng.normal(size=(n, 3))
    if kind == "planar":
        y[:, 2] = offset[2]
    R, s = ao.random_rotation(rng), 10.0 ** rng.uniform(-1, 1)
    x = ((y - offset) / s) @ R + rng.normal(size=3)
    if kind == "reflection":
        x[:, 2] = -x[:, 2]
    x = x + rng.normal(size=x.shape) * 0.02 * np.ptp(x, 0).max()
    ref = ao.poses_from(y, rng)
    if kind == "nonfinite":
        for i, r, c, v in [(0, 3, 3, np.nan), (1, 0, 1, np.inf), (n // 2, 2, 0, -np.inf), (n // 2 + 1, 1, 3, np.nan),
                           (n - 1, 0, 0, np.inf)]:
            ref[i, r, c] = v
        x[n // 2] = np.nan                                   # a skipped row's estimate is never read
    cond = max(1.0, np.abs(y).max() / spread)
    return ref, x, cond


def _check(ref, x, cond):
    want = ao.ape(ref, x)
    got = slam.ape(torch.from_numpy(ref).to(DEV), torch.from_numpy(x).to(DEV))
    tol, tol_r = 1e-9 + 64 * ao.EPS * cond, 1e-12 + 64 * ao.EPS * cond
    # distances are differences of positions: they also carry the rounding of n-term sums of the reference's
    # coordinates, sqrt(n) ulps of the largest one
    m = int(want["kept"].sum())
    d_abs = 4 * np.sqrt(m) * ao.EPS * np.abs(ref[want["kept"]][:, :3, 3]).max()
    e = got.np_arrays["error_array"]
    assert e.shape == want["errors"].shape
    emax = want["errors"].max()
    assert np.abs(e - want["errors"]).max() <= tol * emax + d_abs
    c = want["c"]
    S = got.np_arrays["alignment_transformation_sim3"]
    assert abs(np.linalg.norm(S[0, :3]) - c) <= tol * c
    assert np.abs(S[:3, :3] / c - want["r"]).max() <= tol_r
    assert np.abs(S[:3, 3] - want["t"]).max() <= tol * max(1.0, np.abs(want["t"]).max())
    assert np.array_equal(S[3], [0.0, 0.0, 0.0, 1.0])
    assert np.abs(got.singular_values - want["d"]).max() <= tol * want["d"][0]
    for k in ("rmse", "mean", "std"):
        assert abs(got.stats[k] - want["stats"][k]) <= tol * abs(want["stats"][k]) + d_abs, k
    assert abs(got.stats["sse"] - want["stats"]["sse"]) <= tol * want["stats"]["sse"] + 2 * m * emax * d_abs
    own = ao.statistics(e)
    for k in ("median", "min", "max"):
        assert got.stats[k] == own[k], k
    return got, want


@pytest.mark.parametrize("n", [3, 4, 5, 1000, 6000, 10 ** 6])
def test_noisy_sim3_of_a_smooth_trajectory(n):
    _check(*_case("smooth", n, n))


@pytest.mark.parametrize("kind, n", [(k, n) for k in ("planar", "reflection", "far") for n in (5, 1000, 6000, 10 ** 6)]
                         + [("nonfinite", n) for n in (8, 1000, 6000, 10 ** 6)])
def test_cases(kind, n):
    got, want = _check(*_case(kind, n, 7 * n + len(kind)))
    if kind == "reflection" and n > 5:
        S = got.np_arrays["alignment_transformation_sim3"]
        assert np.linalg.det(S[:3, :3]) > 0                  # a rotation, not the mirror
    if kind == "nonfinite":
        assert len(got.np_arrays["error_array"]) == n - 5 == want["kept"].sum()


def test_float32_inputs_are_widened():
    ref, x, cond = _case("smooth", 1000, 3)
    ref32, x32 = ref.astype(np.float32), x.astype(np.float32)
    got = slam.ape(torch.from_numpy(ref32).to(DEV), torch.from_numpy(x32).to(DEV))
    want = ao.ape(ref32.astype(np.float64), x32.astype(np.float64))
    assert abs(got.stats["rmse"] - want["stats"]["rmse"]) <= 1e-9 * want["stats"]["rmse"]


def test_errors_raise_value_error():
    rng = np.random.default_rng(1)
    ref, x, _ = _case("smooth", 50, 2)
    bad = ref.copy()
    bad[:, 1, 2] = np.nan
    with pytest.raises(ValueError, match="no reference pose"):
        slam.ape(torch.from_numpy(bad).to(DEV), torch.from_numpy(x).to(DEV))
    with pytest.raises(ValueError, match="no reference pose"):
        slam.ape(torch.zeros(0, 4, 4, device=DEV), torch.zeros(0, 3, device=DEV))
    xb = x.copy()
    xb[17, 0] = np.inf
    with pytest.raises(ValueError, match="not finite"):
        slam.ape(torch.from_numpy(ref).to(DEV), torch.from_numpy(xb).to(DEV))
    for n in (1, 2):
        with pytest.raises(ValueError, match="^Degenerate covariance rank, Umeyama alignment is not possible$"):
            slam.ape(torch.from_numpy(ref[:n]).to(DEV), torch.from_numpy(x[:n]).to(DEV))
    line = np.zeros((40, 3))
    line[:, 1] = np.linspace(-2.0, 3.0, 40) + rng.normal(size=40) * 0.1
    with pytest.raises(ValueError, match="Degenerate covariance rank"):
        slam.ape(torch.from_numpy(ref[:40]).to(DEV), torch.from_numpy(line).to(DEV))
    with pytest.raises(ValueError, match="Degenerate covariance rank"):
        ao.ape(ref[:40], line)


def test_two_runs_are_bit_identical():
    for n in (6000, 10 ** 6):
        ref, x, _ = _case("nonfinite", n, 11)
        r, e = torch.from_numpy(ref).to(DEV), torch.from_numpy(x).to(DEV)
        a, b = slam.ape(r, e), slam.ape(r, e)
        assert a.stats == b.stats
        assert np.array_equal(a.np_arrays["alignment_transformation_sim3"], b.np_arrays["alignment_transformation_sim3"])
        assert torch.equal(a.errors, b.errors)


# ---- the drop-in terminate -----------------------------------------------------------------------------------------
def _w2c(n, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(n, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    s = torch.linspace(0, 6.0, n)
    t = torch.stack([torch.cos(s), torch.sin(0.8 * s), 0.3 * s], 1) + 0.01 * torch.randn(n, 3, generator=g)
    return lietorch.SE3(torch.cat([t, q], 1).to(DEV))


class Mesher:
    def __init__(self):
        self.calls = []

    def __call__(self, **kw):
        self.calls.append(kw)


def _stub(tmp_path, n, meshing=1, only_tracking=False):
    comp = torch.tensor([[0.2, -0.1, 0.4, 0.1, 0.2, -0.3, 0.9]])
    comp[0, 3:] /= comp[0, 3:].norm()
    traj = _w2c(n, 5)
    return types.SimpleNamespace(
        optimizing_finished=1, num_running_thread=torch.ones(1, dtype=torch.int), tracking_finished=1,
        output=str(tmp_path), mapping_net=torch.nn.Linear(2, 2), net=torch.nn.Linear(3, 1),
        video=types.SimpleNamespace(timestamp=torch.arange(4.0), pose_compensate=comp.to(DEV)),
        traj_filler=lambda stream: lietorch.SE3(traj.data.clone()), meshing_finished=meshing,
        only_tracking=only_tracking, mesher=Mesher(), _traj=traj, _comp=comp)


def _chain(self):
    w2w = lietorch.SE3(self._comp.to(DEV))
    return w2w * self._traj.inv()


class Stream:
    def __init__(self, n, poses, image_timestamps=None):
        self.input_folder, self.poses, self.image_timestamps, self._n = "stub/scene", poses, image_timestamps, n

    def __len__(self):
        return self._n


def test_terminate_writes_the_oracle_text_and_hands_over_sim3(tmp_path, capsys):
    n = 300
    self = _stub(tmp_path, n)
    est = _chain(self)
    rng = np.random.default_rng(2)
    x = est.data[:, :3].double().cpu().numpy()
    y = (2.5 * x @ ao.random_rotation(rng).T + [1.0, -2.0, 0.5]) + rng.normal(size=(n, 3)) * 0.01
    poses = list(ao.poses_from(y, rng))
    poses[0] = poses[0].copy()
    poses[0][3, 3] = np.nan
    poses[150] = poses[150].copy()
    poses[150][1, 2] = np.inf
    stream = Stream(n, poses)
    for _ in range(2):
        slam.terminate(self, 0, stream)
    out = capsys.readouterr().out
    assert "Results for stub/scene" in out and "skipping 0th pose!" in out and "skipping 150th pose!" in out
    assert np.array_equal(np.load(tmp_path / "checkpoints" / "est_poses.npy"), est.matrix().data.cpu().numpy())
    assert (tmp_path / "checkpoints" / "go.ckpt").exists()
    want = ao.ape(np.stack(poses), x)
    text = (tmp_path / "metrics_traj.txt").read_text()
    assert text == 2 * ao.pretty_str(want["stats"])
    assert len(self.mesher.calls) == 2
    kw = self.mesher.calls[0]
    assert kw["the_end"] is True and torch.equal(kw["estimate_c2w_list"], est.matrix().data.cpu())
    keep = want["kept"]
    assert torch.equal(kw["gt_c2w_list"], torch.from_numpy(np.stack(poses)[keep]))
    assert np.abs(kw["trans_init"] - want["sim3"]).max() <= 1e-9 * np.abs(want["sim3"]).max()


@pytest.mark.parametrize("meshing, only_tracking", [(0, False), (1, True)])
def test_terminate_skips_the_mesher(tmp_path, meshing, only_tracking):
    n = 40
    self = _stub(tmp_path, n, meshing, only_tracking)
    rng = np.random.default_rng(3)
    y = ao.smooth_trajectory(n, rng)
    slam.terminate(self, 0, Stream(n, list(ao.poses_from(y, rng))))
    assert self.mesher.calls == [] and (tmp_path / "metrics_traj.txt").exists()


def test_terminate_without_ground_truth_writes_the_submission(tmp_path):
    n = 20
    self = _stub(tmp_path, n)
    stamps = [1403636579.763555 + 0.05 * i for i in range(n)]
    slam.terminate(self, 0, Stream(n, None, stamps))
    traj = _chain(self).data.cpu().numpy()
    want = "".join(f'{tm:.9f}' + "".join(f' {ps:.14f}' for ps in pos) + "\n" for tm, pos in zip(stamps, traj.tolist()))
    assert (tmp_path / "submission.txt").read_text() == want
    assert not (tmp_path / "metrics_traj.txt").exists()
    kw = self.mesher.calls[0]
    assert kw["trans_init"] is None and kw["gt_c2w_list"] is None
