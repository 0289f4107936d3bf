"""Loop closure and global BA on the device: the banded distance grid, goslam_b200.Backend's edge selection,
FactorGraph.adopt_edges under loop_ba, and the Frontend / Backend scenario against the reference classes
(tests/golden/frontend.npz, written by tests/golden/make_golden_frontend.py).

  * frame_distance_grid equals frame_distance_bidirectional bit for bit on every entry of its band and is +inf
    elsewhere, for dense and loop bands, offset row / column ranges, long videos and frames behind each other;
  * Backend.ba hands add_factors exactly graph.backend_edges of the full video.distance grid;
  * loop_ba leaves the local graph untouched and optimises its edges followed by the selected ones;
  * the scenario's edge lists, ages, counters, keyframe decisions and return values match exactly, its state within
    1e-4 of each field's largest magnitude (as tests/test_gpu_dropin.py)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))
sys.path.insert(0, HERE)

DEV = "cuda:0"


def video_tensors(n, ht, wd, seed, spread=0.05):
    from goslam_b200 import synthetic
    g = torch.Generator().manual_seed(seed)
    poses = synthetic.make_poses(n, g, trans_sigma=spread, rot_sigma=0.02)
    low = torch.rand(n, 1, 4, 6, generator=g)
    disps = 0.3 + 0.6 * torch.nn.functional.interpolate(low, size=(ht, wd), mode="bilinear", align_corners=True)[:, 0]
    intr = torch.tensor([0.9 * wd, 0.9 * wd, wd / 2.0 - 0.3, ht / 2.0 + 0.2])
    return poses.to(DEV).contiguous(), disps.to(DEV).contiguous(), intr.to(DEV)


def reference_grid(poses, disps, intr, r0, r1, c0, c1, beta):
    from goslam_b200 import droid_backends
    ii, jj = torch.meshgrid(torch.arange(r0, r1), torch.arange(c0, c1), indexing="ij")
    d = droid_backends.frame_distance_bidirectional(poses, disps, intr, ii.reshape(-1).to(DEV).contiguous(),
                                                    jj.reshape(-1).to(DEV).contiguous(), beta)
    return d.reshape(r1 - r0, c1 - c0)


def check_grid(poses, disps, intr, r0, r1, c0, c1, k, beta):
    from goslam_b200 import droid_backends
    got = droid_backends.frame_distance_grid(poses, disps, intr, r0, r1, c0, c1, k, beta).cpu().numpy()
    want = reference_grid(poses, disps, intr, r0, r1, c0, c1, beta).cpu().numpy()
    i = np.arange(r0, r1)[:, None]
    j = np.arange(c0, c1)[None, :]
    band = (j - i) <= k
    assert got.shape == want.shape
    np.testing.assert_array_equal(got.view(np.uint32)[band], want.view(np.uint32)[band])
    assert np.all(np.isposinf(got[~band]))
    return got, band


GRID_CASES = [  # (n, ht, wd, r0, r1, c0, c1, k)
    (40, 16, 24, 0, 40, 0, 40, -2),            # dense, radius 2
    (40, 16, 24, 0, 40, 0, 40, 1),             # loop, radius 1: both orientations of |i - j| <= 1 in the band
    (40, 16, 24, 15, 40, 0, 40, 0),            # loop, radius 2, rows from t_start_loop
    (40, 16, 24, 25, 40, 3, 40, -1),           # r0 > 0 and c0 > 0
    (40, 16, 24, 3, 37, 9, 31, 5),             # ranges that cross the band's corners
    (40, 16, 24, 0, 40, 0, 40, -100),          # empty band: all +inf
    (40, 16, 24, 0, 40, 0, 40, 100),           # every pair
    (300, 16, 24, 0, 300, 0, 300, -1),
    (300, 16, 24, 275, 300, 0, 300, -1),
    (128, 48, 64, 0, 128, 0, 128, -2),
    (128, 48, 64, 100, 128, 5, 128, 1),
]


@pytest.mark.parametrize("case", GRID_CASES, ids=lambda c: "n%d_%dx%d_r%d-%d_c%d-%d_k%d" % c)
def test_grid_is_bidirectional_distance_bit_for_bit(case):
    n, ht, wd, r0, r1, c0, c1, k = case
    poses, disps, intr = video_tensors(n, ht, wd, seed=n + ht + k + r0)
    _, band = check_grid(poses, disps, intr, r0, r1, c0, c1, k, 0.75)
    if -100 < k < 100:
        assert band.any() and not band.all()


@pytest.mark.parametrize("name", ["rig_37x45", "strip_7x45", "many_60x80"])
def test_grid_behind_the_camera(name):
    """the crafted rigs of tests/test_features_cases.py: frames facing away, points behind, at infinity, tiny and
    close; pairs with too few valid pixels take the 1000 branch"""
    from test_features_cases import reproject_case
    c = reproject_case(name)
    poses = torch.from_numpy(c["poses"]).to(DEV).contiguous()
    disps = torch.from_numpy(c["disps"]).to(DEV).contiguous()
    intr = torch.from_numpy(c["intrinsics"][0]).to(DEV).contiguous()
    n = poses.shape[0]
    got, band = check_grid(poses, disps, intr, 0, n, 0, n, 0, 0.3)
    got2, _ = check_grid(poses, disps, intr, 1, n, 2, n, 3, 0.75)
    assert np.any(got[band] == 1000.0) or np.any(got2 == 1000.0)


def test_grid_reads_a_pose_snapshot():
    """a pose write issued on the same stream after the call does not reach its result"""
    from goslam_b200 import droid_backends
    poses, disps, intr = video_tensors(60, 16, 24, seed=3)
    want = reference_grid(poses, disps, intr, 0, 60, 0, 60, 0.75).clone()
    got = droid_backends.frame_distance_grid(poses, disps, intr, 0, 60, 0, 60, 0, 0.75)
    poses[:, :3] += 0.5                                       # queued behind the grid
    torch.cuda.synchronize()
    g, w = got.cpu().numpy(), want.cpu().numpy()
    band = (np.arange(60)[None, :] - np.arange(60)[:, None]) <= 0
    np.testing.assert_array_equal(g.view(np.uint32)[band], w.view(np.uint32)[band])


def test_grid_abi_codes(lib):
    import ctypes
    null = ctypes.c_void_p(None)
    assert lib.goslam_frame_distance_grid_workspace_bytes(0, 0, 0, 5) == 0
    assert lib.goslam_frame_distance_grid_workspace_bytes(0, 5, 3, 3) == 0
    assert lib.goslam_frame_distance_grid_workspace_bytes(-1, 5, 0, 5) == 0
    assert lib.goslam_frame_distance_grid_workspace_bytes(0, 5, 0, 9) >= 7 * 9 * 4
    g = lambda r0, r1, c0, c1, ht=4, wd=4, p=null, ws=null, nb=0: lib.goslam_frame_distance_grid(  # noqa: E731
        p, p, p, r0, r1, c0, c1, 0, ht, wd, 0.5, p, ws, nb, null)
    assert g(0, 0, 0, 5) == 0 and g(2, 2, 0, 0) == 0                 # empty ranges: no-op
    assert g(-1, 3, 0, 3) == -1 and g(0, 3, -2, 3) == -1 and g(3, 1, 0, 3) == -1 and g(0, 3, 3, 1) == -1
    assert g(0, 3, 0, 3, ht=0) == -1 and g(0, 3, 0, 3, wd=-1) == -1
    assert g(0, 3, 0, 3) == -1                                       # null tensors
    t = torch.zeros(64, device=DEV)
    p = ctypes.c_void_p(t.data_ptr())
    assert g(0, 3, 0, 3, p=p) == -3                                  # no workspace
    assert g(0, 3, 0, 3, p=p, ws=p, nb=8) == -3                      # workspace too small


# ----------------------------------------------------------------------------------------------- Backend
def make_video(n, seed, spread=0.04):
    import frontend_scenario as fs
    from goslam_b200.depth_video import DepthVideo
    cfg, args = fs.cfg_and_args(DEV)
    cfg = dict(cfg, tracking=dict(cfg["tracking"], buffer=n + 2))
    video = DepthVideo(cfg, args)
    poses, disps, intr = video_tensors(n, fs.HT8, fs.WD8, seed, spread)
    video.poses[:n] = poses
    video.disps[:n] = disps
    video.intrinsics[:n] = intr
    video.counter.value = n
    return video, cfg, args


class Recorder:
    def __init__(self):
        self.ii, self.es = [], None

    def add_factors(self, ii, jj, remove=False):
        self.es = np.stack([ii.cpu().numpy(), jj.cpu().numpy()], 1)

    def update_lowmem(self, **kw):
        pass

    def clear_edges(self):
        pass


@pytest.mark.parametrize("n", [40, 150])
@pytest.mark.parametrize("loop", [False, True], ids=["dense", "loop"])
def test_backend_selection_matches_full_grid(n, loop):
    from goslam_b200 import graph as graph_ops
    from goslam_b200.backend import Backend
    video, cfg, args = make_video(n, seed=n + int(loop))
    be = Backend(types.SimpleNamespace(update=None), video, args, cfg)
    radius, nms = (1, 1) if loop else (2, 2)
    t_start, tsl = (0, n - 25) if loop else (3, None)
    r0 = tsl if loop else t_start
    ii, jj = torch.meshgrid(torch.arange(r0, n), torch.arange(t_start, n), indexing="ij")
    d = video.distance(ii.reshape(-1), jj.reshape(-1), beta=be.beta)
    # a threshold inside the data, so that the selection has candidates beyond the local window
    far = (jj - ii).reshape(-1).to(DEV) <= -radius - 2
    thresh = float(torch.quantile(d[far], 0.5 if loop else 0.3))
    maxf = 8 * 25 if loop else 16 * n
    rec = Recorder()
    got = be.ba(t_start, n, 2, rec, nms, radius, thresh, maxf, t_start_loop=tsl, loop=loop)
    want = graph_ops.backend_edges(d, t_start, n, radius, nms, thresh, maxf, video.stereo, t_start_loop=tsl, loop=loop)
    assert want is not None and rec.es is not None
    want = torch.stack(want, 1).cpu().numpy()
    np.testing.assert_array_equal(rec.es, want)
    n_local = sum(2 * (i - max(i - radius, r0)) for i in range(r0, n))
    assert len(want) > n_local                                        # candidates beyond the local window were taken
    assert got == 0 and video.dirty[t_start:n].all()                  # len(Recorder.ii) is what ba returns


def test_loop_ba_leaves_local_graph_and_prepends_its_edges(monkeypatch):
    import frontend_scenario as fs
    from stub_update_op import update_op
    from goslam_b200.backend import Backend
    from goslam_b200.factor_graph import FactorGraph
    n = 14
    video, cfg, args = make_video(n, seed=11, spread=0.02)
    g = torch.Generator().manual_seed(2)
    video.fmaps[:n] = torch.randn(n, 1, 128, fs.HT8, fs.WD8, generator=g).half().to(DEV)
    video.nets[:n] = (0.5 * torch.randn(n, 128, fs.HT8, fs.WD8, generator=g)).half().to(DEV)
    video.inps[:n] = (0.5 * torch.randn(n, 128, fs.HT8, fs.WD8, generator=g)).half().to(DEV)
    local = FactorGraph(video, update_op, device=DEV, corr_impl="volume", max_factors=48, upsample=False)
    local.add_neighborhood_factors(n - 6, n, r=2)
    local.update(None, None, use_inactive=True)
    before = {k: getattr(local, k).clone() for k in ("ii", "jj", "age", "net", "target", "weight")}
    mirrors = {k: v.copy() for k, v in local._h.items()}
    seen = {}
    orig = FactorGraph.update_lowmem

    def spy(self, *a, **k):
        seen["ii"], seen["jj"] = self.ii.clone(), self.jj.clone()
        seen["h"] = (self._h["ii"].copy(), self._h["jj"].copy())
        return orig(self, *a, **k)
    monkeypatch.setattr(FactorGraph, "update_lowmem", spy)
    be = Backend(types.SimpleNamespace(update=update_op), video, args, cfg)
    m = before["ii"].numel()
    sel = be.select_edges(0, n, be.backend_loop_nms, be.backend_loop_radius, be.backend_loop_thresh,
                          8 * be.backend_loop_window - m, t_start_loop=max(0, n - be.backend_loop_window), loop=True)
    assert sel is not None
    old = set(zip(before["ii"].tolist(), before["jj"].tolist()))
    appended = [e for e in zip(sel[0].tolist(), sel[1].tolist()) if e not in old]
    n_kf, n_edges = be.loop_ba(t_start=0, t_end=n, steps=1, local_graph=local)
    assert n_kf == min(n, be.backend_loop_window) and n_edges == seen["ii"].numel()
    for k, v in before.items():
        assert torch.equal(getattr(local, k), v), k
    for k, v in mirrors.items():
        np.testing.assert_array_equal(local._h[k], v)
    assert torch.equal(seen["ii"][:m], before["ii"]) and torch.equal(seen["jj"][:m], before["jj"])
    np.testing.assert_array_equal(seen["h"][0], seen["ii"].cpu().numpy())
    np.testing.assert_array_equal(seen["h"][1], seen["jj"].cpu().numpy())
    # followed by the selection, less the edges the local graph already had
    assert list(zip(seen["ii"][m:].tolist(), seen["jj"][m:].tolist())) == appended and appended


def test_adopt_edges_from_a_foreign_graph():
    from goslam_b200.factor_graph import FactorGraph
    video, cfg, args = make_video(10, seed=4)
    other = types.SimpleNamespace(ii=torch.tensor([3, 4, 5], device=DEV), jj=torch.tensor([4, 3, 3], device=DEV),
                                  age=torch.tensor([1, 0, 2], device=DEV), net=None,
                                  target=torch.randn(1, 3, 16, 24, 2, device=DEV), weight=None)
    fg = FactorGraph(video, None, device=DEV, corr_impl="alt")
    fg.adopt_edges(other)
    np.testing.assert_array_equal(fg._h["ii"], [3, 4, 5])
    np.testing.assert_array_equal(fg._h["jj"], [4, 3, 3])
    assert fg.net is None and fg.weight.shape[1] == 0 and torch.equal(fg.target, other.target)
    assert fg.target.data_ptr() != other.target.data_ptr() and fg.ii.data_ptr() != other.ii.data_ptr()


# ----------------------------------------------------------------------------------------------- scenario
@pytest.fixture(scope="module")
def scenario():
    import frontend_scenario as fs
    from goslam_b200.depth_video import DepthVideo
    from goslam_b200.frontend import Frontend
    cfg, args = fs.cfg_and_args(DEV)
    video = DepthVideo(cfg, args)
    with torch.no_grad():
        got = fs.run(Frontend, video, DEV)
    want = np.load(os.path.join(HERE, "golden", "frontend.npz"))
    return got, want


N_CALLS = 15
INT_FIELDS = ("ii", "jj", "age", "ii_inac", "jj_inac", "ii_bad", "jj_bad", "t1", "counter", "last_loop_t", "removed",
              "loops")
FLOAT_FIELDS = ("poses", "disps", "target", "weight", "target_inac", "damping", "disps_up")


def rel_err(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    assert a.shape == b.shape
    return 0.0 if b.size == 0 else np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)


def test_scenario_covers_the_decisions(scenario):
    got, want = scenario
    assert int(got["n_calls"]) == int(want["n_calls"]) == N_CALLS
    assert sum(int(want["f%02d_removed" % c]) for c in range(N_CALLS)) >= 1
    assert sum(len(want["f%02d_loops" % c]) for c in range(N_CALLS)) >= 2
    np.testing.assert_array_equal(got["dense_ba"], want["dense_ba"])


@pytest.mark.parametrize("call", range(N_CALLS))
def test_scenario_decisions_and_edges_exact(scenario, call):
    got, want = scenario
    for f in INT_FIELDS:
        k = "f%02d_%s" % (call, f)
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)


@pytest.mark.parametrize("call", range(N_CALLS))
def test_scenario_state_within_1e4(scenario, call):
    got, want = scenario
    for f in FLOAT_FIELDS:
        k = "f%02d_%s" % (call, f)
        err = rel_err(got[k], want[k])
        assert err < 1e-4, "%s: relative error %.3e" % (k, err)


def test_scenario_after_dense_ba(scenario):
    got, want = scenario
    for k in ("final_poses", "final_disps"):
        err = rel_err(got[k], want[k])
        assert err < 1e-4, "%s: relative error %.3e" % (k, err)
    np.testing.assert_array_equal(got["final_dirty"], want["final_dirty"])
