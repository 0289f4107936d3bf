"""The drop-in PoseTrajectoryFiller on the device: the fill kernel against the float64 oracle and the lietorch
composition the reference runs, the hand-over rows against DepthVideo.__setitem__'s semantics, a replay of the
REFERENCE PoseTrajectoryFiller on the golden streams (tests/golden/trajectory_filler.npz), the real encoder's feature
maps, and the documented differences (the caller's images are not written; ValueErrors leave the video as it was)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import filler_oracle as fo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))
DEV = torch.device("cuda:0")
G = np.load(os.path.join(HERE, "golden", "trajectory_filler.npz"))


def _video(buffer, h8=6, w8=10):
    """the buffers the fill kernel touches, filled with sentinels so untouched rows can be checked"""
    g = torch.Generator().manual_seed(buffer)
    v = types.SimpleNamespace(
        timestamp=torch.full((buffer,), -5.0), poses=torch.randn(buffer, 7, generator=g),
        intrinsics=torch.full((buffer, 4), 3.0), disps=torch.full((buffer, h8, w8), 7.0),
        disps_sens=torch.full((buffer, h8, w8), 9.0))
    for k, t in vars(v).items():
        setattr(v, k, t.to(DEV))
    return v


def _random_poses(n, g, angle=None):
    """keyframe poses [n, 7]: each a random rotation of the previous one (angle rad if given) plus a translation"""
    from goslam_b200 import lietorch
    P = [torch.tensor([0.1, -0.2, 0.3, 0, 0, 0, 1.0], dtype=torch.float64)]
    for _ in range(n - 1):
        xi = torch.randn(6, generator=g, dtype=torch.float64) * 0.3
        if angle is not None:
            xi[3:] *= angle / xi[3:].norm()
        P.append(lietorch.SE3.exp(xi).mul(lietorch.SE3(P[-1])).data)
    P = torch.stack(P)
    flip = torch.rand(n, generator=g) < 0.5                     # store half of the quaternions with qw < 0
    P[flip, 3:] *= -1
    return P.float()


CASES = {
    "n1": dict(N=1, buffer=24, frames="after"),
    "buffer": dict(N=1000, buffer=1024, frames="mixed"),      # the count spans 4 x 256 threads, 32 warps each
    "near_pi": dict(N=6, buffer=24, frames="mixed", angle=np.pi - 2e-3),
    "tiny": dict(N=6, buffer=24, frames="mixed", angle=5e-5),
}


def _case(name):
    c = CASES[name]
    g = torch.Generator().manual_seed(len(name) * 7 + c["N"])
    N, M = c["N"], 16
    ts = torch.cumsum(1.0 + torch.floor(6.0 * torch.rand(N, generator=g)), 0) - 1.0   # uneven integer gaps
    if c["frames"] == "after":
        tt = ts[-1] + torch.arange(M, dtype=torch.float32) * 0.25
    else:
        on = ts[torch.randint(0, N, (5,), generator=g)]
        mid = ts[0] + (ts[-1] - ts[0]) * torch.rand(8, generator=g)
        tt = torch.cat([on, mid, ts[-1:] + torch.tensor([0.0, 1.0, 2.5])])
    return N, M, c["buffer"], ts.float(), _random_poses(N, g, c.get("angle")), tt.float()


def _shim(ts, poses, tt):
    """the reference's interpolation lines (src/trajectory_filler.py:42-55) with goslam_b200.lietorch on the GPU"""
    from goslam_b200.lietorch import SE3
    ts, tt = ts.to(DEV), tt.to(DEV)
    N = ts.shape[0]
    Ps = SE3(poses.to(DEV))
    t0 = torch.tensor([ts[ts <= t].shape[0] - 1 for t in tt.tolist()], device=DEV)
    t1 = torch.where(t0 < N - 1, t0 + 1, t0)
    dt = ts[t1] - ts[t0] + 1e-3
    dP = Ps[t1] * Ps[t0].inv()
    v = dP.log() / dt.unsqueeze(dim=-1)
    w = v * (tt - ts[t0]).unsqueeze(dim=-1)
    return (SE3.exp(w) * Ps[t0]).data


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("with_depth", [True, False])
def test_kernel_against_oracle_shim_and_setitem(name, with_depth):
    from goslam_b200.trajectory_filler import fill_interpolate
    N, M, buffer, ts, poses, tt = _case(name)
    v = _video(buffer)
    v.timestamp[:N], v.poses[:N] = ts.to(DEV), poses.to(DEV)
    before = {k: t.clone() for k, t in vars(v).items()}
    g = torch.Generator().manual_seed(5)
    intr = (50.0 + 100.0 * torch.rand(M, 4, generator=g)).to(DEV)
    depth = None
    if with_depth:
        depth = 0.5 + 3.0 * torch.rand(M, 48, 80, generator=g)
        depth[:, 3::16, 3::8] = 0.0
        depth[:, 11::32, 3::24] = -1.0
        depth = depth.to(DEV)
    t0, t1 = fill_interpolate(v, N, tt.to(DEV), intr, depth)
    r0, r1, want = fo.interpolate(ts.numpy(), poses.numpy(), tt.numpy())
    assert t0.dtype == torch.long and t0.tolist() == r0.tolist() and t1.tolist() == r1.tolist()
    got = v.poses[N:N + M].double().cpu().numpy()
    tol = fo.bound(ts.numpy(), poses.numpy(), tt.numpy(), 1e-5)
    np.testing.assert_array_less(np.abs(got - want).max(-1), tol)
    np.testing.assert_array_less(np.abs(got - _shim(ts, poses, tt).double().cpu().numpy()).max(-1), 2 * tol)
    # hand-over rows: DepthVideo.__setitem__ with (tt, ..., Gs, 1, depths, intrinsics / 8), bit for bit
    rows = slice(N, N + M)
    assert torch.equal(v.timestamp[rows], tt.to(DEV))
    assert torch.equal(v.intrinsics[rows], intr / 8.0)
    if with_depth:
        d = depth[..., 3::8, 3::8]
        sens = torch.where(d > 0, 1.0 / d, d)
        assert torch.equal(v.disps_sens[rows], sens) and torch.equal(v.disps[rows], sens)
    else:
        assert torch.equal(v.disps[rows], torch.ones_like(v.disps[rows]))
        assert torch.equal(v.disps_sens, before["disps_sens"])
    for k, t in vars(v).items():                                # nothing outside rows N..N+M moves
        assert torch.equal(t[:N], before[k][:N]) and torch.equal(t[N + M:], before[k][N + M:]), k


def test_kernel_never_synchronises():
    from goslam_b200.trajectory_filler import fill_interpolate
    N, M, buffer, ts, poses, tt = _case("buffer")
    v = _video(buffer)
    v.timestamp[:N], v.poses[:N] = ts.to(DEV), poses.to(DEV)
    tt, intr, depth = tt.to(DEV), torch.ones(M, 4, device=DEV), torch.ones(M, 48, 80, device=DEV)
    fill_interpolate(v, N, tt, intr, depth)                     # loads the library
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        fill_interpolate(v, N, tt, intr, depth)
        fill_interpolate(v, N, tt, intr, None)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------- golden replay
def _filler(kind, fnet=None):
    import filler_scenario as fs
    from goslam_b200.depth_video import DepthVideo
    from goslam_b200.trajectory_filler import PoseTrajectoryFiller
    from stub_update_op import update_op
    cfg, args = fs.cfg_and_args("cuda:0", stereo=kind == "stereo")
    video = DepthVideo(cfg, args)
    fs.fill_keyframes(video, stereo=kind == "stereo")
    filler = PoseTrajectoryFiller(types.SimpleNamespace(cnet=None, fnet=fnet, update=update_op), video, device="cuda:0")
    if fnet is None:
        from stub_fnet import features
        filler._feature_encoder = lambda x: features((x - filler.MEAN) / filler.STDV)
    return filler, video


@pytest.fixture(scope="module", params=["rgbd", "mono", "stereo"])
def replay(request):
    import filler_scenario as fs
    from goslam_b200 import factor_graph
    kind = request.param
    chunks, calls = [], []
    orig = factor_graph.FactorGraph.add_factors

    def spy(self, ii, jj, remove=False):
        if not calls:
            calls.append(self.video.poses[jj].cpu().numpy().copy())
        calls.append(ii.cpu().numpy().copy())
        out = orig(self, ii, jj, remove)
        if len(calls) == 3:
            chunks.append(dict(G=calls[0], t0=calls[1], t1=calls[2], ii=self.ii.cpu().numpy(), jj=self.jj.cpu().numpy()))
            calls.clear()
        return out
    factor_graph.FactorGraph.add_factors = spy
    try:
        filler, video = _filler(kind)
        traj = filler(fs.stream(kind))
    finally:
        factor_graph.FactorGraph.add_factors = orig
    return kind, chunks, traj, video


def test_replay_chunks(replay):
    import filler_scenario as fs
    kind, chunks, traj, video = replay
    assert len(chunks) == int(G[kind + "_chunks"])
    tt = np.array([s[0] for s in fs.stream(kind)], np.float32)
    for c, d in enumerate(chunks):
        for k in ("t0", "t1", "ii", "jj"):
            np.testing.assert_array_equal(d[k], G["%s_c%d_%s" % (kind, c, k)], err_msg="%s chunk %d %s" % (kind, c, k))
        tol = fo.bound(np.array(fs.KF_T, np.float32), fs.keyframe_poses().numpy(), tt[16 * c:16 * (c + 1)], 1e-5)
        np.testing.assert_array_less(np.abs(d["G"] - G["%s_c%d_G" % (kind, c)]).max(-1), 2 * tol)


def test_replay_trajectory(replay):
    """1e-4 of the largest pose component, as the factor-graph drop-in test; a frame after the last keyframe also
    carries the difference its interpolated start may have there (see filler_oracle.bound), which BA inherits"""
    import filler_scenario as fs
    kind, chunks, traj, video = replay
    want = G[kind + "_traj"]
    got = traj.data.cpu().numpy()
    assert got.shape == want.shape == (len(fs.stream(kind)), 7)
    tt = np.array([s[0] for s in fs.stream(kind)], np.float32)
    ts, kp = np.array(fs.KF_T, np.float32), fs.keyframe_poses().numpy()
    tol = 1e-4 * np.abs(want).max() + 2 * (fo.bound(ts, kp, tt, 0.0))
    err = np.abs(got.astype(np.float64) - want).max(-1)
    assert (err < tol).all(), "%s: per-frame error %s, bound %s" % (kind, np.array2string(err, precision=2),
                                                                   np.array2string(tol, precision=2))


def test_replay_rows(replay):
    import filler_scenario as fs
    kind, chunks, traj, video = replay
    assert video.counter.value == int(G[kind + "_counter"]) == len(fs.KF_T)
    N, M = len(fs.KF_T), len(chunks[-1]["t0"])
    rows = slice(N, N + M)
    for name in ("timestamp", "intrinsics", "disps_sens"):
        np.testing.assert_array_equal(getattr(video, name)[rows].cpu().numpy(), G["%s_last_%s" % (kind, name)], err_msg=name)
    d, wd = video.disps[rows].cpu().numpy(), G[kind + "_last_disps"]
    assert np.abs(d - wd).max() <= 1e-6 * np.abs(wd).max()
    assert np.array_equal(video.poses[rows].cpu().numpy(), traj.data[-M:].cpu().numpy())
    # the reference stores the chunk normalised in place (documented difference): ours holds the images as given
    img = video.images[rows, :, ::8, ::8].cpu()
    norm = ((img - fs.MEAN) / fs.STDV).numpy()
    assert np.abs(norm - G[kind + "_last_images"]).max() <= 1e-6
    fm, wf = video.fmaps[rows, :, ::8].float().cpu().numpy(), G[kind + "_last_fmaps"].astype(np.float32)
    assert np.abs(fm - wf).max() <= 2e-3 * np.abs(wf).max()
    if kind == "rgbd":
        last = fs.stream(kind)[-M:]
        assert torch.equal(video.depths_gt[rows].cpu(), torch.stack([s[2] for s in last]))


# ---------------------------------------------------------------------------------------------------- real encoder
def test_real_encoder_feature_maps():
    import filler_scenario as fs
    from goslam_b200.modules.extractor import BasicEncoder
    from oracle import encoder_oracle as eo
    torch.manual_seed(12)
    fnet = BasicEncoder(out_dim=128, norm_fn="instance").to(DEV)
    filler, video = _filler("stereo", fnet=fnet)
    items = fs.stream("stereo", device="cuda")[:5]
    filler(items)
    N = len(fs.KF_T)
    x = torch.stack([s[1] for s in items])                         # [5, 2, 3, H, W]
    mean, std = torch.tensor(eo.MEAN, device=DEV)[:, None, None], torch.tensor(eo.STDV, device=DEV)[:, None, None]
    with torch.autocast("cuda"):
        want = fnet((x - mean) / std)
    assert want.dtype == torch.float16 and torch.equal(video.fmaps[N:N + 5], want)
    sd = fnet.state_dict()
    flat = x.reshape(-1, 3, fs.H, fs.W)
    ref = eo.basic_encoder(sd, "instance", flat, eo.MEAN, eo.STDV)
    auto = eo.basic_encoder(sd, "instance", flat, eo.MEAN, eo.STDV, autocast=True)
    ok, ek, ea = eo.contract_ok(video.fmaps[N:N + 5].reshape(-1, 128, fs.HT8, fs.WD8), auto, ref)
    assert ok, (ek, ea)


# ---------------------------------------------------------------------------------------------------- documented differences
def _state(video):
    return {k: t.clone() for k, t in vars(video).items() if torch.is_tensor(t)}, video.counter.value


def _same(video, snap):
    tensors, counter = snap
    assert video.counter.value == counter
    for k, t in tensors.items():
        assert torch.equal(getattr(video, k), t), k


def test_cuda_stream_images_untouched():
    import filler_scenario as fs
    filler, video = _filler("rgbd")
    items = fs.stream("rgbd", device="cuda")[:20]
    keep = [(s[1].clone(), s[2].clone(), s[3].clone()) for s in items]
    traj = filler(items)
    assert traj.data.shape == (20, 7)
    for s, k in zip(items, keep):
        assert torch.equal(s[1], k[0]) and torch.equal(s[2], k[1]) and torch.equal(s[3], k[2])
    assert torch.equal(video.images[7:11], torch.stack([s[1][0] for s in items[16:]]))


def test_timestamp_before_first_keyframe_raises():
    import filler_scenario as fs
    filler, video = _filler("rgbd")
    video.timestamp[:len(fs.KF_T)] += 1.0                          # frame 0 now precedes keyframe 0
    snap = _state(video)
    with pytest.raises(ValueError, match="before the first keyframe"):
        filler(fs.stream("rgbd")[:16])
    _same(video, snap)


def test_chunk_beyond_buffer_raises():
    import filler_scenario as fs
    from goslam_b200.depth_video import DepthVideo
    from goslam_b200.trajectory_filler import PoseTrajectoryFiller
    from stub_update_op import update_op
    cfg, args = fs.cfg_and_args("cuda:0")
    cfg["tracking"]["buffer"] = 20                                 # 7 keyframes + 16 frames do not fit
    video = DepthVideo(cfg, args)
    fs.fill_keyframes(video)
    filler = PoseTrajectoryFiller(types.SimpleNamespace(cnet=None, fnet=None, update=update_op), video)
    snap = _state(video)
    with pytest.raises(ValueError, match="buffer"):
        filler(fs.stream("rgbd")[:16])
    _same(video, snap)
