"""Per-chunk time of the trajectory fill at the Replica shape (320 x 640 images, 40 x 80 feature maps, RGB-D,
16-frame chunks, 64 keyframes in a 512-frame video): goslam_b200.PoseTrajectoryFiller against the reference's
`__fill` body (src/trajectory_filler.py:29-76) composed from this library's FactorGraph, DepthVideo, BasicEncoder
and lietorch shim, on the same CUDA image stream and the same seeded DroidNet weights.  The drop-in's time is also
split into the encoder, the interpolation / hand-over and the 6 updates (each stage synchronised on its own, so the
three add up to a little more than the chunk).  Host clock around work that ends in a device synchronise, median of
--reps after a warm-up; the card's name and power limit are read in the same run.

    python tools/time_filler.py [--reps 10] [--out result.json]
"""
import argparse
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools import measure  # noqa: E402
measure.require_cuda("time_filler.py")

import numpy as np  # noqa: E402
import torch  # noqa: E402

from goslam_b200 import lietorch  # noqa: E402
from goslam_b200.depth_video import DepthVideo  # noqa: E402
from goslam_b200.droid_net import UpdateModule  # noqa: E402
from goslam_b200.factor_graph import FactorGraph  # noqa: E402
from goslam_b200.modules.extractor import BasicEncoder  # noqa: E402
from goslam_b200.trajectory_filler import PoseTrajectoryFiller, fill_interpolate  # noqa: E402

DEV = torch.device("cuda:0")
H, W, BUFFER, NUM_KF, KF_STEP, M = 320, 640, 512, 64, 5, 16


def seeded(module, seed):
    """every parameter U(-b, b), b = 1 / sqrt(fan_in), from one seeded generator in sorted-name order"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for _, p in sorted(module.named_parameters()):
            b = 1.0 / np.sqrt(p[0].numel() if p.dim() > 1 else max(1, p.numel()))
            p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * b)
    return module


def setup():
    g = torch.Generator().manual_seed(1)
    cfg = {"cam": {"H_out": H, "W_out": W}, "mode": "rgbd", "tracking": {"buffer": BUFFER}}
    video = DepthVideo(cfg, types.SimpleNamespace(device="cuda:0"))
    xi = 0.02 * torch.randn(NUM_KF, 6, generator=g, dtype=torch.float64).cumsum(0)
    video.timestamp[:NUM_KF] = (KF_STEP * torch.arange(NUM_KF)).float().to(DEV)
    video.poses[:NUM_KF] = lietorch.SE3.exp(xi).data.float().to(DEV)
    video.disps[:NUM_KF] = (0.3 + 0.4 * torch.rand(NUM_KF, H // 8, W // 8, generator=g)).to(DEV)
    video.intrinsics[:NUM_KF] = torch.tensor([600.0, 600.0, 319.5, 159.5]).to(DEV) / 8
    for name in ("fmaps", "nets", "inps"):
        buf = getattr(video, name)
        buf[:NUM_KF] = (0.5 * torch.randn((NUM_KF,) + tuple(buf.shape[1:]), generator=g)).half().to(DEV)
    video.counter.value = NUM_KF
    torch.manual_seed(11)
    net = types.SimpleNamespace(fnet=BasicEncoder(128, "instance").to(DEV), cnet=None,
                                update=seeded(UpdateModule(), 3).to(DEV))
    img = torch.rand(M, 1, 3, H, W, generator=g).to(DEV)
    depth = (0.5 + 3.0 * torch.rand(M, H, W, generator=g)).to(DEV)
    intr = torch.tensor([600.0, 600.0, 319.5, 159.5], device=DEV)
    t_first = KF_STEP * NUM_KF // 2 + 1
    chunk = [(t_first + k, img[k], depth[k], intr, None) for k in range(M)]
    return video, net, chunk


def reference_fill(video, net, MEAN, STDV, timestamps, images, depths, intrinsics):
    """src/trajectory_filler.py:29-76 line by line"""
    SE3 = lietorch.SE3
    tt = torch.tensor(timestamps, device=DEV)
    images = torch.stack(images, dim=0)
    depths = torch.stack(depths, dim=0)
    intrinsics = torch.stack(intrinsics, 0)
    inputs = images.to(DEV)
    N = video.counter.value
    M = len(timestamps)
    ts = video.timestamp[:N]
    Ps = SE3(video.poses[:N])
    t0 = torch.tensor([ts[ts <= t].shape[0] - 1 for t in timestamps])
    t1 = torch.where(t0 < N - 1, t0 + 1, t0)
    dt = ts[t1] - ts[t0] + 1e-3
    dP = Ps[t1] * Ps[t0].inv()
    v = dP.log() / dt.unsqueeze(dim=-1)
    w = v * (tt - ts[t0]).unsqueeze(dim=-1)
    Gs = SE3.exp(w) * Ps[t0]
    inputs = inputs.sub_(MEAN).div_(STDV)
    with torch.autocast("cuda"):
        fmap = net.fnet(inputs)
    video.counter.value += M
    video[N:N + M] = (tt, images[:, 0], Gs.data, 1, depths, intrinsics / 8.0, fmap)
    graph = FactorGraph(video, net.update)
    graph.add_factors(t0.cuda(), torch.arange(N, N + M).cuda())
    graph.add_factors(t1.cuda(), torch.arange(N, N + M).cuda())
    for _ in range(6):
        graph.update(N, N + M, motion_only=True)
    Gs = SE3(video.poses[N:N + M].clone())
    video.counter.value -= M
    return [Gs]


def wall(fn):
    """ms of one synchronised call"""
    return measure.host_time(fn, 1, 0)["median_ms"]


def split(filler, video, chunk):
    """the drop-in's chunk stage by stage (trajectory_filler.PoseTrajectoryFiller._fill)"""
    N = video.counter.value
    tt = torch.tensor([float(c[0]) for c in chunk], dtype=torch.float32).to(DEV)
    images = torch.stack([c[1] for c in chunk])
    depths = torch.stack([c[2] for c in chunk])
    intr = torch.stack([c[3] for c in chunk])

    def enc():
        video.fmaps[N:N + M] = filler._feature_encoder(images.reshape(M, 3, H, W)).view(M, 1, 128, H // 8, W // 8)

    def interp():
        out = fill_interpolate(video, N, tt, intr, depths)
        video.images[N:N + M] = images[:, 0]
        video.depths_gt[N:N + M] = depths
        return out

    def updates(t0, t1):
        graph = FactorGraph(video, filler.update, device="cuda:0")
        jj = torch.arange(N, N + M, device=DEV)
        graph.add_factors(t0, jj)
        graph.add_factors(t1, jj)
        for _ in range(6):
            graph.update(N, N + M, motion_only=True)

    video.counter.value += M
    t01 = []
    try:
        te = wall(enc)
        ti = wall(lambda: t01.extend(interp()))
        tu = wall(lambda: updates(*t01))
    finally:
        video.counter.value -= M
    return {"encoder": te, "interp_handover": ti, "updates": tu}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    video, net, chunk = setup()
    filler = PoseTrajectoryFiller(net, video, device="cuda:0")
    MEAN, STDV = filler.MEAN, filler.STDV

    def ours():
        return filler(chunk)

    def ref():
        return lietorch.cat(reference_fill(video, net, MEAN, STDV, [c[0] for c in chunk], [c[1] for c in chunk],
                                           [c[2] for c in chunk], [c[3] for c in chunk]), 0)
    for _ in range(2):                                                 # warm-up: module loads, allocator, weight packs
        ours(), ref(), split(filler, video, chunk)
    runs = {"dropin": [], "reference_body": []}
    parts = []
    for _ in range(a.reps):                                            # alternate the two so drift hits both
        runs["dropin"].append(wall(ours))
        runs["reference_body"].append(wall(ref))
        parts.append(split(filler, video, chunk))
    p_ours, p_ref = ours().data, ref().data
    med = {k: float(np.median(v)) for k, v in runs.items()}
    res = {"shape": [H, W, H // 8, W // 8], "chunk": M, "keyframes": NUM_KF,
           "ms_per_chunk": med, "dropin_split_ms": {k: float(np.median([p[k] for p in parts])) for k in parts[0]},
           "max_pose_diff": float((p_ours - p_ref).abs().max()), "reps": a.reps}
    print("per chunk: drop-in %.2f ms, reference body %.2f ms; split %s; |dpose| %.2e" % (
        med["dropin"], med["reference_body"], res["dropin_split_ms"], res["max_pose_diff"]), flush=True)
    measure.emit(res, a.out)


if __name__ == "__main__":
    main()
