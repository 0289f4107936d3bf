"""Graph-construction cost of Backend.dense_ba / loop_ba's edge selection at 48 x 64 feature maps (the 384 x 512 input
of the configs) for N = 64, 256 and 1024 keyframes:
  old   host meshgrid of the (t_start..t_end)^2 indices + DepthVideo.distance over every pair (index copy to the device,
        both directions) + graph.backend_edges -- the reference's structure on this library's kernels;
  new   droid_backends.frame_distance_grid over the band Backend.ba reads + graph.backend_edges (goslam_b200.Backend);
plus each path without its backend_edges, and backend_edges alone, so the selection kernel's share is visible, and
loop closure's selection (window 25, loop mode) the same two ways.  Both selections must return the same edges.
Host clock around work that ends in a device synchronise, old and new alternated, median of --reps after warm-up;
the card's name and power limit are read in the same run.  Thresholds are the go_slam.yaml backend values.

    python tools/time_backend.py [--reps 20] [--sizes 64 256 1024] [--out result.json]
"""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools import measure  # noqa: E402
measure.require_cuda("time_backend.py")

import numpy as np  # noqa: E402
import torch  # noqa: E402

from goslam_b200 import droid_backends, graph as graph_ops, synthetic  # noqa: E402
from goslam_b200.depth_video import DepthVideo  # noqa: E402

DEV = "cuda:0"
HT8, WD8 = 48, 64
BETA = 0.75
DENSE = dict(radius=1, nms=5, thresh=25.0)
LOOP = dict(radius=1, nms=12, thresh=25.0, window=25)


def make_video(n):
    cfg = {"cam": {"H_out": 8 * HT8, "W_out": 8 * WD8}, "mode": "rgbd", "tracking": {"buffer": n}}
    video = DepthVideo(cfg, types.SimpleNamespace(device=DEV))
    g = torch.Generator().manual_seed(n)
    video.poses[:n] = synthetic.make_poses(n, g, trans_sigma=0.03, rot_sigma=0.01).to(DEV)
    low = torch.rand(n, 1, 6, 8, generator=g)
    video.disps[:n] = (0.3 + 0.6 * torch.nn.functional.interpolate(low, size=(HT8, WD8), mode="bilinear",
                                                                   align_corners=True)[:, 0]).to(DEV)
    video.intrinsics[:n] = torch.tensor([0.9 * WD8, 0.9 * WD8, WD8 / 2.0, HT8 / 2.0]).to(DEV)
    video.counter.value = n
    return video


def old_distance(video, r0, t, c0):
    ii, jj = torch.meshgrid(torch.arange(r0, t), torch.arange(c0, t), indexing="ij")
    return video.distance(ii.reshape(-1), jj.reshape(-1), beta=BETA)


def new_distance(video, r0, t, c0, k):
    v = video
    return droid_backends.frame_distance_grid(v.poses, v.disps, v.intrinsics[0], r0, t, c0, t, k, BETA)


def select(d, n, p, loop):
    t_start_loop = n - p["window"] if loop else None
    maxf = 8 * p["window"] if loop else (p["radius"] + 2) * 2 * n
    return graph_ops.backend_edges(d.reshape(-1), 0, n, p["radius"], p["nms"], p["thresh"], maxf, False,
                                   t_start_loop=t_start_loop, loop=loop)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", type=int, nargs="+", default=[64, 256, 1024])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"feature_map": [HT8, WD8], "reps": a.reps, "rows": []}
    for n in a.sizes:
        video = make_video(n)
        for mode, p, loop in (("dense", DENSE, False), ("loop", LOOP, True)):
            r0 = n - p["window"] if loop else 0
            k = 2 - p["radius"] if loop else -p["radius"]
            paths = {
                "old": lambda: select(old_distance(video, r0, n, 0), n, p, loop),
                "new": lambda: select(new_distance(video, r0, n, 0, k), n, p, loop),
                "old_distance": lambda: old_distance(video, r0, n, 0),
                "new_distance": lambda: new_distance(video, r0, n, 0, k),
            }
            d_full = old_distance(video, r0, n, 0)
            paths["backend_edges"] = lambda: select(d_full, n, p, loop)
            e_old, e_new = paths["old"](), paths["new"]()
            same = (e_old is None and e_new is None) or (e_old is not None and e_new is not None and all(
                torch.equal(x, y) for x, y in zip(e_old, e_new)))
            assert same, (n, mode)
            for fn in paths.values():                         # warm-up
                fn()
            times = {name: [] for name in paths}
            for _ in range(a.reps):
                for name, fn in paths.items():
                    times[name] += measure.host_time(fn, 1, 0)["samples_ms"]
            row = {"n": n, "mode": mode, "edges": 0 if e_new is None else int(e_new[0].numel()),
                   "pairs_old": (n - r0) * n, "pairs_new": int(torch.isfinite(new_distance(video, r0, n, 0, k)).sum()),
                   "index_bytes_old": 2 * 8 * (n - r0) * n}
            for name, ts in times.items():
                row[name + "_ms"] = round(float(np.median(ts)), 4)
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    measure.emit(res, a.out)


if __name__ == "__main__":
    main()
