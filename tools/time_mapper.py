"""Time one Mapper.__call__ (an init call and a steady-state call) against the reference's path on CUDA (the restated
schedule of oracle/mapping_oracle.py: get_mapping_item per list entry, build_rays per frame and torch.cat per
iteration), both training the bench.make_renderer net through this library's renderer.

Setup: Replica 320x640, 100 keyframes with ~70 % masks, the shipped mapping config (pixels 4400, window 22, iters 2).
Reports per call: ms from CUDA events around the whole call (median of --reps after a warm-up), and a split into
snapshot / ray batches / optimize_map from a second set of calls whose stages are each bracketed by synchronises;
launches and host synchronisations per iteration's batch build from a separate profiler run (measure.kernel_times);
the card's name and power limit.  One JSON object per line on stdout.

usage: python tools/time_mapper.py [--reps 5]
"""
import argparse
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_mapper.py")
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from goslam_b200 import lietorch, mapping  # noqa: E402
from goslam_b200.render import Renderer  # noqa: E402
from oracle import mapping_oracle as mo  # noqa: E402

DEV = torch.device("cuda:0")
N, H, W = 100, 320, 640
INTR = (320.0, 320.0, 319.5, 159.5)


def setup():
    video = mo.stub_video(N, H, W, DEV)
    g = torch.Generator().manual_seed(1)
    video.pose_compensate[0] = mo.random_pose(g, 0.3)
    video.bound[0] = torch.tensor([[-2.0, 2.0]] * 3)
    mo.fill_frames(video, range(N), g, density=0.7, zero_frac=0.0, trans=0.4)
    net = bench.make_renderer(DEV, 43)[0]
    rcfg = {'rendering': {'N_samples': 24, 'N_surface': 48, 'lindisp': False, 'perturb': 1.0}}
    slam = mo.stub_slam(video, net, Renderer(rcfg, None, types.SimpleNamespace(H=H, W=W, fx=INTR[0], fy=INTR[1],
                                                                                cx=INTR[2], cy=INTR[3])),
                        INTR, tempfile.mkdtemp())
    slam.video.filtered_id[0] = N
    cfg = mo.mapping_cfg("cuda:0", 4400, 22, 2)
    ours = mapping.Mapper(cfg, None, slam)
    ref = mo.MapperSchedule(cfg, slam, lietorch.SE3, lambda s, *a: mo.reference_optimize_map(s, *a),
                            optimizer=ours.optimizer)
    ref.record_draws = False
    return video, ours, ref


def prime(runner, kind):
    """state before an init call (nothing visited) or a steady-state call (last_visit = 90, 10 new keyframes)"""
    runner.init = kind == "init"
    runner.last_visit = 0 if kind == "init" else N - 10


class Stages:
    """host time of synchronised stages (each wrapped function is bracketed by torch.cuda.synchronize)"""

    def __init__(self):
        self.t = {}

    def wrap(self, owner, attr, key):
        fn = getattr(owner, attr)

        def timed(*a, **k):
            r = []
            self.t[key] = self.t.get(key, 0.0) + measure.host_time(lambda: r.append(fn(*a, **k)), 1, 0)["median_ms"]
            return r[0]
        setattr(owner, attr, timed)
        return fn


def time_call(runner, kind, reps):
    out = []
    for _ in range(reps):
        prime(runner, kind)
        out += measure.cuda_time(runner, 1, warmup=0)["samples_ms"]
    return float(np.median(out))


def split_call(runner, is_ours, kind, reps):
    st = Stages()
    if is_ours:
        saved = [(mapping, "snapshot_frames", st.wrap(mapping, "snapshot_frames", "snapshot")),
                 (mapping, "build_ray_batch", st.wrap(mapping, "build_ray_batch", "ray_batches")),
                 (type(runner), "optimize_map", st.wrap(type(runner), "optimize_map", "optimize_map"))]
    else:
        saved = [(mo, "mapping_item", st.wrap(mo, "mapping_item", "snapshot")),
                 (type(runner), "_batch", st.wrap(type(runner), "_batch", "ray_batches")),
                 (runner, "_optimize_map", st.wrap(runner, "_optimize_map", "optimize_map"))]
    try:
        for _ in range(reps):
            prime(runner, kind)
            runner()
    finally:
        for owner, attr, fn in saved:
            setattr(owner, attr, fn)
    return {k: round(v / reps, 3) for k, v in st.t.items()}


def profile_batch(video, ours, ref):
    """kernels and host synchronisations of one iteration's batch build (22 frames, 200 rays each)"""
    frames = list(range(N - 22, N))
    snap = mapping.snapshot_frames(video, frames, 1.0)
    items = {f: mo.mapping_item(video, f, DEV, 1.0, lietorch.SE3) for f in frames}
    ref.device = "cuda:0"
    res = {}

    # the closing synchronize and the profiler's own flush, counted once here and subtracted below
    overhead = len(measure.kernel_times(lambda: None).host_syncs)
    for label, fn in (("ours", lambda: mapping.build_ray_batch(snap, frames, 200, INTR)),
                      ("reference", lambda: ref._batch(frames, 200, items))):
        fn()
        torch.cuda.synchronize()
        k = measure.kernel_times(fn)
        kernels = {n: c for n, c in k.launches.items() if "emcpy" not in n and "emset" not in n}
        res[label] = {"kernels": round(sum(kernels.values())), "host_syncs": len(k.host_syncs) - overhead,
                      "sync_calls": sorted(set(k.host_syncs)),
                      "copies": round(sum(c for n, c in k.launches.items() if "emcpy" in n)),
                      "kernel_names": sorted(set(n[:60] for n in kernels))}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    video, ours, ref = setup()
    for r in (ref, ours):                      # warm-up: library load, allocator, every shape
        for kind in ("init", "steady"):
            np.random.seed(0)
            prime(r, kind)
            r()
    torch.cuda.synchronize()
    for kind in ("init", "steady"):
        row = {"call": kind}
        for label, r in (("reference", ref), ("ours", ours)):
            np.random.seed(1)
            torch.manual_seed(1)
            row[label + "_ms"] = round(time_call(r, kind, a.reps), 2)
        for label, r in (("reference", ref), ("ours", ours)):
            np.random.seed(1)
            row[label + "_split_ms"] = split_call(r, r is ours, kind, max(1, a.reps // 2))
        row["speedup"] = round(row["reference_ms"] / row["ours_ms"], 2)
        measure.emit(row)
    measure.emit({"per_iteration_batch_build": profile_batch(video, ours, ref)})


if __name__ == "__main__":
    main()
