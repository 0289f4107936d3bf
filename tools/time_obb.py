"""Device time of the scene bound of Mesher.update_param_from_mapping (goslam_b200.mesher) at the Replica shape (250
keyframes, 320x640) and the ScanNet shape (512 keyframes, 240x320) on the multiview filter's analytic scene: the point
selection, the hull (with its extremes, cull and quickhull kernels listed on their own), and the box.  CUDA events
around each call, median of --reps after a warm-up; per-kernel times from measure.kernel_times in a separate pass.
The cull pass reads the points once (24 B) and writes one flag byte per point: its rate is reported against the H100
SXM's 3.35 TB/s.  The card's name and power limit are read in the same run.

    python tools/time_obb.py [--reps 5] [--out result.json]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools import measure  # noqa: E402
measure.require_cuda("time_obb.py")

from goslam_b200 import mesher  # noqa: E402
from oracle import mvfilter_oracle as mv  # noqa: E402
from test_gpu_multiview_filter import make_video, seeded_scene  # noqa: E402

SHAPES = {"replica": (250, 320, 640), "scannet": (512, 240, 320)}
HBM = 3.35e12


KERNELS = ("extremes_kernel", "winners_kernel", "hull_kernel", "cull_kernel", "box_kernel", "DeviceSelect")


def timed(fn, reps):
    """fn's last result and the median ms per call"""
    out = []
    return out, measure.cuda_time(lambda: out.append(fn()), reps, warmup=0)["median_ms"]


def kernels(fn):
    us = measure.kernel_times(fn, match=KERNELS)
    return {k: sum(t for name, t in us.items() if k in name) / 1e3 for k in KERNELS if any(k in name for name in us)}


def run(name, reps):
    T, ht, wd = SHAPES[name]
    intr = [f / 8 for f in mv.full_intrinsics(ht, wd)]
    video = make_video(T, ht, wd, intr)
    seeded_scene(video, T, 11)
    mesher.mapping_points(video, T)                                    # warm-up
    sels, t_sel = timed(lambda: mesher.mapping_points(video, T), reps)
    sel = sels[-1]
    _, t_hull = timed(lambda: mesher.hull_vertices(sel), reps)
    _, t_obb = timed(lambda: mesher.oriented_box(sel, 0.1), reps)
    _, _, _, info = mesher._hull_run(sel, "hull")
    status, n_vert, n_surv, n_win = info.tolist()
    k = kernels(lambda: mesher.hull_vertices(sel))
    n = sel.shape[0]
    cull_ms = k.get("cull_kernel", float("nan"))
    rate = 25.0 * n / (cull_ms * 1e-3)
    return dict(shape=name, keyframes=T, ht=ht, wd=wd, points=n, survivors=n_surv, winners=n_win, hull_vertices=n_vert,
                selection_ms=t_sel, hull_ms=t_hull, hull_and_box_ms=t_obb, kernel_ms=k,
                cull_bytes_per_s=rate, cull_share_of_hbm=rate / HBM)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    measure.emit(dict(runs=[run(s, a.reps) for s in SHAPES]), a.out)


if __name__ == "__main__":
    main()
