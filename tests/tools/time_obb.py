"""Device time of the scene bound of Mesher.update_param_from_mapping (goslam_b200.mesher) at the Replica shape (250
keyframes, 320x640) and the ScanNet shape (512 keyframes, 240x320) on the multiview filter's analytic scene: the point
selection, the hull (with its extremes, cull and quickhull kernels listed on their own), and the box.  CUDA events
around each call, median of --reps after a warm-up; per-kernel times from torch.profiler in a separate pass.  The cull
pass reads the points once (24 B) and writes one flag byte per point: its rate is reported against the H100 SXM's
3.35 TB/s.  The card's name and power limit are read in the same run.

    python tests/tools/time_obb.py [--reps 5] [--out result.json]      (under tests/: it runs the oracle's scene)
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from goslam_b200 import mesher  # noqa: E402
from oracle import mvfilter_oracle as mv  # noqa: E402
from test_gpu_multiview_filter import make_video, seeded_scene  # noqa: E402
from time_mesh_cull import card  # noqa: E402

SHAPES = {"replica": (250, 320, 640), "scannet": (512, 240, 320)}
HBM = 3.35e12


def timed(fn, reps):
    out, ts = None, []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return out, sorted(ts)[len(ts) // 2]


def kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("extremes_kernel", "winners_kernel", "hull_kernel", "cull_kernel", "box_kernel", "DeviceSelect"):
            if k in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                out[k] = out.get(k, 0.0) + t / 1e3
    return out


def run(name, reps):
    T, ht, wd = SHAPES[name]
    intr = [f / 8 for f in mv.full_intrinsics(ht, wd)]
    video = make_video(T, ht, wd, intr)
    seeded_scene(video, T, 11)
    mesher.mapping_points(video, T)                                    # warm-up
    sel, t_sel = timed(lambda: mesher.mapping_points(video, T), reps)
    ids, t_hull = timed(lambda: mesher.hull_vertices(sel), reps)
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
    if not torch.cuda.is_available():
        raise SystemExit("time_obb.py needs a CUDA device")
    name, limit = card()
    res = dict(device=name, nvidia_smi=limit, runs=[run(s, a.reps) for s in SHAPES])
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
