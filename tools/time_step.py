"""in-stream CUDA-event timing of each phase of the config-2 update step: 5 samples of 50 back-to-back calls."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_step.py")
import torch  # noqa: E402
import bench  # noqa: E402
from goslam_b200 import droid_backends  # noqa: E402
from goslam_b200.modules.corr import fmaps_to_kmajor  # noqa: E402

dev = torch.device("cuda:0")
sc = bench.make_window(43)
win = bench.Window(sc, dev)
d = win.d
ii, jj = d["ii"], d["jj"]


def t(fn):
    r = measure.cuda_time(fn, reps=5, warmup=5, batch=50)
    return "%8.1f us (%.1f-%.1f)" % (1e3 * r["median_ms"], 1e3 * r["min_ms"], 1e3 * r["max_ms"])


km = fmaps_to_kmajor(d["fmaps"][:bench.NUM_KF])
corr = win.build(km)
coords, _ = droid_backends.reproject(d["poses"], d["disps"], d["intrinsics"], ii, jj, want_valid=False)


def ba(iters, motion_only=False):
    d["poses"].copy_(win.poses0); d["disps"].copy_(win.disps0)
    droid_backends.ba(d["poses"], d["disps"], d["intrinsics"][0], d["disps_sens"], d["targets"], d["weights"],
                      d["eta"], ii, jj, 1, bench.NUM_KF, iters, 1e-4, 0.1, motion_only)


measure.emit({})
print("kmajor(8 frames)      %s" % t(lambda: fmaps_to_kmajor(d["fmaps"][:bench.NUM_KF])))
print("corr build (36 edges) %s" % t(lambda: win.build(km)))
print("reproject             %s" % t(lambda: droid_backends.reproject(d["poses"], d["disps"], d["intrinsics"], ii, jj, want_valid=False)))
print("lookup (4 levels)     %s" % t(lambda: win.corr(coords)))
print("state reset (2 copies)%s" % t(lambda: (d["poses"].copy_(win.poses0), d["disps"].copy_(win.disps0))))
for it in (1, 2, 3):
    print("ba iters=%d            %s" % (it, t(lambda: ba(it))))
print("ba motion_only it=3   %s" % t(lambda: ba(3, True)))
print("frame_distance 64 prs %s" % t(lambda: droid_backends.frame_distance(d["poses"], d["disps"], d["intrinsics"][0].contiguous(), ii.repeat(2)[:64].contiguous(), jj.repeat(2)[:64].contiguous(), 0.3)))
print("full step             %s" % t(win.step))
