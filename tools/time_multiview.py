"""Time one full MultiviewFilter.forward pass: the native mirror (goslam_b200.MultiviewFilter) against the twin of
the reference's forward running on this library's iproj / depth_filter (oracle/mvfilter_oracle.py, i.e. the
reference's path after goslam_b200.install()).  Replica (320x640) T = 50/100/200 and ScanNet (240x320) T = 200/400,
kernel_size 'inf' (the Replica config).  Each pass ends in a device synchronise (the mirror's, or the twin's host
copies), and CUDA events bracket it.  The two paths' committed buffers are compared at every size.

    python tools/time_multiview.py [--reps 5] [--out results.json]
"""
import argparse
import contextlib
import io
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools import measure  # noqa: E402
measure.require_cuda("time_multiview.py")

import torch  # noqa: E402

from test_gpu_multiview_filter import STATE, make_pair, seeded_scene, state, ulp_diff  # noqa: E402

HBM_TBPS = 3.35          # H100 SXM data sheet
# bytes per pixel the native pass needs: snapshot copy of disps (4 read + 4 write), mean (4), vote (4 read +
# 1 mask write), extend (4 read + 1 mask read + 1 mask write), commit (4 disps read + 1 mask read + 4 + 4 writes)
BYTES_PER_PX = 8 + 4 + 5 + 6 + 13


def time_pass(video, fn, T, reps):
    out = []
    for r in range(reps + 1):
        video.filtered_id.fill_(-1)
        video.counter.value = T
        with contextlib.redirect_stdout(io.StringIO()):
            ms = measure.cuda_time(fn, 1, warmup=0)["samples_ms"]
        if r:                               # the first pass warms up
            out += ms
    out.sort()
    return out[len(out) // 2], out[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    a = ap.parse_args()
    measure.emit({})
    rows = []
    for label, ht, wd, T in (("Replica", 320, 640, 50), ("Replica", 320, 640, 100), ("Replica", 320, 640, 200),
                             ("ScanNet", 240, 320, 200), ("ScanNet", 240, 320, 400)):
        f = round(0.8 * wd * 8) / 8.0
        intr = [f / 8, f / 8, (wd - 1) / 16.0, (ht - 1) / 16.0]
        vm, flt, vt, twin = make_pair(T, ht, wd, intr, "inf", 8)
        for v in (vm, vt):
            seeded_scene(v, T, 4242 + T)
        nat = time_pass(vm, flt.forward, T, a.reps)
        ref = time_pass(vt, twin.forward, T, a.reps)
        sm, st = state(vm), state(vt)
        same = all(torch.equal(sm[k].view(torch.uint8), st[k].view(torch.uint8))
                   for k in STATE if k != "update_priority")
        pri_ulp = ulp_diff(sm["update_priority"], st["update_priority"])
        nbytes = BYTES_PER_PX * T * ht * wd
        share = nbytes / (nat[0] * 1e-3) / (HBM_TBPS * 1e12)
        row = dict(scene=label, ht=ht, wd=wd, T=T, native_ms=nat[0], native_min_ms=nat[1], twin_ms=ref[0],
                   twin_min_ms=ref[1], speedup=ref[0] / nat[0], bytes=nbytes, hbm_share=share,
                   outputs_identical=same, priority_ulp=pri_ulp)
        rows.append(row)
        print("%-8s %3dx%3d T=%3d  native %8.3f ms (min %8.3f)  twin %9.2f ms (min %9.2f)  x%6.1f  "
              "%6.1f MB  %5.1f%% of %.2f TB/s  outputs identical %s (priority %d ulp)" % (
                  label, ht, wd, T, nat[0], nat[1], ref[0], ref[1], ref[0] / nat[0], nbytes / 1e6, 100 * share,
                  HBM_TBPS, same, pri_ulp), flush=True)
        del vm, vt, flt, twin
        torch.cuda.empty_cache()
    measure.emit(dict(reps=a.reps, rows=rows), a.out)
    if not all(r["outputs_identical"] and r["priority_ulp"] <= 2 for r in rows):
        raise SystemExit("native and twin outputs differ")


if __name__ == "__main__":
    main()
