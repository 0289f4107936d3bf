"""Time of the trajectory evaluation, goslam_b200.slam.ape (the Sim(3)-aligned translation APE of SLAM.terminate), at
n = 2 000, 6 000 (a TUM / Replica sequence) and 10^6 poses.  Each timed call is the whole `ape`: the f64 widening, the
library call and the one read of its result.  CUDA events around --reps calls after a warm-up, median per call; the
card's name and power limit are read in the same run.

    python tools/time_ape.py [--reps 20] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from goslam_b200 import slam  # noqa: E402

DEV = torch.device("cuda:0")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        out = "unknown (%s)" % e
    return torch.cuda.get_device_name(0), out


def inputs(n, seed):
    """a smooth reference trajectory (identity rotations) and a rotated, scaled, noisy f32 estimate of it"""
    rng = np.random.default_rng(seed)
    s = np.linspace(0.0, 4.0 * np.pi, n)
    y = np.stack([np.cos(s), np.sin(0.7 * s), 0.5 * np.sin(0.3 * s)], 1) + [1.0, -2.0, 0.5]
    R, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    x = 0.7 * y @ R.T + rng.normal(size=(n, 3)) * 0.01
    ref = np.tile(np.eye(4), (n, 1, 1))
    ref[:, :3, 3] = y
    return torch.from_numpy(ref).to(DEV), torch.from_numpy(x).float().to(DEV)   # the estimate is f32, as in terminate


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    name, smi = card()
    print("card: %s | %s" % (name, smi))
    rows = []
    for n in (2000, 6000, 10 ** 6):
        ref, est = inputs(n, n)
        for _ in range(3):
            slam.ape(ref, est)
        ms = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            slam.ape(ref, est)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        rows.append({"n": n, "median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms))})
        print("n = %8d  ape %.3f ms (min %.3f, max %.3f)" % (n, rows[-1]["median_ms"], rows[-1]["min_ms"],
                                                                rows[-1]["max_ms"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "nvidia_smi": smi, "reps": args.reps, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
