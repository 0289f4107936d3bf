"""Time of the trajectory evaluation, goslam_b200.slam.ape (the Sim(3)-aligned translation APE of SLAM.terminate), at
n = 2 000, 6 000 (a TUM / Replica sequence) and 10^6 poses.  Each timed call is the whole `ape`: the f64 widening, the
library call and the one read of its result.  CUDA events around --reps calls after a warm-up, median per call; the
card's name and power limit are read in the same run.

    python tools/time_ape.py [--reps 20] [--out result.json]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools import measure  # noqa: E402
measure.require_cuda("time_ape.py")

import numpy as np  # noqa: E402
import torch  # noqa: E402

from goslam_b200 import slam  # noqa: E402

DEV = torch.device("cuda:0")


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
    rows = []
    for n in (2000, 6000, 10 ** 6):
        ref, est = inputs(n, n)
        t = measure.cuda_time(lambda: slam.ape(ref, est), args.reps)
        rows.append({"n": n, "median_ms": t["median_ms"], "min_ms": t["min_ms"], "max_ms": t["max_ms"]})
        print("n = %8d  ape %.3f ms (min %.3f, max %.3f)" % (n, t["median_ms"], t["min_ms"], t["max_ms"]))
    measure.emit({"reps": args.reps, "rows": rows}, args.out)


if __name__ == "__main__":
    main()
