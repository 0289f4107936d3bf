"""proximity-edge selection: device kernel vs the reference-shaped Python loops (oracle, CPU).  Device: host clock around
each call and its synchronise, median of 20 after 3 warm-up calls; oracle: one host-timed call.
usage: python tools/time_graph.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_graph.py")
import numpy as np  # noqa: E402
import torch  # noqa: E402
from goslam_b200 import graph  # noqa: E402
from oracle import graph_oracle  # noqa: E402

dev = torch.device("cuda:0")
rng = np.random.default_rng(5)
measure.emit({})
for name, c in [("frontend keyframe (t0=t-5, window 25)", dict(t0=45, t1=25, t=50, rad=2, nms=2, thresh=16.0, maxf=48, stereo=False, n_old=40)),
                ("initialisation (12 x 12)", dict(t0=0, t1=0, t=12, rad=2, nms=2, thresh=16.0, maxf=48, stereo=False, n_old=0)),
                ("global graph (200 x 200)", dict(t0=0, t1=0, t=200, rad=2, nms=2, thresh=20.0, maxf=1600, stereo=False, n_old=400))]:
    ilen, jlen = c["t"] - c["t0"], c["t"] - c["t1"]
    dist = (rng.random(ilen * jlen) * 60).astype(np.float32)
    old = rng.integers(0, c["t"], size=(c["n_old"], 2)).astype(np.int64)
    args = (c["t0"], c["t1"], c["t"], c["rad"], c["nms"], c["thresh"], c["maxf"], c["stereo"])
    want = []
    cpu = measure.host_time(lambda: want.append(graph_oracle.proximity_edges(dist, *args, old[:, 0], old[:, 1])), 1, 0)
    want = want[0]
    dd, io, jo = torch.from_numpy(dist).to(dev), torch.from_numpy(old[:, 0].copy()).to(dev), torch.from_numpy(old[:, 1].copy()).to(dev)
    gpu = measure.host_time(lambda: graph.proximity_edges(dd, *args, io, jo), 20, 3)
    ii, jj = graph.proximity_edges(dd, *args, io, jo)
    ok = np.array_equal(torch.stack([ii, jj], 1).cpu().numpy(), want)
    print("%-40s %4d edges  device %.3f ms (%.3f-%.3f, incl. the one host sync)  numpy loops on the host %.2f ms  %s" %
          (name, len(want), gpu["median_ms"], gpu["min_ms"], gpu["max_ms"], cpu["median_ms"],
           "identical" if ok else "MISMATCH"))
