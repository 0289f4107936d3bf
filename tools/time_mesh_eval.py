"""Time the reconstruction evaluation (align_mesh / eval_mesh) on the device, and the CPU path for context.

A res-512 network mesh of the golden scene (net.extract_mesh(512, 0.0) on the synthetic weights) against a copy moved
by 0.3 degree and 4 mm.  Device stages by CUDA events after warm-up (median of --reps):
  sample       sample_surface of N3d points on each mesh
  metrics      both metric directions: grid index over one sample set + nearest of the other, twice
  icp_index    the ICP target's index (cells >= 0.1)
  icp_iter     one ICP iteration (max_iteration = 1 minus max_iteration = 0, same prebuilt index)
  align_mesh   the whole drop-in align_mesh (host vertices in, T out), default criteria
CPU (this host): cKDTree build + query for both metric directions, and the numpy ICP oracle (index build and one
iteration).  The card's name and power limit are read in the same run.

    python tools/time_mesh_eval.py [--n3d 200000] [--reps 5] [--cpu-icp] [--out result.json]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools import measure  # noqa: E402
measure.require_cuda("time_mesh_eval.py")

import numpy as np  # noqa: E402
import torch  # noqa: E402

from goslam_b200 import mesher, neus, synthetic  # noqa: E402
from oracle import mesh_eval_oracle as meo  # noqa: E402
from oracle import neus_oracle as no  # noqa: E402


def res512_mesh():
    metas, tot = no.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [tot * 2]
    g = np.load(os.path.join(ROOT, "tests", "golden", "mesh.npz"))
    w = synthetic.make_neus_weights(seed=int(g["weights_seed"]), total_grid_params=tot * 2,
                                    layout=(offs, [m["res"] for m in metas]))
    net = neus.InstantNeuS(synthetic.NEUS_CFG, g["bound"].tolist())
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to("cuda:0")
    net.update_bound(torch.from_numpy(g["rt_bound"]))
    out = net.extract_mesh(512, 0.0, color=False)
    return out[0], out[1]


def cuda_ms(fn, reps):
    return measure.cuda_time(fn, reps, warmup=2)["median_ms"]


def host_s(fn, reps=1):
    return measure.host_time(fn, reps, warmup=0)["median_ms"] / 1e3


class StandIn:
    def __init__(self, v, f):
        self.vertices, self.faces = v, f

    def apply_transform(self, M):
        h = np.c_[self.vertices, np.ones(len(self.vertices))] @ np.asarray(M).T
        self.vertices = h[:, :3] / h[:, 3:]
        return self


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n3d", type=int, default=200000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-icp", action="store_true", help="also time the numpy ICP oracle (minutes at res 512)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    v, f = res512_mesh()
    M = meo.rigid([0.4, -0.7, 0.2], np.deg2rad(0.3), [0.004, -0.003, 0.002])
    hv, hf = v.cpu().numpy(), f.cpu().numpy()
    hd = meo.transform(hv, M)
    d = torch.from_numpy(hd).to(dev)
    res = {"verts": int(v.shape[0]), "faces": int(f.shape[0]), "n3d": a.n3d}
    gen = torch.Generator(dev).manual_seed(0)
    res["sample_ms"] = cuda_ms(lambda: (mesher.sample_surface(v, f, a.n3d, gen), mesher.sample_surface(d, f, a.n3d, gen)),
                               a.reps)
    est_pc, gt_pc = mesher.sample_surface(v, f, a.n3d, gen), mesher.sample_surface(d, f, a.n3d, gen)
    res["metrics_ms"] = cuda_ms(lambda: (mesher.NNIndex(est_pc).query(gt_pc), mesher.NNIndex(gt_pc).query(est_pc)),
                                a.reps)
    res["icp_index_ms"] = cuda_ms(lambda: mesher.NNIndex(d, 0.1), a.reps)
    index = mesher.NNIndex(d, 0.1)
    t1 = cuda_ms(lambda: mesher.icp_point_to_point(v, index, 0.1, max_iteration=1), a.reps)
    t0 = cuda_ms(lambda: mesher.icp_point_to_point(v, index, 0.1, max_iteration=0), a.reps)
    res["icp_iter_ms"] = t1 - t0
    T, fit, rmse, it = mesher.icp_point_to_point(v, index, 0.1)
    res["icp_default"] = {"iterations": it, "fitness": fit, "rmse": rmse, "T_err": float(np.abs(T.numpy() - M).max())}
    res["align_mesh_ms"] = 1e3 * host_s(lambda: mesher.align_mesh(StandIn(hv, hf), StandIn(hd, hf), 0.1), a.reps)
    # CPU path on this host, for context
    from scipy.spatial import cKDTree
    e, g = est_pc.cpu().numpy(), gt_pc.cpu().numpy()
    res["cpu_metrics_s"] = host_s(lambda: (cKDTree(e).query(g), cKDTree(g).query(e)))
    res["cpu_icp_index_s"] = host_s(lambda: cKDTree(hd))
    if a.cpu_icp:
        res["cpu_icp_iter_s"] = host_s(lambda: meo.icp(hv, hd, 0.1, max_iteration=1)) - host_s(
            lambda: meo.icp(hv, hd, 0.1, max_iteration=0))
    res["cpu"] = "%s, %d threads" % (os.uname().machine, os.cpu_count())
    measure.emit(res, a.out)


if __name__ == "__main__":
    main()
