"""Mesh extraction stage by stage (what InstantNeuS.extract_geometry(res, 0.0, None, save_path=None, color=True) runs),
on a trained_like net, at the mesher's resolutions.  CUDA events per stage, median of 5 after a warm-up:
  field   goslam_neus_sdf_grid (compared with the marcher's samples/s: the same 16-level gathers, minus the MLP)
  count   goslam_mc_count             emit    goslam_mc_emit
          (marching cubes compared with the bytes it must move: u read twice, plus the vertices and faces written)
  cull    goslam_mesh_cull_count + _emit
  colour  goslam_neus_vertex_color of the kept vertices
  copy    the final device-to-host copy (vertices, faces, colours into pinned memory)
usage: python tools/time_mesh.py [res ...]        (default 256 512 1024)"""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_mesh.py")
import numpy as np  # noqa: E402
import torch  # noqa: E402

from goslam_b200 import _lib, neus, synthetic  # noqa: E402

dev = torch.device("cuda:0")
BOUND = [[-2.0, 1.5], [-1.2, 1.8], [-1.0, 2.2]]
RT_BOUND = [[-1.7, 1.3], [-1.0, 1.6], [-0.8, 2.0]]


def make_net():
    offs, ress, _, total = neus.hashgrid_layout()
    w = synthetic.make_neus_weights(seed=5, total_grid_params=total, layout=(offs, ress))
    net = neus.InstantNeuS(synthetic.NEUS_CFG, BOUND)
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to(dev)
    net.update_bound(torch.tensor(RT_BOUND))
    return net


def timed(fn):
    """fn's result and the ms of that one call"""
    out = []
    return out, measure.cuda_time(lambda: out.append(fn()), 1, warmup=0)["median_ms"]


def one_pass(net, res):
    """one extraction split into its stages; returns ({stage: ms}, (V, F) before the cull, (V, F) after)"""
    lib = _lib.load()
    st = _lib.stream_ptr()
    b = net.bound.cpu().tolist()
    bmin, bmax = [x[0] for x in b], [x[1] for x in b]
    ms = {}
    (u,), ms["field"] = timed(lambda: net._sdf_grid(bmin, bmax, res))
    ws = torch.empty(lib.goslam_mc_workspace_bytes(res, res, res), dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    _, ms["count"] = timed(lambda: _lib.check(lib.goslam_mc_count(_lib.ptr(u), res, res, res, 0.0, _lib.ptr(ws), ws.numel(),
                                                                   _lib.ptr(counts), st), "mc_count"))
    nv, nf = counts.tolist()
    verts = torch.empty((nv, 3), dtype=torch.float64, device=dev)
    faces = torch.empty((nf, 3), dtype=torch.int64, device=dev)
    lo, hi = (ctypes.c_float * 3)(*bmin), (ctypes.c_float * 3)(*bmax)
    _, ms["emit"] = timed(lambda: _lib.check(lib.goslam_mc_emit(_lib.ptr(u), res, res, res, 0.0, lo, hi, _lib.ptr(ws), ws.numel(),
                                                                 _lib.ptr(verts), nv, _lib.ptr(faces), nf, st), "mc_emit"))
    del ws, u
    rt = np.array(net.realtime_bound.cpu().numpy(), np.float32)
    ((cv, cf),), ms["cull"] = timed(lambda: neus.cull_mesh(verts, faces, (rt[:, 0] - 0.01).tolist(), (rt[:, 1] + 0.01).tolist()))
    flat = sum(b, [])
    (rgb,), ms["colour"] = timed(lambda: net._vertex_colors(cv, flat))
    host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in (cv, cf, rgb)]

    def copy():
        for h, t in zip(host, (cv, cf, rgb)):
            h.copy_(t, non_blocking=True)
    _, ms["copy"] = timed(copy)
    return ms, (nv, nf), (cv.shape[0], cf.shape[0])


def marcher_rate(net):
    """samples/s of the fused marcher (InstantNeuS.forward under no_grad) on 2^16 rays x 72 samples"""
    ro, rd, zv, ds = (t.to(dev) for t in synthetic.make_rays(1 << 16, S=72, seed=3))
    with torch.no_grad():
        for _ in range(2):
            net(ro, rd, zv, ds)
        t = measure.cuda_time(lambda: net(ro, rd, zv, ds), 5, warmup=0)
    return zv.numel() / (t["median_ms"] * 1e-3)


def main():
    resolutions = [int(a) for a in sys.argv[1:]] or [256, 512, 1024]
    measure.emit({})
    net = make_net()
    rate = marcher_rate(net)
    print("marcher: %.3g samples/s (2^16 rays x 72 samples)" % rate)
    stages = ("field", "count", "emit", "cull", "colour", "copy")
    print("%5s %10s %10s %10s | %s | %8s | %12s %12s" % ("res", "V", "F", "kept F", " ".join("%8s" % s for s in stages), "total",
                                                       "field pts/s", "MC GB/s"))
    for res in resolutions:
        one_pass(net, res)                              # warm-up
        runs = [one_pass(net, res) for _ in range(5)]
        med = {s: float(np.median([r[0][s] for r in runs])) for s in stages}
        (nv, nf), (kv, kf) = runs[0][1], runs[0][2]
        n = res ** 3
        mc_bytes = 2 * 4 * n + 24 * nv + 24 * nf
        print("%5d %10d %10d %10d | %s | %8.2f | %12.3g %12.1f" % (
            res, nv, nf, kf, " ".join("%8.2f" % med[s] for s in stages), sum(med.values()),
            n / (med["field"] * 1e-3), mc_bytes / ((med["count"] + med["emit"]) * 1e-3) / 1e9))
        torch.cuda.empty_cache()
    print("(times in ms; field pts/s against the marcher's samples/s above)")


if __name__ == "__main__":
    main()
