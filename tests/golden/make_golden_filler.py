"""Generate tests/golden/trajectory_filler.npz by running THE REFERENCE'S OWN PoseTrajectoryFiller.__call__
(src/trajectory_filler.py) on the CPU over the three streams of tests/tools/filler_scenario.py (RGB-D in chunks of
16, 16 and 5; mono in 16 and 9; one stereo chunk).

Stand-ins, as for factor_graph.npz: lietorch -> go-slam_b200/lietorch.py, droid_backends.corr_index_forward and .ba ->
the oracle (make_golden.install_stubs, oracle.ba_oracle), the update operator -> tests/tools/stub_update_op.py, fnet ->
tests/tools/stub_fnet.py.  The reference's FactorGraph is bound to device='cpu' and Tensor.cuda is the identity for the
run.  Spies on DepthVideo.__setitem__ and FactorGraph.add_factors record, per chunk, the interpolated poses, t0 / t1
and the graph's edges after the two add_factors calls; the file also holds the trajectory, the counter afterwards and
the video rows of the last chunk.

Run:  python tests/golden/make_golden_filler.py      (needs the reference source tree, see make_golden.REF)
"""
import functools
import os
import sys
import types

import numpy as np
import torch

import make_golden as mg
from oracle import ba_oracle  # noqa: E402  (make_golden puts the repository on sys.path)

sys.path.insert(0, os.path.join(mg.ROOT, "tests", "tools"))
import filler_scenario as fs  # noqa: E402
from stub_fnet import StubFnet  # noqa: E402
from stub_update_op import update_op  # noqa: E402


def _np(t):
    return t.detach().cpu().numpy().copy()


def main():
    mg.install_stubs()
    db = sys.modules["droid_backends"]

    def ba(poses, disps, intrinsics, disps_sens, targets, weights, eta, ii, jj, t0, t1, iters, lm, ep, motion_only):
        rp, rd, dx, dz, st = ba_oracle.ba(poses.numpy(), disps.numpy(), intrinsics.numpy(), disps_sens.numpy(),
                                          targets.numpy(), weights.numpy(), eta.numpy(), ii.numpy(), jj.numpy(),
                                          int(t0), int(t1), int(iters), lm, ep, bool(motion_only))
        assert list(st) == [0] * int(iters)
        poses.copy_(torch.from_numpy(rp))
        disps.copy_(torch.from_numpy(rd))
        return [torch.from_numpy(dx), torch.from_numpy(dz)]
    db.ba = ba
    dv_mod = mg.ref_import("src.depth_video")
    fg_mod = mg.ref_import("src.factor_graph")
    tf_mod = mg.ref_import("src.trajectory_filler")
    orig_fmt = dv_mod.DepthVideo.format_indices
    dv_mod.DepthVideo.format_indices = staticmethod(lambda ii, jj, device="cpu": orig_fmt(ii, jj, "cpu"))
    tf_mod.FactorGraph = functools.partial(fg_mod.FactorGraph, device="cpu")

    rec = {}
    orig_set, orig_add = dv_mod.DepthVideo.__setitem__, fg_mod.FactorGraph.add_factors

    def spy_set(self, index, item):
        rec["G"] = _np(item[2])
        return orig_set(self, index, item)

    def spy_add(self, ii, jj, remove=False):
        rec.setdefault("args", []).append(_np(ii))
        out = orig_add(self, ii, jj, remove)
        if len(rec["args"]) == 2:
            chunks.append(dict(G=rec.pop("G"), t0=rec["args"][0], t1=rec["args"][1], ii=_np(self.ii), jj=_np(self.jj)))
            rec.clear()
        return out

    out = {}
    orig_cuda = torch.Tensor.cuda
    dv_mod.DepthVideo.__setitem__, fg_mod.FactorGraph.add_factors = spy_set, spy_add
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        for kind in fs.STREAMS:
            chunks = []
            cfg, args = fs.cfg_and_args("cpu", stereo=kind == "stereo")
            video = dv_mod.DepthVideo(cfg, args)
            fs.fill_keyframes(video, stereo=kind == "stereo")
            N = video.counter.value
            net = types.SimpleNamespace(cnet=None, fnet=StubFnet(), update=update_op)
            filler = tf_mod.PoseTrajectoryFiller(net, video, device="cpu")
            traj = filler(fs.stream(kind))
            out[kind + "_traj"] = _np(traj.data)
            out[kind + "_counter"] = np.int64(video.counter.value)
            out[kind + "_chunks"] = np.int64(len(chunks))
            for c, d in enumerate(chunks):
                for k, v in d.items():
                    out["%s_c%d_%s" % (kind, c, k)] = v
            M = len(chunks[-1]["t0"])
            rows = slice(N, N + M)
            for name in ("timestamp", "poses", "intrinsics", "disps", "disps_sens"):
                out["%s_last_%s" % (kind, name)] = _np(getattr(video, name)[rows])
            out[kind + "_last_images"] = _np(video.images[rows, :, ::8, ::8])
            out[kind + "_last_fmaps"] = _np(video.fmaps[rows, :, ::8])
            print("%s: %d chunks of %s frames, t0 %s" % (kind, len(chunks), [len(d["t0"]) for d in chunks],
                                                        [d["t0"].tolist() for d in chunks]))
    finally:
        torch.Tensor.cuda = orig_cuda
        dv_mod.DepthVideo.__setitem__, fg_mod.FactorGraph.add_factors = orig_set, orig_add
    path = os.path.join(mg.HERE, "trajectory_filler.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        raise SystemExit("needs the reference source tree at %s" % mg.REF)
    main()
