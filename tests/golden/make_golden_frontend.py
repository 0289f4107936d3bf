"""Generate tests/golden/frontend.npz by running THE REFERENCE'S OWN Frontend / Backend / FactorGraph / DepthVideo
(src/frontend.py, src/backend.py, src/factor_graph.py, src/depth_video.py) on the CPU through
tests/tools/frontend_scenario.py.

Stand-ins, as for factor_graph.npz (make_golden.gen_factor_graph): lietorch -> go-slam_b200/lietorch.py,
droid_backends.{ba, frame_distance, corr_index_forward, altcorr_forward} -> the oracle, the update operator ->
tests/tools/stub_update_op.py.

Margin check: the GPU replay must make the same discrete decisions from distances that differ in the last bits, so
every decision of the run is re-made from its distances perturbed by up to 1e-3 relative (random signs, several
draws) and must not change -- every keyframe test, every Backend.ba edge selection (dense and loop closure, restated
by oracle.graph_oracle.backend_edges, which must also reproduce what the reference hands to add_factors) and every
add_proximity_factors selection (oracle.graph_oracle.proximity_edges).  The golden is not written otherwise.

Run:  python tests/golden/make_golden_frontend.py      (needs the reference source tree, see make_golden.REF)
"""
import os
import sys

import numpy as np
import torch

import make_golden as mg
from oracle import ba_oracle, corr_oracle, geom_oracle, graph_oracle  # noqa: E402

sys.path.insert(0, os.path.join(mg.ROOT, "tests", "tools"))
import frontend_scenario as fs  # noqa: E402

REL = 1e-3
DRAWS = 8


def perturbed(d, rng):
    return [(d * (1.0 + REL * rng.choice([-1.0, 1.0], size=d.shape))).astype(np.float32) for _ in range(DRAWS)]


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

    def frame_distance(poses, disps, intrinsics, ii, jj, beta):
        return torch.from_numpy(geom_oracle.frame_distance(poses.numpy(), disps.numpy(), intrinsics.numpy(),
                                                           ii.numpy(), jj.numpy(), beta))

    def altcorr_forward(f1, f2, coords, r):
        return [torch.from_numpy(corr_oracle.altcorr_forward(f1.numpy(), f2.numpy(), coords.numpy(), r))]
    db.ba, db.frame_distance, db.altcorr_forward = ba, frame_distance, altcorr_forward
    dv_mod = mg.ref_import("src.depth_video")
    fg_mod = mg.ref_import("src.factor_graph")
    be_mod = mg.ref_import("src.backend")
    fe_mod = mg.ref_import("src.frontend")
    orig_fmt = dv_mod.DepthVideo.format_indices
    dv_mod.DepthVideo.format_indices = staticmethod(lambda ii, jj, device="cpu": orig_fmt(ii, jj, "cpu"))

    rng = np.random.default_rng(0)
    stats = {"keyframe": [], "backend": [], "proximity": 0}
    kf_thresh = fs.CFG_TRACKING["frontend"]["keyframe_thresh"]

    def grid(video, r0, t, c0, beta):
        ii, jj = torch.meshgrid(torch.arange(r0, t), torch.arange(c0, t), indexing="ij")
        return video.distance(ii.reshape(-1), jj.reshape(-1), beta=beta).numpy().astype(np.float32)

    orig_distance = dv_mod.DepthVideo.distance

    def spy_distance(self, ii=None, jj=None, beta=0.3, bidirectional=True):
        d = orig_distance(self, ii, jj, beta=beta, bidirectional=bidirectional)
        if isinstance(ii, list) and len(ii) == 1:             # the keyframe test (src/frontend.py:70)
            v = float(d.item())
            assert abs(v - kf_thresh) > 2 * REL * max(v, kf_thresh), ("keyframe test without margin", v)
            stats["keyframe"].append(v)
        return d

    orig_ba = be_mod.Backend.ba

    def spy_ba(self, t_start, t_end, steps, graph, nms, radius, thresh, max_factors, t_start_loop=None, loop=False,
               motion_only=False):
        tsl = t_start_loop if (t_start_loop is not None and loop) else t_start
        d = grid(self.video, tsl, t_end, t_start, self.beta)
        want = graph_oracle.backend_edges(d, t_start, t_end, radius, nms, thresh, max_factors, self.video.stereo,
                                          t_start_loop=t_start_loop, loop=loop)
        for dp in perturbed(d, rng):
            got = graph_oracle.backend_edges(dp, t_start, t_end, radius, nms, thresh, max_factors, self.video.stereo,
                                             t_start_loop=t_start_loop, loop=loop)
            assert (got is None) == (want is None) and (want is None or np.array_equal(got, want)), \
                ("Backend.ba selection without margin", t_start, t_end, loop)
        seen = {}
        orig_add = graph.add_factors

        def add(ii, jj, remove=False):
            seen["es"] = np.stack([ii.numpy(), jj.numpy()], 1)
            return orig_add(ii, jj, remove)
        graph.add_factors = add
        r = orig_ba(self, t_start, t_end, steps, graph, nms, radius, thresh, max_factors, t_start_loop=t_start_loop,
                    loop=loop, motion_only=motion_only)
        assert (want is None and "es" not in seen) or np.array_equal(seen["es"], want), "oracle != reference selection"
        stats["backend"].append((int(loop), t_start, t_end, 0 if want is None else len(want)))
        return r

    orig_prox = fg_mod.FactorGraph.add_proximity_factors

    def spy_prox(self, t0=0, t1=0, rad=2, nms=2, beta=0.25, thresh=16.0, remove=False):
        t = self.video.counter.value
        d = grid(self.video, t0, t, t1, beta)
        old_i = torch.cat([self.ii, self.ii_bad, self.ii_inac]).numpy()
        old_j = torch.cat([self.jj, self.jj_bad, self.jj_inac]).numpy()
        want = graph_oracle.proximity_edges(d, t0, t1, t, rad, nms, thresh, self.max_factors, self.video.stereo,
                                            old_i, old_j)
        for dp in perturbed(d, rng):
            got = graph_oracle.proximity_edges(dp, t0, t1, t, rad, nms, thresh, self.max_factors, self.video.stereo,
                                               old_i, old_j)
            assert np.array_equal(got, want), ("add_proximity_factors selection without margin", t0, t1, t)
        stats["proximity"] += 1
        return orig_prox(self, t0, t1, rad=rad, nms=nms, beta=beta, thresh=thresh, remove=remove)

    dv_mod.DepthVideo.distance = spy_distance
    be_mod.Backend.ba = spy_ba
    fg_mod.FactorGraph.add_proximity_factors = spy_prox
    try:
        cfg, args = fs.cfg_and_args("cpu")
        video = dv_mod.DepthVideo(cfg, args)
        with torch.no_grad():
            out = fs.run(fe_mod.Frontend, video, "cpu")
    finally:
        dv_mod.DepthVideo.distance = orig_distance
        be_mod.Backend.ba = orig_ba
        fg_mod.FactorGraph.add_proximity_factors = orig_prox
    n = int(out["n_calls"])
    removed = [int(out["f%02d_removed" % c]) for c in range(n)]
    loops = [out["f%02d_loops" % c].tolist() for c in range(n)]
    print("keyframe distances:", ["%.3f" % v for v in stats["keyframe"]], "threshold", kf_thresh)
    print("removed per call:", removed)
    print("loop_ba per call:", loops)
    print("Backend.ba selections (loop, t_start, t_end, edges):", stats["backend"])
    print("proximity selections checked:", stats["proximity"], " dense_ba:", out["dense_ba"].tolist())
    assert sum(removed) >= 1 and any(v >= kf_thresh for v in stats["keyframe"]), "need removed and kept keyframes"
    assert sum(len(x) for x in loops) >= 2, "loop closure must run at least twice"
    assert any(loop and e > 0 for loop, _, _, e in stats["backend"]), "no loop-closure selection"
    path = os.path.join(mg.HERE, "frontend.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        raise SystemExit("needs the reference source tree at %s" % mg.REF)
    main()
