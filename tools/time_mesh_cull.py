"""Per-stage device time of the projection and component culls (goslam_b200.mesher) on a res-512 network mesh at the
Replica shape: 320x640 views, fx = 320, fy = 282, radius 25, 2000 poses along a trajectory (every frame, the final
call of src/slam.py) and 100 keyframe poses.  CUDA events around each stage, median of --reps after a warm-up; the
card's name and power limit are read in the same run.

    python tools/time_mesh_cull.py [--reps 3] [--out result.json]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools import measure  # noqa: E402
measure.require_cuda("time_mesh_cull.py")

import numpy as np  # noqa: E402
import torch  # noqa: E402

from goslam_b200 import mesher  # noqa: E402
from test_gpu_mesh_view import _scene_net, trajectory  # noqa: E402

H, W, FX, FY, CX, CY, RADIUS = 320, 640, 320.0, 282.0, 319.5, 159.5, 25


def timed(fn):
    """fn's result and the ms of that one call"""
    out = []
    return out, measure.cuda_time(lambda: out.append(fn()), 1, warmup=0)["median_ms"]


def stages(verts, faces, rgb, c2w):
    chunk = max(1, mesher.DEPTH_CHUNK_BYTES // (4 * H * W))
    t = [0.0] * 5
    _, t[0] = timed(lambda: [mesher.render_depth(verts, faces, c2w[k0:k0 + chunk], H, W, FX, FY, CX, CY)
                             for k0 in range(0, c2w.shape[0], chunk)])               # the rasterizer alone, chunk by chunk
    ((seen, fore),), t[1] = timed(lambda: mesher.view_masks(verts, faces, c2w, H, W, FX, FY, CX, CY, RADIUS))
    ((hv, hf, hc),), t[2] = timed(lambda: mesher.keep_faces(verts, faces, colors=rgb, vert_mask=seen))
    ((cv, cf, cc),), t[3] = timed(lambda: mesher.filter_components(hv, hf, 0.2, colors=hc))
    _, t[4] = timed(lambda: mesher.keep_faces(verts, faces, colors=rgb, vert_mask=fore))
    return {"depth": t[0], "masks": t[1] - t[0], "masks_incl_depth": t[1], "hole_cull": t[2], "components": t[3],
            "forecast_cull": t[4], "total": t[1] + t[2] + t[3] + t[4]}, int(cf.shape[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    net, gm = _scene_net()
    verts, faces, rgb = net.extract_mesh(512, 0.0, color=True)
    rt = gm["rt_bound"].astype(np.float64)
    poses = torch.from_numpy(trajectory((rt[:, 0] + rt[:, 1]) / 2, 2000)).to(verts.device)
    res = {"V": verts.shape[0], "F": faces.shape[0], "runs": {}}
    for label, c2w in (("2000 frames", poses), ("100 keyframes", poses[::20].contiguous())):
        stages(verts, faces, rgb, c2w)                                            # warm-up
        runs = [stages(verts, faces, rgb, c2w) for _ in range(a.reps)]
        med = {k: float(np.median([r[0][k] for r in runs])) for k in runs[0][0]}
        res["runs"][label] = dict(ms=med, culled_faces=runs[0][1])
        print("%s: %s" % (label, " ".join("%s %.2f" % kv for kv in med.items())), flush=True)
    measure.emit(res, a.out)


if __name__ == "__main__":
    main()
