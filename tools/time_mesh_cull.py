"""Per-stage device time of the projection and component culls (goslam_b200.mesher) on a res-512 network mesh at the
Replica shape: 320x640 views, fx = 320, fy = 282, radius 25, 2000 poses along a trajectory (every frame, the final
call of src/slam.py) and 100 keyframe poses.  CUDA events per stage, median of --reps after a warm-up; the card's name
and power limit are read in the same run.

    python tools/time_mesh_cull.py [--reps 3] [--out result.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from goslam_b200 import mesher  # noqa: E402
from test_gpu_mesh_view import _scene_net, trajectory  # noqa: E402

H, W, FX, FY, CX, CY, RADIUS = 320, 640, 320.0, 282.0, 319.5, 159.5, 25


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        out = "unknown (%s)" % e
    return torch.cuda.get_device_name(0), out


def stages(verts, faces, rgb, c2w):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    ev[0].record()
    chunk = max(1, mesher.DEPTH_CHUNK_BYTES // (4 * H * W))
    for k0 in range(0, c2w.shape[0], chunk):                                 # the rasterizer alone, chunk by chunk
        mesher.render_depth(verts, faces, c2w[k0:k0 + chunk], H, W, FX, FY, CX, CY)
    ev[1].record()
    seen, fore = mesher.view_masks(verts, faces, c2w, H, W, FX, FY, CX, CY, RADIUS)   # rasterizer + masks
    ev[2].record()
    hv, hf, hc = mesher.keep_faces(verts, faces, colors=rgb, vert_mask=seen)
    ev[3].record()
    cv, cf, cc = mesher.filter_components(hv, hf, 0.2, colors=hc)
    ev[4].record()
    mesher.keep_faces(verts, faces, colors=rgb, vert_mask=fore)
    ev[5].record()
    torch.cuda.synchronize()
    t = [ev[i].elapsed_time(ev[i + 1]) for i in range(5)]
    return {"depth": t[0], "masks": t[1] - t[0], "masks_incl_depth": t[1], "hole_cull": t[2], "components": t[3],
            "forecast_cull": t[4], "total": t[1] + t[2] + t[3] + t[4]}, int(cf.shape[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, smi = card()
    net, gm = _scene_net()
    verts, faces, rgb = net.extract_mesh(512, 0.0, color=True)
    rt = gm["rt_bound"].astype(np.float64)
    poses = torch.from_numpy(trajectory((rt[:, 0] + rt[:, 1]) / 2, 2000)).to(verts.device)
    res = {"card": name, "nvidia_smi": smi, "V": verts.shape[0], "F": faces.shape[0], "runs": {}}
    for label, c2w in (("2000 frames", poses), ("100 keyframes", poses[::20].contiguous())):
        stages(verts, faces, rgb, c2w)                                            # warm-up
        runs = [stages(verts, faces, rgb, c2w) for _ in range(a.reps)]
        med = {k: float(np.median([r[0][k] for r in runs])) for k in runs[0][0]}
        res["runs"][label] = dict(ms=med, culled_faces=runs[0][1])
        print("%s: %s" % (label, " ".join("%s %.2f" % kv for kv in med.items())), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
