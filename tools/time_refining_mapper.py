"""Time camera refinement in mapping at the Replica shape (22 frames of 320x640, a 22-entry visit list, 4,400 pixels per
batch) with CUDA events after warm-up, and print the card's name and power limit beside the numbers:
  * one RefiningMapper call (the library's InstantNeuS and Renderer, iters 10) with mapping.BA off and on;
  * per visit iteration, the pose-ray forward + backward (build_pose_ray_batch and its autograd backward);
  * the same batch by the reference's per-entry construction (quaternion_to_Rt + build_rays restated with torch ops,
    torch.cat) and its autograd backward.
Run on the GPU:  python tools/time_refining_mapper.py"""
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_refining_mapper.py")
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from oracle import mapping_oracle as mo  # noqa: E402
from oracle import refine_oracle as ro  # noqa: E402

DEV = torch.device("cuda:0")
N, H, W, PIXELS, WINDOW = 22, 320, 640, 4400, 22
INTR = (320.0, 320.0, 319.5, 159.5)


def timed(fn, n):
    """ms per call of one event pair around n back-to-back calls"""
    return measure.cuda_time(fn, 1, warmup=0, batch=n)["median_ms"]


def video():
    v = mo.stub_video(N, H, W, DEV)
    g = torch.Generator().manual_seed(5)
    v.pose_compensate[0] = mo.random_pose(g, 0.3)
    mo.fill_frames(v, range(N), g, trans=0.4)
    v.bound[0] = torch.tensor([[-2.0, 2.0]] * 3)
    return v


def mapper_call(ba):
    """median ms of one RefiningMapper call at last_visit >= 10 (the visit iterations only: no unvisit list)"""
    from goslam_b200 import mapping
    from goslam_b200.render import Renderer
    cfg = mo.mapping_cfg("cuda:0", PIXELS, WINDOW, 10)
    cfg['mapping']['BA'] = ba
    rend = Renderer({'rendering': {'N_samples': 24, 'N_surface': 48, 'lindisp': False, 'perturb': 1.0}}, None,
                    types.SimpleNamespace(H=H, W=W, fx=INTR[0], fy=INTR[1], cx=INTR[2], cy=INTR[3]), ray_batch_size=5e3)
    net = bench.make_renderer(DEV, 43)[0]
    m = mapping.RefiningMapper(cfg, types.SimpleNamespace(), mo.stub_slam(video(), net, rend, INTR, tempfile.mkdtemp()))
    np.random.seed(1)
    m.video.filtered_id[0] = 12                            # unvisit pass, last_visit -> 12
    m()
    m.video.filtered_id[0] = N                             # from here on every call refines (when BA is on)
    times = []
    for _ in range(5):
        m.last_visit = N
        times.append(timed(m, 1))
    return sorted(times)[2], times


def per_iteration():
    from goslam_b200 import mapping
    from goslam_b200.depth_video import DepthVideo
    v = video()
    snap = mapping.snapshot_frames(v, list(range(N)), 0.8)
    twin = video()
    items = {f: DepthVideo.get_mapping_item(twin, f, DEV, decay=0.8) for f in range(N)}
    fl = list(range(N))
    quadt = mapping.c2w_to_quadt(snap.c2w).requires_grad_(True)
    n_rays = PIXELS // len(fl)
    g = torch.Generator(device=DEV).manual_seed(2)
    grads = [torch.randn((PIXELS, 3), device=DEV, generator=g) for _ in range(2)]

    def ours():
        quadt.grad = None
        b = mapping.build_pose_ray_batch(snap, fl, n_rays, INTR, quadt)
        torch.autograd.backward([b.rays_o, b.rays_d], grads)

    leaves = [q.detach().clone().requires_grad_(True) for q in quadt]

    def theirs():
        for q in leaves:
            q.grad = None
        parts = [[], [], [], []]
        for e, f in enumerate(fl):
            image, depth, _, _, mask = items[f]
            for acc, t in zip(parts, mo.build_rays(n_rays, H, W, *INTR, ro.quaternion_to_rt(leaves[e]), depth, image,
                                                   DEV, mask)):
                acc.append(t.float())
        o, d = torch.cat(parts[0]), torch.cat(parts[1])
        torch.autograd.backward([o, d], grads)

    for fn in (ours, theirs):
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {"ours": [], "theirs": []}
    for _ in range(5):
        res["ours"].append(timed(ours, 50))
        res["theirs"].append(timed(theirs, 10))
    return {k: (sorted(x)[2], min(x), max(x)) for k, x in res.items()}


def main():
    measure.emit({})
    off, t_off = mapper_call(False)
    on, t_on = mapper_call(True)
    print("RefiningMapper call, Replica 320x640, 22-entry visit list, 4400 rays x 10 iterations:")
    print("  BA off %.2f ms (%.2f-%.2f)   BA on %.2f ms (%.2f-%.2f)   extra %.2f ms (%.1f %%)" % (
        off, min(t_off), max(t_off), on, min(t_on), max(t_on), on - off, 100.0 * (on - off) / off))
    r = per_iteration()
    print("per visit iteration, rays + pose gradient of 22 entries x 200 rays:")
    print("  pose-ray kernels  %.3f ms (%.3f-%.3f)" % r["ours"])
    print("  per-entry torch   %.3f ms (%.3f-%.3f)" % r["theirs"])


if __name__ == "__main__":
    main()
