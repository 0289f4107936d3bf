"""Time of the rendering metrics (goslam_b200.render_eval).

  - the metrics alone: image_metrics on K = 100 frames of the Replica mapping shape (320 x 640), and of 480 x 640, as
    GB/s against the 32 bytes per pixel it must read (rendered colour 12, rendered depth 4, reference colour 12,
    reference depth 4);
  - eval_render per frame: render_img with the library's InstantNeuS (the config's 24 + 48 samples, 5 000-ray chunks)
    and the scoring, at 320 x 640, over 8 views.
CUDA events around --reps calls after a warm-up, median per call; the card's name and power limit are read in the
same run.

    python tools/time_render_eval.py [--reps 20] [--out result.json]
"""
import argparse
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools import measure  # noqa: E402
measure.require_cuda("time_render_eval.py")

import torch  # noqa: E402

from goslam_b200 import lietorch, render_eval  # noqa: E402

DEV = torch.device("cuda:0")
BYTES_PER_PIXEL = 32


def timed(fn, reps, warmup=3):
    t = measure.cuda_time(fn, reps, warmup)
    return t["median_ms"], t["min_ms"], t["max_ms"]


def metrics_inputs(K, H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    gt = torch.rand(K, 3, H, W, generator=g, device=DEV)
    color = (gt + 0.05 * torch.randn(K, 3, H, W, generator=g, device=DEV)).clamp(0, 1)
    color = color.permute(0, 2, 3, 1).reshape(K, H * W, 3).contiguous()
    gt_depth = 0.5 + 3.0 * torch.rand(K, H, W, generator=g, device=DEV)
    depth = (gt_depth + 0.1 * torch.randn(K, H, W, generator=g, device=DEV)).reshape(K, H * W)
    return color, depth, gt, gt_depth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    measure.emit({})
    rows = []
    for K, H, W in ((100, 320, 640), (100, 480, 640)):
        inp = metrics_inputs(K, H, W, 1)
        med, lo, hi = timed(lambda: render_eval.image_metrics(*inp, H, W), args.reps)
        gbs = BYTES_PER_PIXEL * K * H * W / (med * 1e-3) / 1e9
        rows.append({"what": "image_metrics", "K": K, "H": H, "W": W, "median_ms": med, "min_ms": lo, "max_ms": hi,
                     "GB_per_s": gbs})
        print("image_metrics K=%d %dx%d: %.3f ms (min %.3f, max %.3f), %.0f GB/s of %d B/pixel"
              % (K, H, W, med, lo, hi, gbs, BYTES_PER_PIXEL))

    import bench
    from goslam_b200.render import Renderer
    H, W, n = 320, 640, 8
    net = bench.make_renderer(DEV, 43)[0]
    rend = Renderer({'rendering': {'N_samples': 24, 'N_surface': 48, 'lindisp': False, 'perturb': 1.0}}, None,
                    types.SimpleNamespace(H=H, W=W, fx=320.0, fy=320.0, cx=319.5, cy=159.5))
    g = torch.Generator().manual_seed(3)
    poses = torch.stack([torch.cat([0.3 * torch.randn(3, generator=g), torch.nn.functional.normalize(
        torch.randn(4, generator=g), dim=0)]) for _ in range(n)])
    c2w = lietorch.SE3(poses).inv().matrix().to(DEV)
    _, _, gt, gt_depth = metrics_inputs(n, H, W, 2)
    torch.manual_seed(0)
    med, lo, hi = timed(lambda: render_eval.eval_render(rend, net, c2w, gt, gt_depth), max(args.reps // 4, 3), warmup=1)
    rows.append({"what": "eval_render", "K": n, "H": H, "W": W, "median_ms_per_frame": med / n,
                 "min_ms_per_frame": lo / n, "max_ms_per_frame": hi / n})
    print("eval_render %d views %dx%d: %.2f ms per frame (min %.2f, max %.2f)" % (n, H, W, med / n, lo / n, hi / n))
    measure.emit({"reps": args.reps, "rows": rows}, args.out)


if __name__ == "__main__":
    main()
