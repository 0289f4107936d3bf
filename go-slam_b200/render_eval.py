"""How good is the map: PSNR, SSIM and depth L1 of rendered keyframe views, on the device.

The reference project has no rendering metric; this is an opt-in evaluation a user calls, like `slam.ape`:

    from goslam_b200 import render_eval
    views = render_eval.keyframe_views(slam.video)
    result = render_eval.eval_render(slam.renderer, slam.mapping_net, views.c2w, views.images, views.depths_gt,
                                     prior_depth=views.depths, out_path=f'{slam.output}/metrics_render.txt')
    print(result.pretty_str())

`image_metrics` scores a batch of rendered images with one library call (goslam_render_metrics, DESIGN §3.20).  The
definitions (PSNR over all values with data range 1, SSIM with an 11-tap sigma-1.5 Gaussian at the valid positions
only, depth L1 over finite positive reference depths) are stated in include/goslam_b200.h and restated in float64 in
oracle/render_eval_oracle.py.  The SSIM is meant to follow pytorch_msssim.ssim(X, Y, data_range=1); that is stated
from memory of its source, as pytorch_msssim is not a dependency of this project.
"""
from collections import namedtuple

import numpy as np
import torch

from . import _lib
from .lietorch import SE3

KeyframeViews = namedtuple("KeyframeViews", "frames c2w images depths depths_gt")


@torch.no_grad()
def image_metrics(color, depth, gt_color, gt_depth, H, W, mask=None):
    """PSNR, SSIM and depth L1 of K rendered views against their references, one library call.

    color [K, H*W, 3] (render_img's 'color', any shape with K*H*W*3 elements), depth [K, H*W] (any shape with K*H*W
    elements), gt_color [K, 3, H, W] with data range 1, gt_depth [K, H, W], mask [K, H, W] (non-zero = counted) or
    None; CUDA tensors on one device, converted to f32 (and the mask to u8) on the device.  Returns (psnr, ssim,
    depth_l1, depth_count): f64 [K], f64 [K], f64 [K], i64 [K] on that device, without a host synchronisation.
    depth_l1 is NaN where depth_count is 0."""
    _lib.need_cuda("image_metrics", color, depth, gt_color, gt_depth, mask)
    H, W = int(H), int(W)
    K = int(gt_color.shape[0]) if gt_color.dim() == 4 else -1
    if tuple(gt_color.shape) != (K, 3, H, W) or color.numel() != K * H * W * 3 or depth.numel() != K * H * W \
            or gt_depth.numel() != K * H * W or (mask is not None and mask.numel() != K * H * W):
        raise ValueError("image_metrics: want color [K, H*W, 3], depth [K, H*W], gt_color [K, 3, %d, %d], gt_depth and "
                         "mask [K, %d, %d]; got %s, %s, %s, %s, %s"
                         % (H, W, H, W, tuple(color.shape), tuple(depth.shape), tuple(gt_color.shape),
                            tuple(gt_depth.shape), None if mask is None else tuple(mask.shape)))
    dev = gt_color.device
    nbytes = int(_lib.load().goslam_render_metrics_workspace_bytes(K, H, W))
    if nbytes == 0:
        raise ValueError("image_metrics: H and W must be at least 11 (the SSIM window), got %d x %d" % (H, W))
    f32 = dict(dtype=torch.float32)
    out = (torch.empty(K, dtype=torch.float64, device=dev), torch.empty(K, dtype=torch.float64, device=dev),
           torch.empty(K, dtype=torch.float64, device=dev), torch.empty(K, dtype=torch.int64, device=dev))
    if K == 0:
        return out
    args = [color.to(**f32).contiguous(), depth.to(**f32).contiguous(), gt_color.to(**f32).contiguous(),
            gt_depth.to(**f32).contiguous(), None if mask is None else (mask != 0).to(torch.uint8).contiguous()]
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.call("render_metrics", *args, K, H, W, ws, nbytes, *out)
    return out


def keyframe_views(video, frames=None):
    """The keyframes the mapper reads, under one hold of the video's mapping lock (as mapping.snapshot_frames):
    frames 0 .. filtered_id - 1, whose poses_filtered / disps_filtered the multiview filter has committed, or the
    given list.  Returns KeyframeViews:
      frames     the frame ids, a list;
      c2w        [F, 4, 4]: (SE3(pose_compensate[0]) * SE3(poses_filtered).inv()).matrix(), the mapper's cameras;
      images     [F, 3, H, W]: the colour the mapping loss trains against;
      depths     [F, H, W]: the mapper's target depth 1 / (disps_filtered + 1e-7) where mask_filtered is set, else 0:
                 the depth render_img samples around (its `gt_depth`);
      depths_gt  [F, H, W]: the sensor depth to score against (all zeros for monocular input, so depth L1 is NaN)."""
    with video.mapping.get_lock():
        if frames is None:
            frames = list(range(max(int(video.filtered_id.item()), 0)))
        frames = [int(f) for f in frames]
        buffer = video.images.shape[0]
        if any(f < 0 or f >= buffer for f in frames):
            raise IndexError("keyframe_views: frame id outside the video buffer [0, %d)" % buffer)
        idx = torch.tensor(frames, dtype=torch.long).to(video.images.device)
        poses = video.poses_filtered.index_select(0, idx)
        comp = video.pose_compensate[0:1].clone()
        images = video.images.index_select(0, idx)
        disps = video.disps_filtered.index_select(0, idx)
        mask = video.mask_filtered.index_select(0, idx)
        depths_gt = video.depths_gt.index_select(0, idx)
    if not frames:
        c2w = torch.empty((0, 4, 4), dtype=poses.dtype, device=poses.device)
    else:
        c2w = (SE3(comp) * SE3(poses).inv()).matrix().contiguous()
    depths = torch.where(mask > 0, 1.0 / (disps + 1e-7), torch.zeros_like(disps))
    return KeyframeViews(frames, c2w, images, depths, depths_gt)


class RenderMetrics:
    """Per-frame results of eval_render (numpy: psnr, ssim, depth_l1 f64 [K], depth_count i64 [K]) and their means.

    stats: psnr and ssim are the means over all frames (an identical view has psnr +inf, and so does the mean);
    depth_l1 is the mean over the frames with at least one valid depth pixel (NaN if there are none), and depth_views
    the number of those frames.

    pretty_str() is fixed: the title line "Rendering metrics (<K> views)", a blank line, then "{:>12}\\t{:.6f}\\n" for
    psnr, ssim and depth_l1 and "{:>12}\\t{:d}\\n" for depth_views, in that order."""

    TITLE = "Rendering metrics ({} views)"

    def __init__(self, psnr, ssim, depth_l1, depth_count):
        self.psnr, self.ssim, self.depth_l1, self.depth_count = psnr, ssim, depth_l1, depth_count
        has_depth = depth_count > 0
        self.stats = {
            "psnr": float(psnr.mean()) if len(psnr) else float("nan"),
            "ssim": float(ssim.mean()) if len(ssim) else float("nan"),
            "depth_l1": float(depth_l1[has_depth].mean()) if has_depth.any() else float("nan"),
            "depth_views": int(has_depth.sum()),
        }

    def pretty_str(self):
        text = self.TITLE.format(len(self.psnr)) + "\n\n"
        for name in ("psnr", "ssim", "depth_l1"):
            text += "{:>12}\t{:.6f}\n".format(name, self.stats[name])
        text += "{:>12}\t{:d}\n".format("depth_views", self.stats["depth_views"])
        return text


@torch.no_grad()
def eval_render(renderer, net, c2w, gt_color, gt_depth, prior_depth=None, out_path=None, frames_per_call=16):
    """Render every view with renderer.render_img(net, c2w[k], device, prior_depth[k]) and score it against
    gt_color [K, 3, H, W] and gt_depth [K, H, W] with image_metrics, frames_per_call views per call.

    prior_depth [K, H, W] is the depth render_img samples around; None uses gt_depth (as the reference's
    visualiser does), which suits RGB-D input.  For monocular input pass keyframe_views(...).depths.  The views are
    rendered one at a time, exactly as render_img renders them; the only host synchronisation is the final read of
    the results.  Returns a RenderMetrics; with out_path, its pretty_str() is appended to that file."""
    K = int(c2w.shape[0])
    H, W = int(renderer.H), int(renderer.W)
    dev = gt_color.device
    if prior_depth is None:
        prior_depth = gt_depth
    if frames_per_call < 1:
        raise ValueError("eval_render: frames_per_call must be at least 1")
    parts = []
    for b0 in range(0, K, frames_per_call):
        b1 = min(b0 + frames_per_call, K)
        color = torch.empty((b1 - b0, H * W, 3), dtype=torch.float32, device=dev)
        depth = torch.empty((b1 - b0, H * W), dtype=torch.float32, device=dev)
        for k in range(b0, b1):
            out = renderer.render_img(net, c2w[k], dev, prior_depth[k])
            color[k - b0] = out["color"]
            depth[k - b0] = out["depth"].reshape(-1)
        parts.append(image_metrics(color, depth, gt_color[b0:b1], gt_depth[b0:b1], H, W))
    if parts:
        host = [torch.cat(p).cpu().numpy() for p in zip(*parts)]
    else:
        host = [np.empty(0), np.empty(0), np.empty(0), np.empty(0, np.int64)]
    result = RenderMetrics(*host)
    if out_path is not None:
        with open(out_path, "a") as fp:
            fp.write(result.pretty_str())
    return result
