"""GPU checks of the rendering metrics (goslam_render_metrics, goslam_b200.render_eval) against the float64 oracle
(oracle/render_eval_oracle.py), per frame.

Tolerances.  The kernel and the oracle compute the same float64 expressions from the same f32 inputs, in different
orders, so they differ only by f64 rounding:
  - SSIM: x^2, y^2 and xy of f32 values are exact in f64.  Each filtered moment is a 121-term weighted sum of values in
    [0, 1] with weights summing to 1, so each side's rounding is at most ~22 * 2^-53 < 3e-15, and sigma^2, sigma_xy
    differ by < 1e-14.  SSIM's derivative with respect to a variance term is at most ~2 / C2 < 2.3e3 (C2 = 9e-4
    bounds the denominator from below, the numerator is at most ~2), so a position differs by < 3e-11 and so does the
    mean.  Bound: 1e-9 absolute.
  - PSNR: MSE is a sum of n = 3 H W squared f64 differences; each side's relative rounding is < n * 2^-53 < 1e-9 at
    480 x 640 (a linear worst case; the actual error is far smaller).  PSNR moves by (10 / ln 10) * that: < 5e-9 dB.
    Bound: 1e-8 dB (relative 1e-9 of PSNR would be looser; the absolute bound is used).
  - depth L1: a mean of at most H W f64 terms: relative bound 1e-9; the count is exact.
Each bound is shown not to be vacuous: a one-pixel perturbation of the inputs moves the oracle's value by more than
the bound, so a kernel that dropped or misplaced a pixel would fail.
"""
import os
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle import render_eval_oracle as ro

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL_SSIM, TOL_PSNR, TOL_L1 = 1e-9, 1e-8, 1e-9


def make_batch(K, H, W, seed, mask=False):
    """references in [0, 1] with a smooth region; renders = references + noise, clipped; depths with zeros, NaN and
    Inf in the reference"""
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(K, 3, H, W, generator=g)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    gt[:, :, : H // 2, : W // 2] = (0.2 + 0.6 * xx * yy)[: H // 2, : W // 2]          # a flat-ish corner
    noise = 0.05 * torch.randn(K, 3, H, W, generator=g)
    color = (gt + noise).clamp(0, 1).permute(0, 2, 3, 1).reshape(K, H * W, 3).contiguous()
    gt_depth = 0.5 + 3.0 * torch.rand(K, H, W, generator=g)
    u = torch.rand(K, H, W, generator=g)
    gt_depth[u < 0.05] = 0.0
    gt_depth[(u >= 0.05) & (u < 0.06)] = float("nan")
    gt_depth[(u >= 0.06) & (u < 0.07)] = float("inf")
    depth = (gt_depth.nan_to_num(1.0, 1.0, 1.0) + 0.1 * torch.randn(K, H, W, generator=g)).reshape(K, H * W)
    m = (torch.rand(K, H, W, generator=g) < 0.8).to(torch.uint8) if mask else None
    return color, depth, gt, gt_depth, m


def run(color, depth, gt, gt_depth, H, W, mask=None):
    from goslam_b200 import render_eval
    out = render_eval.image_metrics(color.to(DEV), depth.to(DEV), gt.to(DEV), gt_depth.to(DEV), H, W,
                                    None if mask is None else mask.to(DEV))
    return [t.cpu().numpy() for t in out]


def check_against_oracle(got, color, depth, gt, gt_depth, H, W, mask=None):
    want = ro.metrics(color.numpy(), depth.numpy(), gt.numpy(), gt_depth.numpy(), H, W,
                      None if mask is None else mask.numpy())
    psnr, ssim, l1, n = got
    assert np.array_equal(n, want["depth_count"])
    assert np.all(np.abs(ssim - want["ssim"]) <= TOL_SSIM), np.abs(ssim - want["ssim"]).max()
    same = psnr == want["psnr"]                                      # +inf where the images are identical
    assert np.all(same | (np.abs(psnr - want["psnr"]) <= TOL_PSNR)), np.abs(psnr - want["psnr"]).max()
    assert np.array_equal(np.isnan(l1), np.isnan(want["depth_l1"])) and np.all(np.isnan(l1[n == 0]))
    ok = ~np.isnan(l1)
    assert np.all(np.abs(l1[ok] - want["depth_l1"][ok]) <= TOL_L1 * np.abs(want["depth_l1"][ok]))
    return want


SHAPES = [   # (H, W, K): the smallest frame, the 16 x 32 tile's edges in positions (H-10, W-10), the 31/32/33 and 63/65
             # sizes, ScanNet's and Replica's mapping frames, a full 480 x 640 frame, and K = 1, 3, 17, 300
    (11, 11, 3), (11, 12, 1), (25, 41, 3), (26, 42, 3), (27, 43, 3), (42, 74, 3), (43, 75, 1), (31, 31, 3),
    (32, 32, 3), (33, 33, 3), (63, 65, 17), (65, 63, 3), (24, 40, 300), (240, 320, 3), (320, 640, 3), (480, 640, 1),
]


@pytest.mark.parametrize("H,W,K", SHAPES)
def test_kernel_matches_oracle_per_frame(H, W, K):
    color, depth, gt, gt_depth, mask = make_batch(K, H, W, seed=H * 1000 + W + K, mask=(K == 3))
    got = run(color, depth, gt, gt_depth, H, W, mask)
    want = check_against_oracle(got, color, depth, gt, gt_depth, H, W, mask)
    # the bounds are not vacuous: one changed pixel of frame 0 moves every metric past its bound
    c2, d2 = color[:1].clone(), depth[:1].clone()
    p = (H // 2) * W + W // 2
    c2[0, p, 1] += 2.0
    valid = torch.isfinite(gt_depth[0].reshape(-1)) & (gt_depth[0].reshape(-1) > 0)
    if mask is not None:
        valid &= mask[0].reshape(-1) != 0
    q = int(torch.nonzero(valid)[0])
    d2[0, q] += 10.0
    moved = ro.metrics(c2.numpy(), d2.numpy(), gt[:1].numpy(), gt_depth[:1].numpy(), H, W,
                       None if mask is None else mask[:1].numpy())
    psnr, ssim, l1, _ = got
    assert abs(moved["ssim"][0] - ssim[0]) > TOL_SSIM
    assert abs(moved["psnr"][0] - psnr[0]) > TOL_PSNR
    assert abs(moved["depth_l1"][0] - l1[0]) > TOL_L1 * abs(l1[0])
    assert want["depth_count"][0] > 0


def test_edge_cases():
    H, W = 37, 53
    color, depth, gt, gt_depth, _ = make_batch(5, H, W, seed=3)
    # frame 0: identical images; 1: two constants; 2: no valid depth; 3: NaN / Inf only in depth; 4: render NaN depth
    color[0] = gt[0].permute(1, 2, 0).reshape(H * W, 3)
    gt[1] = 0.3
    color[1] = 0.7
    gt_depth[2] = 0.0
    gt_depth[3, :, : W // 2] = float("nan")
    gt_depth[3, :, W // 2:] = float("inf")
    gt_depth[3, 0, 0] = 2.0
    depth[3, 0] = 1.25
    depth[4, 7] = float("nan")
    gt_depth[4].reshape(-1)[7] = 1.0
    got = run(color, depth, gt, gt_depth, H, W)
    psnr, ssim, l1, n = got
    assert psnr[0] == np.inf and ssim[0] == 1.0
    check_against_oracle(got, color, depth, gt, gt_depth, H, W)
    # constant images: mu only, no variance; SSIM = (2 * 0.3 * 0.7 + C1) / (0.3^2 + 0.7^2 + C1) in f32 inputs
    x, y = np.float64(np.float32(0.7)), np.float64(np.float32(0.3))
    assert abs(ssim[1] - (2 * x * y + ro.C1) / (x * x + y * y + ro.C1)) <= 1e-12
    assert abs(psnr[1] + 10 * np.log10((x - y) ** 2)) <= 1e-9
    assert n[2] == 0 and np.isnan(l1[2])
    assert n[3] == 1 and l1[3] == 0.75
    assert np.isnan(l1[4]) and n[4] > 0                 # a NaN render is reported, not skipped
    # a mask: only its pixels count
    mask = torch.zeros(5, H, W, dtype=torch.uint8)
    mask[:, 3, :10] = 1
    got = run(color, depth, gt, gt_depth, H, W, mask)
    check_against_oracle(got, color, depth, gt, gt_depth, H, W, mask)
    assert got[3][3] == 0 and np.array_equal(got[0], psnr) and np.array_equal(got[1], ssim)


def test_bit_identical_across_runs_and_batch_splits():
    from goslam_b200 import render_eval
    H, W, K = 70, 90, 17
    color, depth, gt, gt_depth, mask = (t.to(DEV) if t is not None else None
                                        for t in make_batch(K, H, W, seed=9, mask=True))
    a = render_eval.image_metrics(color, depth, gt, gt_depth, H, W, mask)
    b = render_eval.image_metrics(color, depth, gt, gt_depth, H, W, mask)
    bits = lambda t: t.view(torch.int64)          # noqa: E731  (NaN == NaN, bit for bit)
    for x, y in zip(a, b):
        assert torch.equal(bits(x), bits(y))
    for splits in ([0, 1, 17], [0, 5, 6, 12, 17], list(range(18))):
        parts = [render_eval.image_metrics(color[s:e], depth[s:e], gt[s:e], gt_depth[s:e], H, W, mask[s:e])
                 for s, e in zip(splits[:-1], splits[1:])]
        for x, y in zip(a, (torch.cat(p) for p in zip(*parts))):
            assert torch.equal(bits(x), bits(y))


def test_no_host_synchronisation():
    from goslam_b200 import render_eval
    H, W, K = 40, 60, 4
    args = [t.to(DEV) for t in make_batch(K, H, W, seed=1, mask=True)]
    render_eval.image_metrics(*args[:4], H, W, args[4])               # library loaded, allocator warm
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = render_eval.image_metrics(*args[:4], H, W, args[4])
        out = render_eval.image_metrics(*args[:4], H, W)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(t.is_cuda for t in out)


def _video(n, H, W, seed):
    from goslam_b200.depth_video import DepthVideo
    from oracle import mapping_oracle as mo
    cfg = {"cam": {"H_out": H, "W_out": W}, "mode": "rgbd", "tracking": {"buffer": n}}
    video = DepthVideo(cfg, types.SimpleNamespace(device="cuda:0"))
    g = torch.Generator().manual_seed(seed)
    video.pose_compensate[0] = mo.random_pose(g, 0.3).to(DEV)
    mo.fill_frames(video, range(n), g)
    video.depths_gt[:] = (0.5 + 2 * torch.rand(n, H, W, generator=g)).to(DEV)
    video.depths_gt[:, :2] = 0.0
    return video


def test_keyframe_views_match_the_mapping_items():
    from goslam_b200 import lietorch, render_eval
    from oracle import mapping_oracle as mo
    n, H, W = 12, 24, 32
    video = _video(n, H, W, seed=5)
    video.filtered_id[0] = 9
    priority = video.update_priority.clone()
    views = render_eval.keyframe_views(video)
    assert views.frames == list(range(9)) and torch.equal(video.update_priority, priority)
    for i, f in enumerate(views.frames):
        image, depth, c2w, _, mask = mo.mapping_item(video, f, DEV, 1.0, lietorch.SE3)
        assert torch.equal(views.c2w[i], c2w)
        assert torch.equal(views.images[i], image.permute(2, 0, 1))
        assert torch.equal(views.depths[i], torch.where(mask > 0, depth, torch.zeros_like(depth)))
        assert torch.equal(views.depths_gt[i], video.depths_gt[f])
    picked = render_eval.keyframe_views(video, [11, 3, 3])
    assert picked.frames == [11, 3, 3] and torch.equal(picked.c2w[1], views.c2w[3])
    assert torch.equal(picked.images[0], video.images[11])
    video.filtered_id[0] = -1
    assert render_eval.keyframe_views(video).c2w.shape == (0, 4, 4)


def test_eval_render_end_to_end_with_instant_neus():
    import bench
    from goslam_b200 import lietorch, render_eval
    from goslam_b200.render import Renderer
    from oracle import mapping_oracle as mo
    n, H, W = 5, 30, 40
    intr = (35.0, 36.0, 19.5, 14.5)
    net = bench.make_renderer(DEV, 43)[0]
    rend = Renderer({'rendering': {'N_samples': 24, 'N_surface': 48, 'lindisp': False, 'perturb': 1.0}}, None,
                    types.SimpleNamespace(H=H, W=W, fx=intr[0], fy=intr[1], cx=intr[2], cy=intr[3]),
                    ray_batch_size=500)
    video = _video(n, H, W, seed=8)
    video.filtered_id[0] = n
    views = render_eval.keyframe_views(video)
    seen = []
    real = rend.render_img

    def recording(net_, c2w, device, gt_depth):
        out = real(net_, c2w, device, gt_depth)
        seen.append((out["color"].cpu().numpy().copy(), out["depth"].reshape(-1).cpu().numpy().copy()))
        return out
    rend.render_img = recording
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "metrics_render.txt")
        with open(path, "w") as fp:
            fp.write("before\n")
        torch.manual_seed(2)
        res = render_eval.eval_render(rend, net, views.c2w, views.images, views.depths_gt, prior_depth=views.depths,
                                      out_path=path, frames_per_call=2)
        text = open(path).read()
    assert len(seen) == n
    assert text == "before\n" + res.pretty_str() and text.count("Rendering metrics (5 views)") == 1
    color = torch.from_numpy(np.stack([s[0] for s in seen]))
    depth = torch.from_numpy(np.stack([s[1] for s in seen]))
    assert np.isfinite(color.numpy()).all() and (color.numpy() != 0).any()
    check_against_oracle([res.psnr, res.ssim, res.depth_l1, res.depth_count], color, depth, views.images.cpu(),
                         views.depths_gt.cpu(), H, W)
    assert res.stats["depth_views"] == n and res.stats["psnr"] == pytest.approx(res.psnr.mean())
    # the renders are render_img's own: the same generator state renders the same first view
    torch.manual_seed(2)
    again = real(net, views.c2w[0], DEV, views.depths[0])
    assert np.array_equal(again["color"].cpu().numpy(), seen[0][0])
