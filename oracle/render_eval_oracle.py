"""CPU restatement (numpy f64) of the rendering-quality metrics of goslam_render_metrics (csrc/render_eval.cu) and
goslam_b200.render_eval.  The reference project has no such metric; these definitions are the contract:

* Inputs of one frame: color [H*W, 3] (Renderer.render_img's 'color'), depth [H*W] in metres, gt_color [3, H, W]
  (DepthVideo.images; data range 1), gt_depth [H, W], mask [H, W] or None.
* PSNR: -10 log10(MSE), MSE = the mean of (color - gt)^2 over all H*W*3 values; MSE = 0 gives +inf.
* SSIM: per channel, with the separable 11-tap Gaussian window w_i = exp(-(i-5)^2 / 4.5) normalised to sum 1
  (sigma 1.5), evaluated only where the window fits ((H-10) x (W-10) positions, no padding).  With mu_x, mu_y the
  window means, sigma_x^2 = E[x^2] - mu_x^2, sigma_y^2 = E[y^2] - mu_y^2, sigma_xy = E[xy] - mu_x mu_y,
  C1 = 0.01^2, C2 = 0.03^2:
      SSIM = (2 mu_x mu_y + C1)(2 sigma_xy + C2) / ((mu_x^2 + mu_y^2 + C1)(sigma_x^2 + sigma_y^2 + C2)),
  averaged over the positions, then over the three channels.  This is meant to be pytorch_msssim.ssim(X, Y,
  data_range=1, size_average=False)'s convention (its default window, valid-only filtering and K = (0.01, 0.03)).
  That is stated from memory of its source: pytorch_msssim is not a dependency of this project and is not run here.
* Depth L1: the mean of |depth - gt_depth| over the pixels where gt_depth is finite and > 0 and the mask, if given, is
  set; the count of those pixels; NaN when the count is 0.
"""
import numpy as np

F64 = np.float64
WIN = 11
SIGMA = 1.5
C1 = 0.01 ** 2
C2 = 0.03 ** 2


def gaussian_window():
    """[11] f64: exp(-(i-5)^2 / (2 sigma^2)) normalised to sum 1"""
    i = np.arange(WIN, dtype=F64)
    g = np.exp(-(i - WIN // 2) ** 2 / (2.0 * SIGMA ** 2))
    return g / g.sum()


def _filter_valid(img):
    """[..., H, W] -> [..., H-10, W-10]: the separable Gaussian at every position where the window fits"""
    g = gaussian_window()
    H, W = img.shape[-2:]
    h = sum(g[t] * img[..., :, t:t + W - WIN + 1] for t in range(WIN))
    return sum(g[t] * h[..., t:t + H - WIN + 1, :] for t in range(WIN))


def ssim_map(x, y):
    """x, y [..., H, W] f64 -> the SSIM map [..., H-10, W-10]"""
    x, y = np.asarray(x, F64), np.asarray(y, F64)
    mx, my = _filter_valid(x), _filter_valid(y)
    sx = _filter_valid(x * x) - mx * mx
    sy = _filter_valid(y * y) - my * my
    sxy = _filter_valid(x * y) - mx * my
    return (2 * mx * my + C1) * (2 * sxy + C2) / ((mx * mx + my * my + C1) * (sx + sy + C2))


def _planar(color, H, W):
    """color [H*W, 3] -> [3, H, W] f64"""
    return np.asarray(color, F64).reshape(H, W, 3).transpose(2, 0, 1)


def psnr(color, gt_color, H, W):
    mse = np.mean((_planar(color, H, W) - np.asarray(gt_color, F64)) ** 2)
    with np.errstate(divide="ignore"):
        return float(-10.0 * np.log10(mse))


def ssim(color, gt_color, H, W):
    return float(ssim_map(_planar(color, H, W), gt_color).mean(axis=(-2, -1)).mean())


def depth_l1(depth, gt_depth, mask=None):
    """(mean |depth - gt_depth| over the valid pixels or NaN, their count)"""
    d = np.asarray(depth, F64).reshape(-1)
    g = np.asarray(gt_depth, F64).reshape(-1)
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(g) & (g > 0)
    if mask is not None:
        ok &= np.asarray(mask).reshape(-1) != 0
    n = int(ok.sum())
    return (float(np.abs(d[ok] - g[ok]).mean()) if n else float("nan")), n


def metrics(color, depth, gt_color, gt_depth, H, W, mask=None):
    """per frame of a batch: psnr, ssim, depth_l1 [K] f64 and depth_count [K] i64"""
    K = len(gt_color)
    out = {"psnr": np.empty(K), "ssim": np.empty(K), "depth_l1": np.empty(K), "depth_count": np.empty(K, np.int64)}
    for k in range(K):
        out["psnr"][k] = psnr(color[k], gt_color[k], H, W)
        out["ssim"][k] = ssim(color[k], gt_color[k], H, W)
        out["depth_l1"][k], out["depth_count"][k] = depth_l1(depth[k], gt_depth[k],
                                                             None if mask is None else mask[k])
    return out
