"""CPU oracle (TEST INFRASTRUCTURE — never imported by the product path) for the correlation ops.

  corr_build           CorrBlock.corr + pyramid, src/modules/corr.py:25-41,67-76 (the reference's
                       own torch code, restated; tests/golden pins it against the reference
                       module imported from /root/reference)
  corr_index_forward   src/lib/correlation_kernels.cu:19-70 — same tap order (x outer, y inner)
                       and the same rounding sequence: fp32 instantiation = chained FMAs,
                       c10::Half instantiation = every product and every add rounded to half;
                       a tap outside the level adds nothing (the reference's within_bounds), so a
                       NaN or infinite coordinate, whose weights are NaN, leaves 0 wherever all
                       four taps of an output lie outside
  altcorr_forward      src/lib/altcorr_kernel.cu:27-149 (fp32)
Parity pin: on the GPU box the reference's own CUDA kernels (oracle/_ref) are run on the same
inputs; here, corr_index_forward is additionally checked against F.grid_sample (SURVEY §8c).
"""
import numpy as np
import torch
import torch.nn.functional as Fn

F32 = np.float32
F16 = np.float16


def corr_build(fmap1, fmap2, num_levels=4):
    """fmap [N,D,h,w] (torch, float16 or float32) -> list of [N,h,w,h>>i,w>>i].
    float16 follows the autocast path: fp32 accumulate, one rounding per level."""
    N, D, h, w = fmap1.shape
    half = fmap1.dtype == torch.float16
    a = (fmap1.reshape(N, D, h * w) / 4.0)
    b = (fmap2.reshape(N, D, h * w) / 4.0)
    corr = torch.matmul(a.float().transpose(1, 2), b.float())
    if half:
        corr = corr.half()
    corr = corr.reshape(N * h * w, 1, h, w)
    out = []
    for i in range(num_levels):
        out.append(corr.view(N, h, w, h >> i, w >> i))
        if i + 1 < num_levels:
            p = Fn.avg_pool2d(corr.float(), 2, stride=2)
            corr = p.half() if half else p
    return out


def _gather_taps(volume, coords, r):
    """taps[n,y,x,i,j] = volume[n,y,x, floor(y0)-r+j, floor(x0)-r+i] or 0 outside, and the mask of the
    taps inside.  floor(NaN) counts as 0 and huge floors are clamped, as the device's saturating
    float-to-int conversion treats them (every tap of a clamped coordinate is outside)."""
    N, h1, w1, h2, w2 = volume.shape
    x0 = coords[:, 0].astype(F32)
    y0 = coords[:, 1].astype(F32)
    with np.errstate(invalid="ignore"):
        fx = np.floor(x0)
        fy = np.floor(y0)
        dx = (x0 - fx).astype(F32)          # NaN for a NaN or infinite coordinate
        dy = (y0 - fy).astype(F32)
    fxi = np.clip(np.nan_to_num(fx, nan=0.0), -2 ** 30, 2 ** 30).astype(np.int64)
    fyi = np.clip(np.nan_to_num(fy, nan=0.0), -2 ** 30, 2 ** 30).astype(np.int64)
    rd = 2 * r + 1
    taps = np.zeros((N, h1, w1, rd + 1, rd + 1), volume.dtype)
    inside = np.zeros(taps.shape, bool)
    nn, yy, xx = np.meshgrid(np.arange(N), np.arange(h1), np.arange(w1), indexing="ij")
    for i in range(rd + 1):
        for j in range(rd + 1):
            x1 = fxi - r + i
            y1 = fyi - r + j
            ok = (x1 >= 0) & (x1 < w2) & (y1 >= 0) & (y1 < h2)
            v = volume[nn, yy, xx, np.clip(y1, 0, h2 - 1), np.clip(x1, 0, w2 - 1)]
            taps[..., i, j] = np.where(ok, v, 0)
            inside[..., i, j] = ok
    return taps, inside, dx, dy


def corr_index_forward(volume, coords, r=3):
    """volume [N,h1,w1,h2,w2] (np float16/float32), coords [N,2,h1,w1] -> [N,rd,rd,h1,w1]."""
    volume = np.asarray(volume)
    coords = np.asarray(coords, F32)
    N, h1, w1, h2, w2 = volume.shape
    rd = 2 * r + 1
    taps, inside, dx, dy = _gather_taps(volume, coords, r)
    one = F32(1.0)
    # an outside tap gets weight 0: it adds +0 where the reference adds nothing.  With finite
    # coordinates that changes no value (the tap is 0 and the weight finite); with a non-finite one it
    # keeps 0 * NaN out of the sum.
    def weight(w, i, j):
        return np.where(inside[..., i:i + rd, j:j + rd], w.astype(F32)[..., None, None], F32(0))
    w00 = weight((one - dx) * (one - dy), 0, 0)
    w01 = weight((one - dx) * dy, 0, 1)
    w10 = weight(dx * (one - dy), 1, 0)
    w11 = weight(dx * dy, 1, 1)
    s00 = taps[..., :rd, :rd]
    s01 = taps[..., :rd, 1:]
    s10 = taps[..., 1:, :rd]
    s11 = taps[..., 1:, 1:]
    if volume.dtype == F16:
        def hmul(a, b):
            return (a.astype(np.float64) * b.astype(np.float64)).astype(F16)

        def hadd(a, b):
            return (a.astype(np.float64) + b.astype(np.float64)).astype(F16)
        acc = hmul(s00, w00.astype(F16))
        acc = hadd(acc, hmul(s01, w01.astype(F16)))
        acc = hadd(acc, hmul(s10, w10.astype(F16)))
        acc = hadd(acc, hmul(s11, w11.astype(F16)))
    else:
        def fma(a, b, c):
            return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)
        acc = (s00.astype(F32) * w00).astype(F32)
        acc = fma(s01, w01, acc)
        acc = fma(s10, w10, acc)
        acc = fma(s11, w11, acc)
    # [N,h1,w1,i,j] -> [N,i,j,h1,w1]   (x-offset-major)
    return np.ascontiguousarray(acc.transpose(0, 3, 4, 1, 2))


def corr_pyramid_lookup(pyramid, coords_hw2, r=3):
    """CorrBlock.__call__ (src/modules/corr.py:43-53): pyramid list of np arrays, coords [N,h,w,2]."""
    outs = []
    c = np.ascontiguousarray(np.asarray(coords_hw2, F32).transpose(0, 3, 1, 2))
    for i, vol in enumerate(pyramid):
        o = corr_index_forward(vol, (c / F32(2 ** i)).astype(F32), r)
        N, rd, _, h1, w1 = o.shape
        outs.append(o.reshape(N, rd * rd, h1, w1))
    return np.concatenate(outs, axis=1)


def corr_index_forward_grid_sample(volume, coords, r=3):
    """independent formulation (SURVEY §8c): zero-padded bilinear grid_sample, align_corners."""
    vol = torch.from_numpy(np.asarray(volume, F32))
    N, h1, w1, h2, w2 = vol.shape
    rd = 2 * r + 1
    c = torch.from_numpy(np.asarray(coords, F32))
    dx = torch.arange(-r, r + 1, dtype=torch.float32)
    x = c[:, 0].reshape(N * h1 * w1, 1, 1) + dx.view(1, rd, 1)      # i (x-offset) major
    y = c[:, 1].reshape(N * h1 * w1, 1, 1) + dx.view(1, 1, rd)
    gx = 2 * x / (w2 - 1) - 1
    gy = 2 * y / (h2 - 1) - 1
    grid = torch.stack([gx.expand(-1, rd, rd), gy.expand(-1, rd, rd)], dim=-1)
    out = Fn.grid_sample(vol.reshape(N * h1 * w1, 1, h2, w2), grid, mode="bilinear",
                         padding_mode="zeros", align_corners=True)
    return out.view(N, h1, w1, rd, rd).permute(0, 3, 4, 1, 2).contiguous().numpy()


def altcorr_forward(fmap1, fmap2, coords, r=3):
    """fmap1 [B,H,W,C], fmap2 [B,H2,W2,C] fp32, coords [B,S,H,W,2] -> [B,S,rd*rd,H,W]."""
    f1 = np.asarray(fmap1, F32)
    f2 = np.asarray(fmap2, F32)
    coords = np.asarray(coords, F32)
    B, H, W, C = f1.shape
    _, H2, W2, _ = f2.shape
    S = coords.shape[1]
    rd = 2 * r + 1
    out = np.zeros((B, S, rd * rd, H, W), F32)
    bb, hh, ww = np.meshgrid(np.arange(B), np.arange(H), np.arange(W), indexing="ij")
    for s in range(S):
        x0, y0 = coords[:, s, ..., 0], coords[:, s, ..., 1]
        fx, fy = np.floor(x0), np.floor(y0)
        dx, dy = (x0 - fx).astype(F32), (y0 - fy).astype(F32)
        fxi, fyi = fx.astype(np.int64), fy.astype(np.int64)
        taps = np.zeros((B, H, W, rd + 1, rd + 1), F32)      # [iy, ix]
        for iy in range(rd + 1):
            for ix in range(rd + 1):
                h2 = fyi - r + iy
                w2 = fxi - r + ix
                ok = (h2 >= 0) & (h2 < H2) & (w2 >= 0) & (w2 < W2)
                g = f2[bb, np.clip(h2, 0, H2 - 1), np.clip(w2, 0, W2 - 1)]      # [B,H,W,C]
                d = np.einsum("bhwc,bhwc->bhw", f1.astype(np.float64), g.astype(np.float64))
                taps[..., iy, ix] = np.where(ok, d, 0).astype(F32)
        one = F32(1)
        w_se = ((one - dy) * (one - dx))[..., None, None]
        w_sw = ((one - dy) * dx)[..., None, None]
        w_ne = (dy * (one - dx))[..., None, None]
        w_nw = (dy * dx)[..., None, None]
        v = taps[..., :rd, :rd] * w_se + taps[..., :rd, 1:] * w_sw + taps[..., 1:, :rd] * w_ne + taps[..., 1:, 1:] * w_nw
        # v[b,h,w,oy,ox] -> channel ox*rd + oy
        out[:, s] = v.transpose(0, 4, 3, 1, 2).reshape(B, rd * rd, H, W)
    return out


def altcorr_pyramid(pyr, coords, ii, jj, num_levels, dtype=torch.float64, chunk=16):
    """AltCorrBlock.__call__ (src/modules/corr.py:113-145) on the half pyramid values widened to `dtype`:
    pyr[l] [F, H >> l, W >> l, C] (torch or numpy, any device), coords [N, H, W, 2] f32, ii / jj [N] frame ids.
    Returns (out, mag), both [N, L * 49, H, W] in `dtype` on pyr's device:
      out = sum over the 4 bilinear taps of w * <f1, f2>, with dx, dy the float32 fractions of coords * 2^-l
            (scaling by a power of two and flooring are exact in float32) and w in `dtype`;
      mag = sum over the taps of |w| * sum_c |f1_c * f2_c|, the magnitude a rounding-error bound scales with.
    Channel = ox * 7 + oy inside a level (x-offset-major), level-major across levels."""
    pyr = [torch.as_tensor(p) for p in pyr[:num_levels]]
    dev = pyr[0].device
    coords = torch.as_tensor(coords).to(dev, torch.float32)
    ii = torch.as_tensor(ii).to(dev).long()
    jj = torch.as_tensor(jj).to(dev).long()
    N, H, W, _ = coords.shape
    C = pyr[0].shape[-1]
    r, rd = 3, 7
    out = torch.zeros((N, num_levels * rd * rd, H * W), dtype=dtype, device=dev)
    mag = torch.zeros_like(out)
    p1 = pyr[0].to(dtype).reshape(-1, H * W, C)
    for lvl in range(num_levels):
        H2, W2 = pyr[lvl].shape[1], pyr[lvl].shape[2]
        p2 = pyr[lvl].to(dtype).reshape(-1, H2 * W2, C)
        c = coords.reshape(N, H * W, 2) * (1.0 / (1 << lvl))
        f = torch.floor(c)
        fr = (c - f).to(dtype)                                  # exact in float32, widened
        f = f.clamp(-2.0 ** 30, 2.0 ** 30).long()
        dx, dy = fr[..., 0], fr[..., 1]
        wts = {(0, 0): (1 - dy) * (1 - dx), (0, 1): (1 - dy) * dx, (1, 0): dy * (1 - dx), (1, 1): dy * dx}
        for n0 in range(0, N, chunk):
            sl = slice(n0, min(N, n0 + chunk))
            f1 = p1[ii[sl]]                                                          # [n, HW, C]
            f2 = p2[jj[sl]]                                                          # [n, H2W2, C]
            taps = torch.zeros((f1.shape[0], H * W, rd + 1, rd + 1), dtype=dtype, device=dev)
            atap = torch.zeros_like(taps)
            for iy in range(rd + 1):
                for ix in range(rd + 1):
                    y = f[sl, :, 1] - r + iy
                    x = f[sl, :, 0] - r + ix
                    ok = (y >= 0) & (y < H2) & (x >= 0) & (x < W2)
                    idx = (y.clamp(0, H2 - 1) * W2 + x.clamp(0, W2 - 1))
                    g = torch.gather(f2, 1, idx[..., None].expand(-1, -1, C))
                    prod = f1 * g
                    taps[..., iy, ix] = torch.where(ok, prod.sum(-1), 0)
                    atap[..., iy, ix] = torch.where(ok, prod.abs().sum(-1), 0)
            for ox in range(rd):
                for oy in range(rd):
                    ch = lvl * rd * rd + ox * rd + oy
                    o = torch.zeros_like(dx[sl])
                    m = torch.zeros_like(dx[sl])
                    for (jy, jx), w in wts.items():
                        o = o + w[sl] * taps[..., oy + jy, ox + jx]
                        m = m + w[sl].abs() * atap[..., oy + jy, ox + jx]
                    out[sl, ch] = o
                    mag[sl, ch] = m
    return out.reshape(N, -1, H, W), mag.reshape(N, -1, H, W)
