"""CPU oracle (TEST INFRASTRUCTURE — never imported by the product path) for the renderer's gradient with respect to its
rays (camera refinement, src/mapping.py:173-194 with mapping.BA: rays built from a quaternion-translation leaf):
  * ray_backward_closed_form — the float64 closed form neus_ray_bwd_kernel implements (csrc/neus.cu);
  * TorchHashGrid64 — oracle/neus_grad_oracle.py's TorchHashGrid evaluated in float64 (cell and fraction still taken from
    the float32 position, as tcnn and the kernel take them), so that double-backward autograd pins the closed form to
    rounding level;
  * quat_to_rotation / pose_rays — the quaternion-to-rotation and pinhole ray construction of the reference's camera
    refinement, restated (src/nerf_func.py:45-66, 91-112, 115-179 with nerf_coordinate=False, no normalisation).
"""
import numpy as np
import torch

from . import neus_grad_oracle as ngo
from . import neus_oracle as no

F32 = np.float32


class TorchHashGrid64(ngo.TorchHashGrid):
    """the same encoding in float64: the value of each cell fraction is the float32 one (pos = fmaf(scale, x, 0.5) in
    float32, as the forward kernel computes it), its derivative is scale; weights, table and sums are float64"""

    def forward(self, x):
        x = x.double()
        table = ngo._ste_half(self.params.double()).view(-1, no.N_FEAT)
        outs = []
        for m in self.metas:
            lin = x * float(m["scale"])
            pos = (lin.detach() + 0.5).to(torch.float32).double()
            fl = torch.floor(pos)
            fr = (pos - fl) + (lin - lin.detach())
            pg = fl.to(torch.int64).numpy().astype(np.uint32)
            acc = 0
            with np.errstate(over="ignore"):
                for idx in range(8):
                    w = 1.0
                    c = []
                    for d in range(3):
                        if (idx >> d) & 1:
                            w = w * fr[:, d]
                            c.append(pg[:, d] + np.uint32(1))
                        else:
                            w = w * (1.0 - fr[:, d])
                            c.append(pg[:, d])
                    gi = torch.from_numpy(m["offset"] + no._grid_index(m, *c))
                    acc = acc + w[:, None] * table[gi]
            outs.append(acc)
        return torch.cat(outs, dim=1)


def sample_positions(rays_o, rays_d, z_mid):
    """p = o + z d per sample [R,S,3], op by op in the inputs' precision (float32: what the forward kernel computes)"""
    o, d, z = np.asarray(rays_o), np.asarray(rays_d), np.asarray(z_mid)
    return o[:, None, :] + (d[:, None, :] * z[..., None]).astype(z.dtype)


def normalise(p, bound):
    """(x, dscale, x01): x = clamp((p - b0)/(b1 - b0) 2 - 1, -1, 1) op by op in p's precision, dscale = 2/(b1 - b0) where the
    clamp passes the gradient (bounds included, as torch.clamp's backward) else 0, x01 = (x + 1)/2"""
    b = np.asarray(bound, p.dtype).reshape(3, 2)
    b0, b1 = b[:, 0], b[:, 1]
    one, two = p.dtype.type(1.0), p.dtype.type(2.0)
    raw = (p - b0) / (b1 - b0) * two - one
    x = np.clip(raw, -one, one)
    dscale = np.where((raw >= -1.0) & (raw <= 1.0), 2.0 / (b1.astype(np.float64) - b0), 0.0)
    return x, dscale, (x + one) / two


def ray_backward_closed_form(rays_o, rays_d, z_mid, inb, bound, table, w_sdf, color_B, d_enc, d_xyz, dE, d_grad, d_true_cos,
                             gy=None):
    """dL/d rays_o [R,3] and dL/d rays_d [R,3] in float64 for one call of InstantNeuS.forward.
    Inputs per sample [R,S,...]: z_mid (z_vals + dists/2, no gradient), inb (the samples the forward put through the
    network), d_enc [.,32] = dL/d encoding, d_xyz [.,3] = dL/d x through sdf_layer's include_xyz columns, dE [.,33] =
    dL/d(p . B_j), d_grad [.,3] = dL/d normal (all paths), d_true_cos [.] = dL/d(d . normal) through get_alpha alone.
    table [entries,2] (the f16 values), w_sdf [32,35], color_B [3,33]; gy = what the normal contracts the encoding with
    (default: W_sdf[0,3:] rounded to half, as the forward kernel).  With x01 = u and pos_l = scale_l u + 1/2:
      normal_a = (W0[a] + 1/2 genc_a) dscale_a,  genc_a = sum_l scale_l dF_l/dpos_a,  F_l = trilinear(table_l . gy_l)
      dL/dp_a = dscale_a (d_xyz_a + 1/2 sum_l scale_l dG_l/dpos_a
                          + 1/2 sum_l scale_l^2 sum_{b != a} q_b d2F_l/dpos_a dpos_b) + sum_j dE_j B[a,j]
    with G_l = trilinear(table_l . d_enc_l) and q_b = 1/2 dscale_b d_grad_b; the trilinear interpolant has no pure second
    derivative, d2w_c/du_a du_b = (+-1)(+-1) w_c(third axis).  Then dL/do = sum_s dL/dp_s and
    dL/dd = sum_s z_s dL/dp_s + sum_s d_true_cos_s normal_s."""
    f8 = np.float64
    p = sample_positions(rays_o, rays_d, z_mid)
    R, S = p.shape[:2]
    n = R * S
    x, dscale, x01 = normalise(p.reshape(n, 3), bound)
    tab = np.asarray(table).astype(f8).reshape(-1, 2)
    w_sdf = np.asarray(w_sdf, f8)
    gy = np.asarray(w_sdf[0, 3:], np.float32).astype(np.float16).astype(f8) if gy is None else np.asarray(gy, f8)
    d_enc = np.asarray(d_enc, f8).reshape(n, 32)
    q = 0.5 * dscale * np.asarray(d_grad, f8).reshape(n, 3)
    g1, g2, genc = np.zeros((n, 3)), np.zeros((n, 3)), np.zeros((n, 3))
    metas, _ = no.hashgrid_meta()
    with np.errstate(over="ignore"):
        for l, m in enumerate(metas):
            pg, fr, scale = no._pos(m, np.asarray(x01))
            fr, scale = fr.astype(f8), float(scale)
            for idx in range(8):
                bits = [(idx >> a) & 1 for a in range(3)]
                sg = [1.0 if bits[a] else -1.0 for a in range(3)]
                wa = [fr[:, a] if bits[a] else 1.0 - fr[:, a] for a in range(3)]
                v = tab[m["offset"] + no._grid_index(m, *[pg[:, a] + np.uint32(bits[a]) for a in range(3)])]
                cg = v @ gy[2 * l:2 * l + 2]
                cd = (v * d_enc[:, 2 * l:2 * l + 2]).sum(1)
                for a in range(3):
                    b, c = (a + 1) % 3, (a + 2) % 3
                    dw = sg[a] * wa[b] * wa[c]
                    g1[:, a] += scale * cd * dw
                    genc[:, a] += scale * cg * dw
                    g2[:, a] += scale * scale * cg * sg[a] * (q[:, b] * sg[b] * wa[c] + q[:, c] * sg[c] * wa[b])
    dp = dscale * (np.asarray(d_xyz, f8).reshape(n, 3) + 0.5 * g1 + 0.5 * g2)
    dp = dp + np.asarray(dE, f8).reshape(n, -1)[:, :33] @ np.asarray(color_B, f8).T
    nrm = (w_sdf[0, :3] + 0.5 * genc) * dscale
    m = np.asarray(inb, bool).reshape(n, 1)
    dp, nrm = np.where(m, dp, 0.0).reshape(R, S, 3), np.where(m, nrm, 0.0).reshape(R, S, 3)
    z = np.asarray(z_mid, f8)
    d_o = dp.sum(1)
    d_d = (z[..., None] * dp).sum(1) + (np.asarray(d_true_cos, f8).reshape(R, S, 1) * nrm).sum(1)
    return d_o, d_d


def quat_to_rotation(quad):
    """[B,4] (r, i, j, k), not necessarily unit -> [B,3,3] (src/nerf_func.py:45-66): 2/|q|^2 scaling, torch, differentiable"""
    r, i, j, k = quad[:, 0], quad[:, 1], quad[:, 2], quad[:, 3]
    two_s = 2.0 / (quad * quad).sum(-1)
    rows = [1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
            two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
            two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)]
    return torch.stack(rows, dim=-1).reshape(-1, 3, 3)


def pose_rays(quadt, px, py, fx, fy, cx, cy):
    """rays of pixels (px, py) [N] from one quaternion-translation leaf quadt [7] = (r, i, j, k, tx, ty, tz)
    (src/nerf_func.py:91-112 quaternion_to_Rt, :166-179 build_rays with nerf_coordinate=False, unnormalised):
    rays_d = [(x - cx)/fx, (y - cy)/fy, 1] R^T, rays_o = t"""
    R = quat_to_rotation(quadt[None, :4])[0]
    dirs = torch.stack([(px - cx) / fx, (py - cy) / fy, torch.ones_like(px)], dim=-1).to(quadt.dtype)
    rays_d = dirs @ R.t()
    rays_o = quadt[4:].reshape(1, 3).repeat(px.shape[0], 1)
    return rays_o, rays_d
