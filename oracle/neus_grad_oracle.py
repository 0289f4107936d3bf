"""CPU oracle (TEST INFRASTRUCTURE — never imported by the product path) for the renderer BACKWARD
(SURVEY 8f-3): differentiable torch restatements of the two tiny-cuda-nn modules InstantNeuS uses
(src/InstantNeuS.py:62 `tcnn.Encoding` HashGrid, :201 `tcnn.Network` FullyFusedMLP), so that the REFERENCE's own
InstantNeuS.forward — including its `torch.autograd.grad(..., create_graph=True)` normal (:139-146) — and the losses of
Mapper.optimize_map (src/mapping.py:97-128) can be differentiated by plain autograd.

PARITY UNPINNED for tiny-cuda-nn's own backward arithmetic (no version pin, source absent: see oracle/neus_oracle.py):
what is restated is the mathematical gradient of the published forward algorithm, with fp16 ROUNDING treated as the
identity in the backward pass (straight-through), which is also what tcnn's mixed-precision backward amounts to.
Everything outside tcnn is the reference's own code (tests/golden/make_golden.py neus_grad imports it).
"""
import numpy as np
import torch

from . import neus_oracle as no


def _ste_half(x):
    """value rounded to fp16, gradient of the identity"""
    return x + (x.detach().half().to(x.dtype) - x.detach())


class TorchHashGrid(torch.nn.Module):
    """tcnn.Encoding(HashGrid, 16 levels x 2 features, T = 2^19, base 16, per-level scale 1.4473): fp32 master params,
    fp16 values at use; trilinear interpolation; differentiable w.r.t. the params AND the input (twice)."""

    def __init__(self, n_input_dims=3, encoding_config=None):
        super().__init__()
        self.metas, total = no.hashgrid_meta()
        self.n_output_dims = no.N_LEVELS * no.N_FEAT
        self.params = torch.nn.Parameter((torch.rand(total * 2) * 2 - 1) * 1e-4)

    def forward(self, x):
        table = _ste_half(self.params).view(-1, no.N_FEAT)
        outs = []
        for m in self.metas:
            pos = (x.double() * float(m["scale"]) + 0.5).to(torch.float32)          # fmaf(scale, x, 0.5)
            fl = torch.floor(pos).detach()
            fr = pos - fl
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


class TorchMLP(torch.nn.Module):
    """tcnn.Network(FullyFusedMLP 67 -> 64 -> 64 -> 3): input padded to 80 with ones, output padded to 16, no biases,
    ReLU, fp16 weights and activations (straight-through), fp32 accumulation."""

    def __init__(self, n_input_dims=67, n_output_dims=3, network_config=None):
        super().__init__()
        self.params = torch.nn.Parameter(torch.zeros(64 * 80 + 64 * 64 + 16 * 64))

    def forward(self, x):
        p = _ste_half(self.params)
        W1 = p[:64 * 80].view(64, 80)
        W2 = p[64 * 80:64 * 80 + 64 * 64].view(64, 64)
        W3 = p[64 * 80 + 64 * 64:].view(16, 64)
        xin = torch.cat([x.float(), torch.ones(x.shape[0], 13)], dim=1)
        h = _ste_half(torch.relu(_ste_half(xin) @ W1.t()))
        h = _ste_half(torch.relu(h @ W2.t()))
        return _ste_half(h @ W3.t())[:, :3]


def mapping_loss(net, out, rays_color, rays_depth, w_color=1.0, w_sdf=None, w_eikonal=None):
    """the loss of Mapper.optimize_map (src/mapping.py:97-128) with uncertainty_based off; `net` supplies
    compute_sdf_error (the reference's own method when `net` is the reference class)."""
    rays_depth = rays_depth.reshape(-1, 1)
    valid = (rays_depth > 0).reshape(-1)
    total = torch.abs(out["color"][valid] - rays_color[valid]).mean() * w_color
    total = total + torch.abs(out["depth"][valid] - rays_depth[valid]).mean()
    if w_sdf:
        sdf_loss, sparse_loss = net.compute_sdf_error(sdf=out["sdf"][valid], z_vals=out["z_vals"][valid], gt_depth=rays_depth[valid])
        total = total + (sdf_loss + sparse_loss) * w_sdf
    if w_eikonal:
        total = total + w_eikonal * out["gradient_error"].mean()
    return total


def composite_backward_closed_form(alpha, rgb, sdf, grad, z_mid, dists, dirs, inb, inv_s, d_color, d_depth, d_sdf, d_gerr,
                                   cos_anneal_ratio=1.0, total_samples=None):
    """The closed form neus_composite_bwd_kernel implements (csrc/neus.cu), in float64 numpy, for ONE call of
    InstantNeuS.forward: given the per-sample alpha / rgb (after the sigmoid) / sdf / normal the forward produced and the
    upstream gradients of color [R,3], depth [R,1], sdf [R,S] and gradient_error (scalar), returns
    (d_mlp_out [R,S,3] w.r.t. the colour network's pre-sigmoid output, d_sdf_out [R,S], d_normal [R,S,3], d_inv_s).
      weights w_s = alpha_s T_s, T_s = prod_{j<s}(1 - alpha_j + 1e-7)
      G_s = dL/dw_s = d_color . rgb_s + d_depth z_s
      dL/dalpha_s = G_s T_s - (sum_{k>s} G_k w_k) / (1 - alpha_s + 1e-7)
      alpha = clip((p - n + 1e-5)/(p + 1e-5), 0, 1), p = sigmoid((sdf - h) inv_s), n = sigmoid((sdf + h) inv_s),
      h = iter_cos * dist / 2, iter_cos = -(relu(-tc/2 + 1/2)(1 - car) + relu(-tc) car), tc = dir . normal
      gradient_error = mean over ALL samples of (|normal| - 1)^2 [in bound]
    total_samples: the number of samples gradient_error averages over when these rays are a slice of a larger call
    (default R*S).  d_color / d_depth / d_gerr may be None (zero)."""
    R0, S0 = np.shape(alpha)
    d_color = np.zeros((R0, 3)) if d_color is None else d_color
    d_depth = np.zeros((R0, 1)) if d_depth is None else d_depth
    d_gerr = 0.0 if d_gerr is None else float(d_gerr)
    total_samples = R0 * S0 if total_samples is None else total_samples
    f8 = np.float64
    alpha, rgb, sdf, grad, z_mid, dists, dirs = [np.asarray(x, f8) for x in (alpha, rgb, sdf, grad, z_mid, dists, dirs)]
    inb = np.asarray(inb, bool)
    R, S = alpha.shape
    T = np.cumprod(np.concatenate([np.ones((R, 1)), 1.0 - alpha + 1e-7], axis=1), axis=1)[:, :-1]
    w = alpha * T
    G = (rgb * np.asarray(d_color, f8)[:, None, :]).sum(-1) + np.asarray(d_depth, f8).reshape(R, 1) * z_mid
    gw = G * w
    suffix = gw.sum(1, keepdims=True) - np.cumsum(gw, axis=1)
    d_alpha = G * T - suffix / (1.0 - alpha + 1e-7)
    d_x = np.asarray(d_color, f8)[:, None, :] * w[..., None] * rgb * (1.0 - rgb)
    tc = (dirs[:, None, :] * grad).sum(-1)
    r0, r1 = -tc * 0.5 + 0.5, -tc
    car = cos_anneal_ratio
    iter_cos = -(np.maximum(r0, 0) * (1 - car) + np.maximum(r1, 0) * car)
    h = iter_cos * dists / 2.0
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))      # noqa: E731
    p, n = sig((sdf - h) * inv_s), sig((sdf + h) * inv_s)
    araw = (p - n + 1e-5) / (p + 1e-5)
    passes = (araw >= 0) & (araw <= 1) & inb
    d_p = d_alpha * n / (p + 1e-5) ** 2
    d_n = -d_alpha / (p + 1e-5)
    d_ap, d_an = d_p * p * (1 - p), d_n * n * (1 - n)
    d_sdf_out = np.where(passes, (d_ap + d_an) * inv_s, 0.0)
    d_h = np.where(passes, (d_an - d_ap) * inv_s, 0.0)
    d_inv_s = np.where(passes, d_ap * (sdf - h) + d_an * (sdf + h), 0.0).sum()
    d_tc = d_h * dists / 2.0 * ((r0 > 0) * 0.5 * (1 - car) + (r1 > 0) * car)
    d_normal = d_tc[..., None] * dirs[:, None, :]
    gn = np.linalg.norm(grad, axis=-1)
    eik = d_gerr / total_samples * 2.0 * (gn - 1.0) / np.where(gn > 0, gn, 1.0)
    d_normal = d_normal + np.where((gn > 0)[..., None], eik[..., None] * grad, 0.0)
    if d_sdf is not None:
        d_sdf_out = d_sdf_out + np.asarray(d_sdf, f8)
    m = inb[..., None]
    return np.where(m, d_x, 0.0), np.where(inb, d_sdf_out, 0.0), np.where(m, d_normal, 0.0), d_inv_s


def grid_backward_closed_form(x01, table, d_enc, q, gy, with_abs=False):
    """The closed form neus_grid_bwd_kernel implements (csrc/neus.cu), float64 numpy.  For samples x01 [n,3] in [0,1],
    table [entries,2] (fp16 values), d_enc [n,32] = dL/d(encoding), q [n,3] = dL/d(d sdf / d x01) (the upstream gradient of
    the input-gradient of the scalar field enc . gy), gy [32]:
      L = sum_n d_enc . enc(x) + q . d/dx [enc(x) . gy]
    returns (dL/d table [entries,2], dL/d gy [32]).  Per level l, corner c with trilinear weight w_c and index i_c:
      dL/d table[i_c, f] += d_enc[2l+f] w_c + gy[2l+f] scale_l (q . grad_u w_c),
      dL/d gy[2l+f]      += scale_l sum_c table[i_c, f] (q . grad_u w_c),
    grad_u w_c along axis a = (+1 if the corner takes the upper cell face on a else -1) x the other two axes' weights.
    with_abs=True also returns, per entry and feature, the sum of |contribution| over the samples and corners that touch
    it (with sdot's three axis terms summed unsigned), and per gy entry the same sum of |table value x sdot|: the scale
    against which fp32 arithmetic and a reduction in any order are measured."""
    f8 = np.float64
    metas, _ = no.hashgrid_meta()
    x01 = np.asarray(x01, np.float32)
    tab = np.asarray(table).astype(f8)
    d_enc, q, gy = np.asarray(d_enc, f8), np.asarray(q, f8), np.asarray(gy, f8)
    g_tab = np.zeros_like(tab)
    g_gy = np.zeros(32, f8)
    a_tab = np.zeros_like(tab)
    a_gy = np.zeros(32, f8)
    with np.errstate(over="ignore"):
        for l, m in enumerate(metas):
            pg, fr, scale = no._pos(m, x01)
            fr = fr.astype(f8)
            for idx in range(8):
                bits = [(idx >> d) & 1 for d in range(3)]
                wa = [fr[:, d] if bits[d] else 1.0 - fr[:, d] for d in range(3)]
                w = wa[0] * wa[1] * wa[2]
                sdot = float(scale) * ((1 if bits[0] else -1) * q[:, 0] * wa[1] * wa[2] + (1 if bits[1] else -1) * q[:, 1] * wa[0] * wa[2]
                                       + (1 if bits[2] else -1) * q[:, 2] * wa[0] * wa[1])
                gi = m["offset"] + no._grid_index(m, *[pg[:, d] + np.uint32(bits[d]) for d in range(3)])
                for f in range(2):
                    contrib = d_enc[:, 2 * l + f] * w + gy[2 * l + f] * sdot
                    np.add.at(g_tab[:, f], gi, contrib)
                    g_gy[2 * l + f] += (tab[gi, f] * sdot).sum()
                    if with_abs:
                        # sdot's three terms are each ~scale |q| and may cancel: their unsigned sum is the fp32 scale
                        sabs = float(scale) * (np.abs(q[:, 0]) * wa[1] * wa[2] + np.abs(q[:, 1]) * wa[0] * wa[2]
                                               + np.abs(q[:, 2]) * wa[0] * wa[1])
                        np.add.at(a_tab[:, f], gi, np.abs(d_enc[:, 2 * l + f] * w) + np.abs(gy[2 * l + f]) * sabs)
                        a_gy[2 * l + f] += (np.abs(tab[gi, f]) * sabs).sum()
    if with_abs:
        return g_tab, g_gy, a_tab, a_gy
    return g_tab, g_gy
