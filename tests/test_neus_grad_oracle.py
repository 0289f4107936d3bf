"""CPU: the differentiable tcnn restatements of oracle/neus_grad_oracle.py are pinned to the forward oracle
(oracle/neus_oracle.py, itself pinned to the reference golden), and the compute_sdf_error mirror to the values the
REFERENCE's method produced inside tests/golden/neus_grad.npz."""
import os

import numpy as np
import torch

from oracle import neus_grad_oracle as ngo
from oracle import neus_oracle as no


def test_torch_hashgrid_matches_numpy_oracle_and_its_input_gradient():
    torch.manual_seed(0)
    enc = ngo.TorchHashGrid()
    with torch.no_grad():
        enc.params.copy_(torch.randn(enc.params.numel()) * 0.05)
    x = torch.rand(200, 3, requires_grad=True)
    y = enc(x)
    table = enc.params.detach().half().numpy().reshape(-1, 2)
    want = no.hashgrid_encode(x.detach().numpy(), table).astype(np.float32)
    assert np.abs(y.detach().numpy() - want).max() <= 2e-3 * np.abs(want).max()       # half accumulation in the oracle
    gy = torch.randn(32)
    (gx,) = torch.autograd.grad((y * gy).sum(), x)
    want_g = no.hashgrid_input_grad(x.detach().numpy(), table, gy.numpy())
    assert np.abs(gx.numpy() - want_g).max() <= 2e-3 * np.abs(want_g).max()


def test_torch_mlp_matches_numpy_oracle():
    torch.manual_seed(1)
    mlp = ngo.TorchMLP()
    with torch.no_grad():
        mlp.params.copy_(torch.randn(mlp.params.numel()) * 0.2)
    x = torch.randn(100, 67)
    got = mlp(x).detach().numpy()
    want = no.mlp_forward(x.numpy(), mlp.params.detach().half().numpy()).astype(np.float32)
    assert np.abs(got - want).max() <= 4e-3 * max(1.0, np.abs(want).max())


def test_compute_sdf_error_mirror_matches_reference_values():
    from goslam_b200 import neus, synthetic
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "neus_grad.npz"))
    cfg = synthetic.NEUS_CFG

    class Shell:                      # the method only reads two config numbers
        sdf_truncation, sdf_sparse_factor = cfg["sdf_truncation"], cfg["sdf_sparse_factor"]
    depth = torch.from_numpy(g["rays_depth"]).reshape(-1, 1)
    valid = (depth > 0).reshape(-1)
    sdf_loss, sparse_loss = neus.InstantNeuS.compute_sdf_error(Shell, torch.from_numpy(g["out_sdf"])[valid],
                                                               torch.from_numpy(g["out_z_vals"])[valid], depth[valid])
    assert abs(float(sdf_loss) - float(g["parts"][2])) <= 1e-5 * abs(float(g["parts"][2]))
    assert abs(float(sparse_loss) - float(g["parts"][3])) <= 1e-5 * max(abs(float(g["parts"][3])), 1e-3)


def test_composite_backward_closed_form_matches_autograd():
    """the closed form the CUDA compositing / alpha backward kernel implements == autograd through the reference's
    get_alpha + compositing + eikonal code path (src/InstantNeuS.py:276-293,343-358), in float64"""
    torch.manual_seed(5)
    R, S = 7, 40
    dd = torch.float64
    sdf = (torch.randn(R, S, dtype=dd) * 0.3).requires_grad_(True)
    grad = (torch.randn(R, S, 3, dtype=dd) * 0.8).requires_grad_(True)
    x = torch.randn(R, S, 3, dtype=dd).requires_grad_(True)                 # colour network output before the sigmoid
    log_inv_s = torch.tensor(2.0, dtype=dd, requires_grad=True)
    z = torch.sort(torch.rand(R, S, dtype=dd) * 3 + 0.2, dim=1)[0]
    dists = torch.rand(R, S, dtype=dd) * 0.1 + 0.01
    dirs = torch.randn(R, 3, dtype=dd)
    inb = torch.rand(R, S) > 0.15
    inv_s = torch.exp(log_inv_s)
    g_m = grad * inb[..., None]                      # out-of-bound samples: normal 0, sdf 100, rgb 0 (constants)
    s_m = torch.where(inb, sdf, torch.full_like(sdf, 100.0))
    true_cos = (dirs[:, None, :] * g_m).sum(-1)
    iter_cos = -torch.relu(-true_cos)
    est_next, est_prev = s_m + iter_cos * dists / 2.0, s_m - iter_cos * dists / 2.0
    prev_cdf, next_cdf = torch.sigmoid(est_prev * inv_s), torch.sigmoid(est_next * inv_s)
    alpha = ((prev_cdf - next_cdf + 1e-5) / (prev_cdf + 1e-5)).clip(0.0, 1.0) * inb
    rgb = torch.sigmoid(x) * inb[..., None]
    w = alpha * torch.cumprod(torch.cat([torch.ones(R, 1, dtype=dd), 1 - alpha + 1e-7], dim=1), dim=1)[:, :-1]
    color, depth = (rgb * w[..., None]).sum(1), (z * w).sum(1, keepdim=True)
    gerr = (((torch.linalg.norm(g_m, dim=2) - 1.0) ** 2) * inb).mean()
    dc, ddp, ds = torch.randn(R, 3, dtype=dd), torch.randn(R, 1, dtype=dd), torch.randn(R, S, dtype=dd) * 0.1
    (((color * dc).sum() + (depth * ddp).sum() + (s_m * ds * inb).sum() + 3.0 * gerr)).backward()
    got = ngo.composite_backward_closed_form(alpha.detach().numpy(), rgb.detach().numpy(), s_m.detach().numpy(), g_m.detach().numpy(),
                                             z.numpy(), dists.numpy(), dirs.numpy(), inb.numpy(), float(inv_s), dc.numpy(), ddp.numpy(),
                                             (ds * inb).numpy(), 3.0)
    m = inb.numpy()
    assert np.allclose(got[0], x.grad.numpy() * m[..., None], rtol=1e-9, atol=1e-12)
    assert np.allclose(got[1], sdf.grad.numpy(), rtol=1e-9, atol=1e-12)
    assert np.allclose(got[2], grad.grad.numpy(), rtol=1e-9, atol=1e-12)
    assert abs(got[3] * float(inv_s) - float(log_inv_s.grad)) <= 1e-9 * abs(float(log_inv_s.grad))


def test_grid_backward_closed_form_matches_double_backward_autograd():
    """the scatter formula of the CUDA hash-grid backward, including the SECOND-ORDER term (the normal is the input
    gradient of enc . W0), == autograd with create_graph=True through the differentiable hash grid"""
    torch.manual_seed(9)
    enc = ngo.TorchHashGrid()
    with torch.no_grad():
        enc.params.copy_((torch.randn(enc.params.numel()) * 0.05).half().float())      # fp16-representable: no rounding term
    n = 150
    x = torch.rand(n, 3, requires_grad=True)
    gy = (torch.randn(32) * 0.3).requires_grad_(True)
    d_enc, q = torch.randn(n, 32), torch.randn(n, 3)
    y = enc(x)
    (gx,) = torch.autograd.grad((y * gy).sum(), x, create_graph=True)
    ((y * d_enc).sum() + (gx * q).sum()).backward()
    g_tab, g_gy = ngo.grid_backward_closed_form(x.detach().numpy(), enc.params.detach().numpy().reshape(-1, 2), d_enc.numpy(), q.numpy(),
                                                gy.detach().numpy())
    want_tab = enc.params.grad.numpy().reshape(-1, 2)
    assert np.abs(g_tab - want_tab).max() <= 2e-4 * np.abs(want_tab).max()               # the autograd side runs in float32
    # dL/dgy has the first-order part sum_n enc * 0 (none: d_enc does not multiply gy) and the second-order part only
    assert np.abs(g_gy - gy.grad.numpy()).max() <= 2e-4 * np.abs(gy.grad.numpy()).max()


def test_closed_form_options_for_the_kernel_tests():
    """the options the per-kernel GPU tests use: a ray slice of a larger call (total_samples), upstream gradients passed
    as None, and the per-entry sum of |contribution| of the grid scatter"""
    rng = np.random.default_rng(4)
    R, S = 9, 20
    alpha = rng.uniform(0, 0.4, (R, S))
    rgb = rng.uniform(0.05, 0.95, (R, S, 3))
    sdf, grad = rng.normal(0, 0.3, (R, S)), rng.normal(0, 0.8, (R, S, 3))
    z = np.sort(rng.uniform(0.2, 3, (R, S)), axis=1)
    dists, dirs = rng.uniform(0.01, 0.1, (R, S)), rng.normal(0, 1, (R, 3))
    inb = rng.uniform(size=(R, S)) > 0.2
    dc, dd, ds = rng.normal(size=(R, 3)), rng.normal(size=(R, 1)), rng.normal(size=(R, S))
    full = ngo.composite_backward_closed_form(alpha, rgb, sdf, grad, z, dists, dirs, inb, 7.0, dc, dd, ds, 2.5)
    sl = slice(3, 7)
    part = ngo.composite_backward_closed_form(alpha[sl], rgb[sl], sdf[sl], grad[sl], z[sl], dists[sl], dirs[sl], inb[sl], 7.0,
                                              dc[sl], dd[sl], ds[sl], 2.5, total_samples=R * S)
    for a, b in zip(part[:3], full[:3]):
        np.testing.assert_allclose(a, b[sl], rtol=1e-12, atol=1e-15)
    none = ngo.composite_backward_closed_form(alpha, rgb, sdf, grad, z, dists, dirs, inb, 7.0, None, None, None, None)
    zero = ngo.composite_backward_closed_form(alpha, rgb, sdf, grad, z, dists, dirs, inb, 7.0, np.zeros((R, 3)),
                                              np.zeros((R, 1)), None, 0.0)
    for a, b in zip(none, zero):
        np.testing.assert_array_equal(a, b)
    assert not np.any(none[0]) and not np.any(none[2]) and none[3] == 0.0

    table = (rng.normal(0, 0.05, (no.hashgrid_meta()[1], 2))).astype(np.float16)
    x01 = rng.uniform(0, 1, (40, 3)).astype(np.float32)
    x01[:10] = x01[0]                                        # ten samples on the same point: shared entries
    d_enc, q, gy = rng.normal(size=(40, 32)), rng.normal(size=(40, 3)), rng.normal(size=32)
    g_tab, g_gy = ngo.grid_backward_closed_form(x01, table, d_enc, q, gy)
    g2, gy2, a_tab, a_gy = ngo.grid_backward_closed_form(x01, table, d_enc, q, gy, with_abs=True)
    np.testing.assert_array_equal(g_tab, g2)
    np.testing.assert_array_equal(g_gy, gy2)
    assert np.all(a_tab >= np.abs(g_tab)) and np.all(a_gy >= np.abs(g_gy))
    assert np.array_equal(a_tab != 0, g_tab != 0)            # touched entries (a zero sum of non-zero terms is measure-zero)
    # with no normal term and non-negative d_enc every contribution is non-negative: the two sums coincide
    g3, _, a3, _ = ngo.grid_backward_closed_form(x01, table, np.abs(d_enc), np.zeros_like(q), gy, with_abs=True)
    np.testing.assert_allclose(a3, g3, rtol=1e-12, atol=0)
