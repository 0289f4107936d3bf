"""Renderer backward (SURVEY 8f-3) on the GPU: InstantNeuS.forward under grad + loss.backward() through
goslam_neus_composite_backward / cuBLAS GEMMs / goslam_neus_grid_backward against
  (1) tests/golden/neus_grad.npz — the REFERENCE's InstantNeuS.forward + the Mapper.optimize_map loss differentiated by
      autograd (tests/golden/make_golden.py neus_grad; tcnn modules = differentiable restatements), and
  (2) central finite differences of the CUDA forward itself on the fp32 parameters.
Tolerances: the kernel rounds the encoding, the colour network's activations and the colours to fp16 (like tcnn), the
golden graph is fp32 with straight-through fp16 rounding; gradients agree to a few 1e-3 relative — asserted: relative
L2 error <= 2e-2 and cosine >= 0.9995 per parameter tensor."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def _net(seed, bound, rt_bound):
    from goslam_b200 import neus, synthetic
    offs, ress, _, total = neus.hashgrid_layout()
    w = synthetic.make_neus_weights(seed=seed, total_grid_params=total, layout=(offs, ress))
    net = neus.InstantNeuS(synthetic.NEUS_CFG, bound)
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to(dev())
    net.update_bound(torch.as_tensor(rt_bound))
    return net


def _mapping_loss(net, out, rays_color, rays_depth):
    """src/mapping.py:97-128 with the weights of configs/go_slam.yaml (uncertainty weighting on)"""
    depth = rays_depth.reshape(-1, 1)
    valid = (depth > 0).reshape(-1)
    unc = 1.0 / torch.sqrt(out["depth_variance"][valid].detach() + 1e-10)
    color_loss = torch.abs(out["color"][valid] - rays_color[valid]).mean()
    depth_loss = (torch.abs(out["depth"][valid] - depth[valid]) * unc).mean()
    sdf_loss, sparse_loss = net.compute_sdf_error(sdf=out["sdf"][valid], z_vals=out["z_vals"][valid], gt_depth=depth[valid])
    total = color_loss * 2.0 + depth_loss * 1.0 + (sdf_loss + sparse_loss) * 2.0 + 0.1 * out["gradient_error"].mean()
    return total, (color_loss, depth_loss, sdf_loss, sparse_loss, out["gradient_error"].mean())


def _cmp(name, got, want, rel_tol=2e-2, cos_tol=0.9995):
    got, want = np.asarray(got, np.float64).reshape(-1), np.asarray(want, np.float64).reshape(-1)
    rel = np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30)
    cos = float(got @ want) / max(np.linalg.norm(got) * np.linalg.norm(want), 1e-30)
    print("%-10s |want| %.4e  rel L2 err %.3e  cos %.6f" % (name, np.linalg.norm(want), rel, cos))
    assert rel <= rel_tol and cos >= cos_tol, (name, rel, cos)


def _golden_run():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "neus_grad.npz"))
    net = _net(int(g["weights_seed"]), g["bound"].tolist(), g["rt_bound"])
    args = [torch.from_numpy(g[k]).to(dev()) for k in ("rays_o", "rays_d", "z_vals_in", "dists")]
    with torch.enable_grad():
        out = net(*args)
        total, parts = _mapping_loss(net, out, torch.from_numpy(g["rays_color"]).to(dev()), torch.from_numpy(g["rays_depth"]).to(dev()))
    return g, net, out, total, parts


def test_training_forward_matches_reference_golden():
    g, net, out, total, parts = _golden_run()
    assert out["color"].requires_grad and out["depth"].requires_grad and out["sdf"].requires_grad and out["gradient_error"].requires_grad
    assert not out["depth_variance"].requires_grad
    for k in ("color", "depth", "depth_variance", "weight_sum", "z_vals"):
        want = g["out_" + k]
        got = out[k].detach().cpu().numpy().reshape(want.shape)
        assert np.abs(got - want).max() <= 2e-3 * max(1.0, np.abs(want).max()), k
    assert abs(float(total.detach()) - float(g["loss"])) <= 2e-3 * abs(float(g["loss"]))
    for a, b in zip(parts, g["parts"]):
        assert abs(float(a) - float(b)) <= 3e-3 * max(abs(float(b)), 1e-2)


def test_backward_matches_reference_autograd_golden():
    g, net, out, total, _ = _golden_run()
    total.backward()
    grid_grad = net.sdf_network.encoding.encoding.params.grad.cpu().numpy()
    want_grid = np.zeros_like(grid_grad)
    want_grid[g["grid_grad_idx"]] = g["grid_grad_val"]
    _cmp("grid", grid_grad, want_grid)
    # the scatter touches exactly the entries autograd touches (entries whose gradient is exactly 0.0 in fp32 may differ)
    touched = np.nonzero(grid_grad)[0]
    assert np.setdiff1d(touched, g["grid_grad_idx"]).size <= 0.01 * touched.size
    _cmp("sdf_w", net.sdf_network.sdf_layer.weight.grad.cpu().numpy(), g["g_sdf_w"])
    _cmp("sdf_w[0]", net.sdf_network.sdf_layer.weight.grad.cpu().numpy()[0], g["g_sdf_w"][0])     # the second-order row
    _cmp("sdf_b", net.sdf_network.sdf_layer.bias.grad.cpu().numpy(), g["g_sdf_b"])
    _cmp("color_B", net.color_network._B.grad.cpu().numpy(), g["g_color_B"])
    _cmp("mlp", net.color_network.network.params.grad.cpu().numpy(), g["g_mlp"])
    gv, wv = float(net.variance_network.variance.grad), float(g["g_variance"])
    print("variance   got %.6e want %.6e" % (gv, wv))
    assert abs(gv - wv) <= 2e-2 * abs(wv)
    assert net.sdf_network.encoding._B.grad is None          # unused by the non-directional encoding, as in the reference


@pytest.mark.parametrize("term", ["color", "depth", "sdf", "eikonal", "all"])
def test_backward_matches_finite_differences_of_the_cuda_forward(term):
    """independent of any oracle: d loss / d theta for fp32 parameters against central differences of the fused forward,
    one loss term at a time (each exercises one upstream gradient of the backward) and all together"""
    from goslam_b200 import synthetic
    net = _net(5, [[-2.0, 2.0]] * 3, [[-1.9, 1.9], [-2.0, 2.0], [-1.7, 2.0]])
    ro, rd, zv, ds = [t.to(dev()) for t in synthetic.make_rays(256, S=48, seed=21, n_uniform=16)]
    gen = torch.Generator().manual_seed(3)
    cc = torch.randn(256, 3, generator=gen).to(dev()).double()
    cd = torch.randn(256, 1, generator=gen).to(dev()).double()
    cs = (0.05 * torch.randn(256, 48, generator=gen)).to(dev()).double()
    on = {k: float(term in (k, "all")) for k in ("color", "depth", "sdf", "eikonal")}

    def loss_of(out):                  # accumulated in float64: the differences below are ~1e-4 of the value
        inb = (out["sdf"] != 100.0).double()
        return (on["color"] * (out["color"].double() * cc).sum() + on["depth"] * (out["depth"].double() * cd).sum()
                + on["sdf"] * (out["sdf"].double() * inb * cs).sum() + on["eikonal"] * 50.0 * out["gradient_error"].double().sum())

    with torch.enable_grad():
        loss_of(net(ro, rd, zv, ds)).backward()
    # parameters whose effect does not pass through an fp16-quantised tensor first (the sdf / alpha / normal paths);
    # rows 1.. of sdf_layer feed the colour network's fp16 input row, where a 1e-3 step is below one ulp
    checks = [("sdf_b[0]", net.sdf_network.sdf_layer.bias, (0,), 1e-3), ("sdf_w[0,0]", net.sdf_network.sdf_layer.weight, (0, 0), 1e-3),
              ("sdf_w[0,1]", net.sdf_network.sdf_layer.weight, (0, 1), 1e-3), ("sdf_w[0,2]", net.sdf_network.sdf_layer.weight, (0, 2), 1e-3),
              ("variance", net.variance_network.variance, (), 1e-3)]
    if term in ("color", "all"):
        # d colour / d sdf_w[0,:3] runs through the NORMAL columns of the colour network's fp16 input row: a 1e-3 step
        # moves them by half an ulp, finite differences of that path are quantisation noise (measured: -8.44 vs -8.67,
        # 1.54 vs 1.15).  That path is pinned by the autograd golden above.
        checks = [c for c in checks if not c[0].startswith("sdf_w")]
    bad = []
    for name, prm, idx, eps in checks:
        an = float(prm.grad[idx])
        vals = []
        for sgn in (+1, -1):
            with torch.no_grad():
                old = prm[idx].clone()
                prm[idx] = old + sgn * eps
                vals.append(float(loss_of(net(ro, rd, zv, ds))))
                prm[idx] = old
        fd = (vals[0] - vals[1]) / (2 * eps)
        print("[%s] %-12s analytic %.5e  finite-diff %.5e" % (term, name, an, fd))
        if not abs(an - fd) <= 5e-2 * max(abs(fd), abs(an)) + 2e-3:
            bad.append((name, an, fd))
    assert not bad, bad


def test_adamw_trajectory_matches_the_reference_mapping_loop():
    """tests/golden/neus_adamw.npz: 8 iterations of Mapper.optimize_map's loop body (src/mapping.py:84-131) run by the
    REFERENCE's InstantNeuS (make_golden.py neus_adamw: uncertainty weighting off, learning rates x0.1).  Ours — the same
    torch.optim.AdamW / clip_grad_norm_ calls on our InstantNeuS, gradients from the CUDA backward — must follow the same
    loss trajectory: every step's total within 1 %, and it must decrease."""
    ga = np.load(os.path.join(os.path.dirname(__file__), "golden", "neus_adamw.npz"))
    g, net, _, _, _ = _golden_run()
    opt = torch.optim.AdamW([{"params": net.get_training_parameters(), "lr": float(ga["net_lr"])},
                             {"params": net.get_volume_parameters(), "lr": float(ga["grid_lr"])}],
                            betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    args = [torch.from_numpy(g[k]).to(dev()) for k in ("rays_o", "rays_d", "z_vals_in", "dists")]
    rc, rdp = torch.from_numpy(g["rays_color"]).to(dev()), torch.from_numpy(g["rays_depth"]).to(dev())
    depth = rdp.reshape(-1, 1)
    valid = (depth > 0).reshape(-1)
    losses = []
    for _ in range(ga["rows"].shape[0]):
        opt.zero_grad()
        with torch.enable_grad():
            out = net(*args)
            cl = torch.abs(out["color"][valid] - rc[valid]).mean()
            dl = torch.abs(out["depth"][valid] - depth[valid]).mean()
            sl, spl = net.compute_sdf_error(sdf=out["sdf"][valid], z_vals=out["z_vals"][valid], gt_depth=depth[valid])
            total = cl * 2.0 + dl * 1.0 + (sl + spl) * 2.0 + 0.1 * out["gradient_error"].mean()
        total.backward()
        torch.nn.utils.clip_grad_norm_(net.get_training_parameters() + net.get_volume_parameters(), max_norm=35.0)
        opt.step()
        losses.append(float(total.detach()))
    want = ga["rows"][:, 0]
    print("ours     :", " ".join("%.4f" % v for v in losses))
    print("reference:", " ".join("%.4f" % v for v in want))
    assert np.all(np.abs(np.array(losses) - want) <= 1e-2 * want)
    assert losses[-1] < 0.85 * losses[0]


def test_backward_is_independent_of_ray_chunking(monkeypatch):
    """the backward walks the rays in chunks (bounded activations); gradient_error's 1/(R*S) and every accumulated gradient
    must not depend on the chunk size.  R = 37 rays x S = 72 samples (three 32-sample warp chunks per ray, partial tiles)."""
    from goslam_b200 import neus, synthetic
    ro, rd, zv, ds = [t.to(dev()) for t in synthetic.make_rays(37, S=72, seed=29)]
    gen = torch.Generator().manual_seed(8)
    cc, cd = torch.randn(37, 3, generator=gen).to(dev()), torch.randn(37, 1, generator=gen).to(dev())
    grads = []
    for chunk in (1 << 16, 8):
        monkeypatch.setattr(neus._NeusFunction, "CHUNK_RAYS", chunk)
        net = _net(5, [[-2.0, 2.0]] * 3, [[-1.9, 1.9], [-2.0, 2.0], [-1.7, 2.0]])
        with torch.enable_grad():
            o = net(ro, rd, zv, ds)
            ((o["color"] * cc).sum() + (o["depth"] * cd).sum() + 0.01 * o["sdf"][o["sdf"] != 100.0].sum() + 30.0 * o["gradient_error"].sum()).backward()
        grads.append([p.grad.clone() for p in net.trainable_tensors()])
    for a, b in zip(*grads):
        scale = float(a.abs().max())
        assert scale > 0
        # different loss scales per chunk and a different summation order (fp16 operands on the colour network, fp32
        # reductions in scheduling order): a chunking bug (a wrong 1/(R*S), a dropped chunk) is an O(1) error, 1e-2 is ample
        assert float((a - b).abs().max()) <= 1e-2 * scale, (a.shape, float((a - b).abs().max()), scale)


GRAD_CASES = ["s24", "s48", "s72", "fallback"]


@pytest.mark.parametrize("tag", GRAD_CASES)
def test_backward_matches_reference_autograd_cases(tag):
    """tests/golden/neus_grad_cases.npz (make_golden.py neus_grad_cases): the reference's forward + loss + autograd at
    S = 24, 48, 72 and on a batch with no sample inside realtime_bound, where the reference forces its first 100 samples
    into the network and gradients flow through them.  Every parameter gradient: relative L2 <= 2e-2, cosine >= 0.9995."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "neus_grad_cases.npz"))
    c = {k[len(tag) + 1:]: g[k] for k in g.files if k.startswith(tag + "_")}
    net = _net(int(g["weights_seed"]), g["bound"].tolist(), c["rt_bound"])
    args = [torch.from_numpy(c[k]).to(dev()) for k in ("rays_o", "rays_d", "z_vals_in", "dists")]
    with torch.enable_grad():
        out = net(*args)
        total, _ = _mapping_loss(net, out, torch.from_numpy(c["rays_color"]).to(dev()), torch.from_numpy(c["rays_depth"]).to(dev()))
    for k in ("color", "depth", "weight_sum", "z_vals"):
        want = c["out_" + k]
        assert np.abs(out[k].detach().cpu().numpy().reshape(want.shape) - want).max() <= 2e-3 * max(1.0, np.abs(want).max()), k
    total.backward()
    grid_grad = net.sdf_network.encoding.encoding.params.grad.cpu().numpy()
    idx = np.cumsum(c["grid_grad_didx"].astype(np.int64))
    want_grid = np.zeros_like(grid_grad)
    want_grid[idx] = c["grid_grad_val"]
    _cmp("grid", grid_grad, want_grid)
    touched = np.nonzero(grid_grad)[0]
    assert np.setdiff1d(touched, idx).size <= 0.01 * touched.size
    _cmp("sdf_w", net.sdf_network.sdf_layer.weight.grad.cpu().numpy(), c["g_sdf_w"])
    _cmp("sdf_w[0]", net.sdf_network.sdf_layer.weight.grad.cpu().numpy()[0], c["g_sdf_w"][0])
    _cmp("sdf_b", net.sdf_network.sdf_layer.bias.grad.cpu().numpy(), c["g_sdf_b"])
    _cmp("color_B", net.color_network._B.grad.cpu().numpy(), c["g_color_B"])
    _cmp("mlp", net.color_network.network.params.grad.cpu().numpy(), c["g_mlp"])
    gv, wv = float(net.variance_network.variance.grad), float(c["g_variance"])
    print("variance   got %.6e want %.6e" % (gv, wv))
    assert abs(gv - wv) <= 2e-2 * abs(wv)


def test_fallback_backward_is_independent_of_ray_chunking(monkeypatch):
    """nothing in bound at S = 24 with CHUNK_RAYS = 2: the 100 forced samples span three backward chunks (48 samples
    each), so each chunk must place itself in the call (sample0) and read the forward's fallback flag"""
    from goslam_b200 import neus, synthetic
    ro, rd, zv, ds = [t.to(dev()) for t in synthetic.make_rays(11, S=24, seed=34, n_uniform=8)]
    rt = [[1.9, 1.99], [1.9, 1.99], [1.9, 1.99]]
    gen = torch.Generator().manual_seed(8)
    cc, cd = torch.randn(11, 3, generator=gen).to(dev()), torch.randn(11, 1, generator=gen).to(dev())
    grads = []
    for chunk in (1 << 16, 2):
        monkeypatch.setattr(neus._NeusFunction, "CHUNK_RAYS", chunk)
        net = _net(5, [[-2.0, 2.0]] * 3, rt)
        with torch.enable_grad():
            o = net(ro, rd, zv, ds)
            assert int((o["sdf"] != 100.0).sum()) == 100
            ((o["color"] * cc).sum() + (o["depth"] * cd).sum() + 0.01 * o["sdf"][o["sdf"] != 100.0].sum() + 30.0 * o["gradient_error"].sum()).backward()
        grads.append([p.grad.clone() for p in net.trainable_tensors()])
    for a, b in zip(*grads):
        scale = float(a.abs().max())
        assert scale > 0
        # as in test_backward_is_independent_of_ray_chunking: a chunk that misses its forced samples is an O(1) error
        assert float((a - b).abs().max()) <= 1e-2 * scale, (a.shape, float((a - b).abs().max()), scale)
