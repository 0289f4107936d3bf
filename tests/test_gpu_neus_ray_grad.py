"""Renderer gradient w.r.t. its rays on the GPU (goslam_neus_composite_backward_ex + goslam_neus_ray_backward, reached from
InstantNeuS.forward when rays_o / rays_d require grad, as camera refinement in mapping builds them from pose leaves):
  (1) the kernel against the float64 closed form of oracle/neus_ray_grad_oracle.py at every sample count it takes,
  (2) end to end against tests/golden/neus_ray_grad.npz (the REFERENCE's forward + mapping loss through autograd),
  (3) against central differences of the CUDA forward, one loss term at a time,
  (4)-(5) what must not change: the parameter gradients, and the ray gradients under re-chunking and re-running,
  (6)-(7) pose-only gradients and a camera-refinement trajectory against the reference's."""
import os

import numpy as np
import pytest
import torch

from oracle import neus_ray_grad_oracle as nro

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "neus_ray_grad.npz")
RT = [[-1.9, 1.9], [-2.0, 2.0], [-1.7, 2.0]]


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


def _cmp(name, got, want, rel_tol=2e-2, cos_tol=0.9995):
    """as tests/test_gpu_neus_train.py: relative L2 error and cosine"""
    got, want = np.asarray(got, np.float64).reshape(-1), np.asarray(want, np.float64).reshape(-1)
    rel = np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30)
    cos = float(got @ want) / max(np.linalg.norm(got) * np.linalg.norm(want), 1e-30)
    print("%-10s |want| %.4e  rel L2 err %.3e  cos %.6f" % (name, np.linalg.norm(want), rel, cos))
    assert rel <= rel_tol and cos >= cos_tol, (name, rel, cos)


def _loss(net, out, rays_color, rays_depth, uncertainty):
    """src/mapping.py:97-128 with the weights of configs/go_slam.yaml"""
    depth = rays_depth.reshape(-1, 1)
    valid = (depth > 0).reshape(-1)
    unc = 1.0 / torch.sqrt(out["depth_variance"][valid].detach() + 1e-10) if uncertainty else 1.0
    cl = torch.abs(out["color"][valid] - rays_color[valid]).mean()
    dl = (torch.abs(out["depth"][valid] - depth[valid]) * unc).mean()
    sl, spl = net.compute_sdf_error(sdf=out["sdf"][valid], z_vals=out["z_vals"][valid], gt_depth=depth[valid])
    return cl * 2.0 + dl * 1.0 + (sl + spl) * 2.0 + 0.1 * out["gradient_error"].mean()


def _golden():
    return np.load(GOLDEN)


# ---- (1) kernel against the closed form ---------------------------------------------------------------------------
@pytest.mark.parametrize("S", [24, 48, 72, 100, 128])
@pytest.mark.parametrize("mode", ["whole", "slice", "fallback"])
def test_kernel_matches_closed_form(S, mode):
    """random upstream gradients into goslam_neus_ray_backward against ray_backward_closed_form (float64).  'slice': the
    call covers rays 5.. of a larger forward call (sample0 = 5 S); 'fallback': nothing in bound, the forward call's first
    100 samples forced in, the call a slice starting at ray 1 (at S < 100) so part of them lie before it."""
    from goslam_b200 import _lib, synthetic
    rt = [[5.0, 6.0]] * 3 if mode == "fallback" else RT
    net = _net(5, [[-2.0, 2.0]] * 3, rt)
    Rall = 23
    ro, rd, zv, ds = synthetic.make_rays(Rall, S=S, seed=40 + S, n_uniform=S // 3)
    r0 = {"whole": 0, "slice": 5, "fallback": 1 if S < 100 else 0}[mode]
    ro, rd, zv, ds = ro[r0:].contiguous(), rd[r0:].contiguous(), zv[r0:].contiguous(), ds[r0:].contiguous()
    R = Rall - r0
    n = R * S
    gen = torch.Generator().manual_seed(S)
    d_enc = torch.randn(n, 32, generator=gen) * 64.0              # scaled units: *scale = 64
    d_xyz = torch.randn(n, 3, generator=gen) * 64.0
    dE = (torch.randn(n, 40, generator=gen) * 64.0).half()
    dE[:, 33:] = 0
    d_grad = torch.randn(n, 3, generator=gen) * 0.1
    d_tc = torch.randn(n, generator=gen)
    scale = torch.tensor([64.0])
    fallback = torch.tensor([1 if mode == "fallback" else 0], dtype=torch.int32)
    t = [x.to(dev()) for x in (ro, rd, zv, ds, d_enc, d_xyz, dE, d_grad, d_tc, scale, fallback)]
    p, keep, _ = net._params_struct()
    g_o, g_d = torch.empty(R, 3, device=dev()), torch.empty(R, 3, device=dev())
    import ctypes
    _lib.call("neus_ray_backward", ctypes.byref(p), t[0], t[1], t[2], t[3], t[10], r0 * S, R, S, t[4], t[5], t[6], t[9],
              t[7], t[8], g_o, g_d)
    torch.cuda.synchronize()
    # which samples went through the network, decided as the forward does (float32 positions, strict test, fallback)
    zm = zv.numpy() + ds.numpy() / np.float32(2.0)
    pts = nro.sample_positions(ro.numpy(), rd.numpy(), zm)
    rtn = np.array(rt, np.float32)
    inb = np.all((pts > rtn[:, 0]) & (pts < rtn[:, 1]), axis=-1)
    if mode == "fallback":
        assert not inb.any()
        inb = (r0 * S + np.arange(n) < 100).reshape(R, S)
    assert inb.sum() > 0
    table = net.sdf_network.encoding.encoding.params.detach().half().cpu().numpy().reshape(-1, 2)
    want_o, want_d = nro.ray_backward_closed_form(
        ro.numpy(), rd.numpy(), zm, inb, [[-2.0, 2.0]] * 3, table, net.sdf_network.sdf_layer.weight.detach().cpu().numpy(),
        net.color_network._B.detach().cpu().numpy(), d_enc.numpy() / 64.0, d_xyz.numpy() / 64.0,
        dE.float().numpy()[:, :33] / 64.0, d_grad.numpy(), d_tc.numpy())
    for name, got, want in (("d_rays_o", g_o, want_o), ("d_rays_d", g_d, want_d)):
        got = got.cpu().numpy().astype(np.float64)
        rows = np.abs(want).max(axis=1) > 0
        # fp32 sums of O(100) terms per ray against float64: 1e-4 of the largest entry
        err = np.abs(got - want).max() / np.abs(want).max()
        print("S=%d %s %s: max err / max %.3e" % (S, mode, name, err))
        assert err <= 1e-4, (name, err)
        assert not np.any(got[~rows]), name                    # rays with nothing in the network get exact zeros


# ---- (2) end to end against the reference ------------------------------------------------------------------------------
def _golden_grad_run(chunk=None, monkeypatch=None):
    g = _golden()
    net = _net(int(g["weights_seed"]), g["bound"].tolist(), g["rt_bound"])
    ro = torch.from_numpy(g["grad_rays_o"]).to(dev()).requires_grad_(True)
    rd = torch.from_numpy(g["grad_rays_d"]).to(dev()).requires_grad_(True)
    zv, ds = torch.from_numpy(g["grad_z_vals_in"]).to(dev()), torch.from_numpy(g["grad_dists"]).to(dev())
    with torch.enable_grad():
        out = net(ro, rd, zv, ds)
        total = _loss(net, out, torch.from_numpy(g["grad_rays_color"]).to(dev()), torch.from_numpy(g["grad_rays_depth"]).to(dev()), True)
    total.backward()
    return g, net, ro, rd, total


def test_ray_gradients_match_reference_autograd_golden():
    g, net, ro, rd, total = _golden_grad_run()
    assert abs(float(total.detach()) - float(g["grad_loss"])) <= 2e-3 * abs(float(g["grad_loss"]))
    assert ro.grad.dtype == torch.float32 and ro.grad.shape == ro.shape
    _cmp("d_rays_o", ro.grad.cpu().numpy(), g["grad_d_rays_o"])
    _cmp("d_rays_d", rd.grad.cpu().numpy(), g["grad_d_rays_d"])
    _cmp("sdf_w", net.sdf_network.sdf_layer.weight.grad.cpu().numpy(), g["grad_g_sdf_w"])


def test_ray_gradients_come_back_in_the_callers_dtype():
    g = _golden()
    net = _net(int(g["weights_seed"]), g["bound"].tolist(), g["rt_bound"])
    ro = torch.from_numpy(g["grad_rays_o"]).double().to(dev()).requires_grad_(True)
    rd = torch.from_numpy(g["grad_rays_d"]).to(dev())
    zv, ds = torch.from_numpy(g["grad_z_vals_in"]).to(dev()), torch.from_numpy(g["grad_dists"]).to(dev())
    with torch.enable_grad():
        out = net(ro, rd, zv, ds)
        _loss(net, out, torch.from_numpy(g["grad_rays_color"]).to(dev()), torch.from_numpy(g["grad_rays_depth"]).to(dev()), True).backward()
    assert ro.grad.dtype == torch.float64
    _cmp("d_rays_o", ro.grad.cpu().numpy(), g["grad_d_rays_o"])
    with pytest.raises(RuntimeError, match="z_vals"):
        with torch.enable_grad():
            net(ro, rd, zv.clone().requires_grad_(True), ds)


# ---- (3) finite differences of the CUDA forward ------------------------------------------------------------------------
FD_LEVELS, FD_EPS = 4, 2e-4


def _cells(o, d, zm, rt):
    """per sample of float32 rays: the in-bound test and the cell of every level the finite-difference net uses"""
    from oracle import neus_oracle as no
    pts = nro.sample_positions(o, d, zm)
    rtn = np.array(rt, np.float32)
    inb = np.all((pts > rtn[:, 0]) & (pts < rtn[:, 1]), axis=-1)
    _, _, x01 = nro.normalise(pts.reshape(-1, 3), [[-2.0, 2.0]] * 3)
    metas, _ = no.hashgrid_meta()
    cells = [no._pos(m, x01)[0].reshape(o.shape[0], -1, 3) for m in metas[:FD_LEVELS]]
    return inb, cells


@pytest.mark.parametrize("term", ["depth", "sdf", "eikonal"])
def test_ray_gradients_match_finite_differences_of_the_cuda_forward(term):
    """d loss / d rays against central differences of the fused forward, one loss term at a time, perturbing one component
    of every ray's origin or direction by 2e-4.  The forward is piecewise: a sample that crosses a cell face (the normal
    jumps) or the real-time bound changes the loss by a step, so only rays none of whose samples change cell or bound
    status under the perturbation are perturbed, and only the grid's four coarsest levels are non-zero so that most rays
    qualify.  The sdf and depth terms read the sdf, which the forward computes from the fp16 encoding: there a 2e-4 step
    moves each level's encoding by a few ulps, so those two terms run with the grid's amplitude scaled by 0.05 (the
    include_xyz and normal paths then carry the signal, the fp16 rounding stays below the tolerance).  The eikonal term
    reads only the normal, computed in fp32 from the table, and runs at full amplitude (first- and second-order grid paths).
    The colour term is left out: colour reaches the rays only through the colour network's fp16 input row (sin(p B) and the
    normal columns), where such a step is below an ulp, so its differences are quantisation noise (as for the colour term of
    the parameter test in test_gpu_neus_train.py); the reference golden above pins that path."""
    from goslam_b200 import neus, synthetic
    net = _net(5, [[-2.0, 2.0]] * 3, RT)
    offs, _, _, _ = neus.hashgrid_layout()
    with torch.no_grad():
        grid = net.sdf_network.encoding.encoding.params
        grid[offs[FD_LEVELS]:] = 0.0
        if term != "eikonal":
            grid.mul_(0.05)
    R, S = 512, 24
    ro, rd, zv, ds = synthetic.make_rays(R, S=S, seed=21, n_uniform=8)
    zm = zv.numpy() + ds.numpy() / np.float32(2.0)
    inb0, cells0 = _cells(ro.numpy(), rd.numpy(), zm, RT)
    gen = torch.Generator().manual_seed(3)
    cd = torch.randn(R, 1, generator=gen).to(dev()).double()
    cs = (0.05 * torch.randn(R, S, generator=gen)).to(dev()).double()
    on = {k: float(term == k) for k in ("depth", "sdf", "eikonal")}

    def loss_of(out):
        inb = (out["sdf"] != 100.0).double()
        return (on["depth"] * (out["depth"].double() * cd).sum() + on["sdf"] * (out["sdf"].double() * inb * cs).sum()
                + on["eikonal"] * 50.0 * out["gradient_error"].double().sum())

    t = [x.to(dev()) for x in (ro, rd, zv, ds)]
    ro_l, rd_l = t[0].clone().requires_grad_(True), t[1].clone().requires_grad_(True)
    with torch.enable_grad():
        loss_of(net(ro_l, rd_l, t[2], t[3])).backward()
    grads = (ro_l.grad.cpu().numpy().astype(np.float64), rd_l.grad.cpu().numpy().astype(np.float64))
    bad = []
    for name, which, c in (("o.x", 0, 0), ("o.y", 0, 1), ("o.z", 0, 2), ("d.x", 1, 0), ("d.y", 1, 1), ("d.z", 1, 2)):
        moved = []
        clean = np.ones(R, bool)
        for sgn in (+1, -1):
            o2, d2 = ro.numpy().copy(), rd.numpy().copy()
            (o2 if which == 0 else d2)[:, c] += np.float32(sgn * FD_EPS)
            inb, cells = _cells(o2, d2, zm, RT)
            clean &= np.all(inb == inb0, axis=1)
            for a, b in zip(cells, cells0):
                clean &= np.all(a == b, axis=(1, 2))
            moved.append((o2, d2))
        assert clean.sum() >= R // 5, (name, int(clean.sum()))
        vals, steps = [], []
        for o2, d2 in moved:
            o2 = np.where(clean[:, None], o2, ro.numpy())
            d2 = np.where(clean[:, None], d2, rd.numpy())
            steps.append((o2 if which == 0 else d2)[:, c].astype(np.float64))
            with torch.no_grad():
                vals.append(float(loss_of(net(torch.from_numpy(o2).to(dev()), torch.from_numpy(d2).to(dev()), t[2], t[3]))))
        an = float((grads[which][:, c] * (steps[0] - steps[1])).sum()) / (2 * FD_EPS)     # the steps fp32 actually took
        fd = (vals[0] - vals[1]) / (2 * FD_EPS)
        print("[%s] %-4s %3d clean rays  analytic %.5e  finite-diff %.5e" % (term, name, int(clean.sum()), an, fd))
        if not abs(an - fd) <= 5e-2 * max(abs(fd), abs(an)) + 1e-6:
            bad.append((name, an, fd))
    assert not bad, bad


# ---- (4)-(5) what must not change ---------------------------------------------------------------------------------------
def _train_grads(rays_grad, chunk, monkeypatch):
    from goslam_b200 import neus, synthetic
    monkeypatch.setattr(neus._NeusFunction, "CHUNK_RAYS", chunk)
    net = _net(5, [[-2.0, 2.0]] * 3, RT)
    ro, rd, zv, ds = [t.to(dev()) for t in synthetic.make_rays(37, S=72, seed=29)]
    gen = torch.Generator().manual_seed(8)
    cc, cd = torch.randn(37, 3, generator=gen).to(dev()), torch.randn(37, 1, generator=gen).to(dev())
    if rays_grad:
        ro, rd = ro.requires_grad_(True), rd.requires_grad_(True)
    with torch.enable_grad():
        o = net(ro, rd, zv, ds)
        ((o["color"] * cc).sum() + (o["depth"] * cd).sum() + 0.01 * o["sdf"][o["sdf"] != 100.0].sum()
         + 30.0 * o["gradient_error"].sum()).backward()
    return [p.grad.clone() for p in net.trainable_tensors()], (ro.grad, rd.grad)


def test_parameter_gradients_do_not_change_when_rays_require_grad(monkeypatch):
    """the ray path only adds work: every parameter gradient computed without atomics (colour network, sdf_layer rows
    1.., its bias, colour _B) is bit-identical; the ones the kernels accumulate with float atomics (hash grid, sdf_layer
    row 0 through the normal, the variance) are summed in scheduling order, so they are held to fp32 reordering"""
    base, _ = _train_grads(False, 1 << 16, monkeypatch)
    with_rays, (go, gd) = _train_grads(True, 1 << 16, monkeypatch)
    assert go is not None and gd is not None
    names = ("grid", "mlp", "sdf_w", "sdf_b", "color_B", "variance")
    for name, a, b in zip(names, base, with_rays):
        if name in ("mlp", "sdf_b", "color_B"):
            assert torch.equal(a, b), name
        elif name == "sdf_w":
            assert torch.equal(a[1:], b[1:]), name
            assert float((a[0] - b[0]).abs().max()) <= 1e-5 * float(a[0].abs().max()), name
        else:
            assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max()), name


def test_ray_gradients_are_deterministic_and_independent_of_chunking(monkeypatch):
    """per-ray sums in a fixed order, no atomics: two runs are bit-identical.  With 8-ray chunks each chunk picks its own
    loss scale, so the fp16 operands of the colour network's backward round differently: the ray gradients then agree
    to fp16 rounding, not bit for bit"""
    _, (o1, d1) = _train_grads(True, 1 << 16, monkeypatch)
    _, (o2, d2) = _train_grads(True, 1 << 16, monkeypatch)
    assert torch.equal(o1, o2) and torch.equal(d1, d2)
    _, (o3, d3) = _train_grads(True, 8, monkeypatch)
    for a, b in ((o1, o3), (d1, d3)):
        assert float((a - b).abs().max()) <= 2e-3 * float(a.abs().max())


# ---- (6)-(7) poses ----------------------------------------------------------------------------------------------------
def test_pose_only_gradient_with_frozen_network_matches_the_reference():
    """frozen network, rays from a 4x4 c2w leaf (build_rays, src/nerf_func.py:166-179): dL/d c2w is non-None and matches
    the reference's autograd"""
    g = _golden()
    net = _net(int(g["weights_seed"]), g["bound"].tolist(), g["rt_bound"])
    for prm in net.parameters():
        prm.requires_grad_(False)
    fx, fy, cx, cy = g["traj_cam"].tolist()
    H, W = g["pose_depth"].shape
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    dirs = torch.stack([(xx.reshape(-1) - cx) / fx, (yy.reshape(-1) - cy) / fy, torch.ones(H * W)], -1).to(dev())
    c2w = torch.from_numpy(g["pose_c2w"]).to(dev()).requires_grad_(True)
    with torch.enable_grad():
        rd = dirs @ c2w[:3, :3].t()
        ro = c2w[:3, 3].reshape(1, 3).repeat(H * W, 1)
        np.testing.assert_allclose(rd.detach().cpu().numpy(), g["pose_rays_d"], atol=1e-6)
        out = net(ro, rd, torch.from_numpy(g["pose_z_vals_in"]).to(dev()), torch.from_numpy(g["pose_dists"]).to(dev()))
        total = _loss(net, out, torch.from_numpy(g["pose_color"]).reshape(-1, 3).to(dev()),
                      torch.from_numpy(g["pose_depth"]).reshape(-1).to(dev()), False)
    total.backward()
    assert abs(float(total.detach()) - float(g["pose_loss"])) <= 2e-3 * abs(float(g["pose_loss"]))
    assert c2w.grad is not None
    assert all(p.grad is None for p in net.parameters())
    _cmp("d_c2w", c2w.grad.cpu().numpy()[:3], g["pose_g_c2w"][:3])


def test_camera_refinement_trajectory_matches_the_reference():
    """6 iterations of the mapping loop with the quaternion-translation leaves in their own AdamW group (src/mapping.py:
    173-194, 266-273), rays rebuilt from the leaves every iteration.  Losses within 1 %.  AdamW moves every leaf entry by
    about its learning rate (1e-3) per iteration whatever the gradient's size, so the leaves are held to 1e-3 absolute —
    one step — at every iteration; a wrong sign or a missing ray gradient moves an entry by up to 2e-3 per iteration."""
    g = _golden()
    net = _net(int(g["weights_seed"]), g["bound"].tolist(), g["rt_bound"])
    net_lr, grid_lr, cam_lr = g["traj_lr"].tolist()
    quadt = [torch.nn.Parameter(torch.from_numpy(q).to(dev())) for q in g["traj_quadt0"]]
    opt = torch.optim.AdamW([{"params": net.get_training_parameters(), "lr": net_lr},
                             {"params": net.get_volume_parameters(), "lr": grid_lr}], betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    opt.add_param_group({"params": quadt, "lr": cam_lr})
    train_params = net.get_training_parameters() + net.get_volume_parameters()
    fx, fy, cx, cy = g["traj_cam"].tolist()
    px, py = torch.from_numpy(g["traj_px"]).to(dev()), torch.from_numpy(g["traj_py"]).to(dev())
    depth = torch.from_numpy(g["traj_depth"]).reshape(-1).to(dev())
    color = torch.from_numpy(g["traj_color"]).reshape(-1, 3).to(dev())
    S = 32
    n = px.shape[0] * px.shape[1]
    zv = torch.linspace(0.3, 3.4, S + 1)[:-1].reshape(1, S).repeat(n, 1).to(dev())
    ds = torch.full((n, S), (3.4 - 0.3) / S, device=dev())
    losses, leaves = [], []
    for _ in range(g["traj_losses"].shape[0]):
        opt.zero_grad()
        with torch.enable_grad():
            rays = [nro.pose_rays(quadt[f], px[f], py[f], fx, fy, cx, cy) for f in range(len(quadt))]
            out = net(torch.cat([r[0] for r in rays]), torch.cat([r[1] for r in rays]), zv, ds)
            total = _loss(net, out, color, depth, False)
        total.backward()
        torch.nn.utils.clip_grad_norm_(train_params, max_norm=35.0)
        opt.step()
        losses.append(float(total.detach()))
        leaves.append(torch.stack([q.detach() for q in quadt]).cpu().numpy())
    want = g["traj_losses"]
    print("ours     :", " ".join("%.5f" % v for v in losses))
    print("reference:", " ".join("%.5f" % v for v in want))
    assert np.all(np.abs(np.array(losses) - want) <= 1e-2 * np.abs(want))
    dev_leaf = np.abs(np.stack(leaves) - g["traj_quadt"]).max(axis=(1, 2))
    print("max |quadt - reference| per iteration:", " ".join("%.2e" % v for v in dev_leaf))
    assert np.all(dev_leaf <= 1e-3), dev_leaf
    moved = np.abs(g["traj_quadt"][-1] - g["traj_quadt0"]).max()
    assert moved > 1e-3                                        # the leaves did move
