"""Generate tests/golden/neus_ray_grad.npz by running THE REFERENCE'S OWN PYTHON (imported from /root/reference, which
exists only in the build container) with the rays requiring grad, tcnn replaced by the differentiable restatements of
oracle/neus_grad_oracle.py as in make_golden.py's neus_grad.

What the fixture pins:
    grad_*   InstantNeuS.forward (src/InstantNeuS.py:295-370) + the Mapper.optimize_map loss (src/mapping.py:97-128,
             uncertainty weighting on) differentiated by autograd w.r.t. rays_o and rays_d (and every parameter)
    pose_*   the same loss with the network frozen, rays from a 4x4 c2w leaf through build_rays
             (src/nerf_func.py:115-179): dL/d c2w
    traj_*   camera refinement (src/mapping.py:173-194, 266-273 with mapping.BA): 6 iterations of AdamW over the network
             groups plus one group of quaternion-translation leaves (BA_cam_lr), rays of every frame rebuilt each
             iteration through quaternion_to_Rt + build_rays from the current leaf; the losses and leaves per iteration
z_vals / dists are fixed inputs (the reference samples them under no_grad from detached rays; they carry no gradient).
Run:  python tests/golden/make_golden_ray_grad.py      (writes next to this file)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

NET_LR, GRID_LR, CAM_LR = 1e-4, 1e-3, 1e-3        # x0.1 of the config's network rates as in neus_adamw; BA_cam_lr as configured
TRAJ_ITERS = 6
H, W = 6, 8
CAM = (4.0, 4.0, 3.5, 2.5)                         # fx, fy, cx, cy


def _ref_net(neus_mod, bound, rt):
    from oracle import neus_oracle
    from goslam_b200 import synthetic
    metas, total_entries = neus_oracle.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [total_entries * 2]
    w = synthetic.make_neus_weights(seed=9, total_grid_params=total_entries * 2, layout=(offs, [m["res"] for m in metas]))
    net = neus_mod.InstantNeuS(synthetic.NEUS_CFG, bound, device="cpu")
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net.update_bound(torch.tensor(rt))
    return net


def _loss(net, out, rays_color, rays_depth, uncertainty):
    depth = rays_depth.reshape(-1, 1)
    valid = (depth > 0).reshape(-1)
    unc = 1.0 / torch.sqrt(out["depth_variance"][valid].detach() + 1e-10) if uncertainty else 1.0
    cl = torch.abs(out["color"][valid] - rays_color[valid]).mean()
    dl = (torch.abs(out["depth"][valid] - depth[valid]) * unc).mean()
    sl, spl = net.compute_sdf_error(sdf=out["sdf"][valid], z_vals=out["z_vals"][valid], gt_depth=depth[valid])
    return cl * 2.0 + dl * 1.0 + (sl + spl) * 2.0 + 0.1 * out["gradient_error"].mean()


def _z(R, S, near=0.3, far=3.4):
    zv = torch.linspace(near, far, S + 1)[:-1].reshape(1, S).repeat(R, 1)
    return zv.contiguous(), torch.full((R, S), (far - near) / S)


def main():
    if not os.path.isdir(mg.REF):
        raise SystemExit("needs /root/reference (build container only)")
    mg.install_stubs()
    neus_mod = mg.ref_import("src.InstantNeuS")
    nf = mg.ref_import("src.nerf_func")
    import tinycudann
    from oracle import neus_grad_oracle as ngo
    from goslam_b200 import synthetic
    old = tinycudann.Encoding, tinycudann.Network, torch.Tensor.get_device
    tinycudann.Encoding, tinycudann.Network = ngo.TorchHashGrid, ngo.TorchMLP
    # quad2rotation allocates with .to(quad.get_device()), which is -1 for a CPU tensor
    torch.Tensor.get_device = lambda t: "cpu" if t.device.type == "cpu" else old[2](t)
    store = {}
    bound = [[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]]
    rt = [[-1.8, 1.9], [-2.0, 2.0], [-1.5, 2.0]]
    try:
        # ---- ray gradients: the inputs of neus_grad.npz with rays requiring grad ----
        net = _ref_net(neus_mod, bound, rt)
        R, S = 40, 32
        ro, rd, zv, ds = synthetic.make_rays(R, S=S, seed=13, n_uniform=12)
        g = torch.Generator().manual_seed(17)
        rays_color = torch.rand(R, 3, generator=g)
        rays_depth = 0.5 + 2.5 * torch.rand(R, generator=g)
        rays_depth[::9] = 0.0
        ro_l, rd_l = ro.clone().requires_grad_(True), rd.clone().requires_grad_(True)
        with torch.enable_grad():
            out = net(ro_l, rd_l, zv, ds)
            total = _loss(net, out, rays_color, rays_depth, True)
            total.backward()
        store.update(grad_rays_o=ro.numpy(), grad_rays_d=rd.numpy(), grad_z_vals_in=zv.numpy(), grad_dists=ds.numpy(),
                     grad_rays_color=rays_color.numpy(), grad_rays_depth=rays_depth.numpy(), grad_loss=np.float32(total.item()),
                     grad_d_rays_o=ro_l.grad.numpy(), grad_d_rays_d=rd_l.grad.numpy(),
                     grad_g_sdf_w=net.sdf_network.sdf_layer.weight.grad.numpy())
        print("grad: loss %.6f |d rays_o| %.4e |d rays_d| %.4e" % (total.item(), ro_l.grad.norm(), rd_l.grad.norm()))

        # ---- pose only: frozen network, rays of a pixel grid from a c2w leaf ----
        net = _ref_net(neus_mod, bound, rt)
        for prm in net.parameters():
            prm.requires_grad_(False)
        c2w = torch.eye(4)
        c2w[:3, 3] = torch.tensor([0.1, -0.2, -1.6])
        ang = 0.1
        c2w[:3, :3] = torch.tensor([[np.cos(ang), 0.0, np.sin(ang)], [0.0, 1.0, 0.0], [-np.sin(ang), 0.0, np.cos(ang)]])
        gen = torch.Generator().manual_seed(23)
        depth_img = 1.2 + 0.8 * torch.rand(H, W, generator=gen)
        color_img = torch.rand(H, W, 3, generator=gen)
        c2w_l = c2w.clone().requires_grad_(True)
        with torch.enable_grad():
            pro, prd, pdep, pcol = nf.build_rays(0, H, 0, W, 0, H, W, *CAM, c2w_l, depth_img, color_img, "cpu",
                                                 nerf_coordinate=False, dir_normalize=False)
            pz, pds = _z(pro.shape[0], S)
            out = net(pro.float(), prd.float(), pz, pds)
            total = _loss(net, out, pcol.float(), pdep.float(), False)
            total.backward()
        store.update(pose_c2w=c2w.numpy(), pose_depth=depth_img.numpy(), pose_color=color_img.numpy(), pose_z_vals_in=pz.numpy(),
                     pose_dists=pds.numpy(), pose_rays_o=pro.detach().numpy(), pose_rays_d=prd.detach().numpy(),
                     pose_loss=np.float32(total.item()), pose_g_c2w=c2w_l.grad.numpy())
        print("pose: loss %.6f |d c2w| %.4e" % (total.item(), c2w_l.grad.norm()))

        # ---- camera refinement trajectory: two frames, quadt leaves in their own AdamW group ----
        net = _ref_net(neus_mod, bound, rt)
        quadt0 = torch.tensor([[0.995, 0.04, -0.03, 0.02, 0.1, -0.2, -1.6],
                               [0.990, -0.05, 0.06, -0.01, -0.25, 0.15, -1.5]])
        quadt = [torch.nn.Parameter(q.clone()) for q in quadt0]
        gen = torch.Generator().manual_seed(29)
        depths = 1.0 + 1.0 * torch.rand(2, H, W, generator=gen)
        colors = torch.rand(2, H, W, 3, generator=gen)
        opt = torch.optim.AdamW([{"params": net.get_training_parameters(), "lr": NET_LR},
                                 {"params": net.get_volume_parameters(), "lr": GRID_LR}],
                                betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
        opt.add_param_group({"params": quadt, "lr": CAM_LR})
        train_params = net.get_training_parameters() + net.get_volume_parameters()
        losses, leaves = [], []
        px, py, ro0, rd0 = [], [], [], []
        for it in range(TRAJ_ITERS):
            opt.zero_grad()
            with torch.enable_grad():
                ros, rds, dps, cols = [], [], [], []
                for f in range(2):
                    c2w = nf.quaternion_to_Rt(quadt[f])
                    a, b, c, d = nf.build_rays(0, H, 0, W, 0, H, W, *CAM, c2w, depths[f], colors[f], "cpu",
                                               nerf_coordinate=False, dir_normalize=False)
                    ros.append(a.float()); rds.append(b.float()); dps.append(c.float()); cols.append(d.float())
                    if it == 0:
                        yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
                        px.append(xx.reshape(-1).numpy()); py.append(yy.reshape(-1).numpy())
                        ro0.append(a.detach().numpy()); rd0.append(b.detach().numpy())
                vro, vrd = torch.cat(ros), torch.cat(rds)
                tz, tds = _z(vro.shape[0], S)
                out = net(vro, vrd, tz, tds)
                total = _loss(net, out, torch.cat(cols), torch.cat(dps), False)
                total.backward()
            torch.nn.utils.clip_grad_norm_(train_params, max_norm=35.0)
            opt.step()
            losses.append(total.item())
            leaves.append(torch.stack([q.detach().clone() for q in quadt]).numpy())
            print("traj %d: loss %.6f quadt %s" % (it, total.item(), np.array2string(leaves[-1][0], precision=5)))
        store.update(traj_quadt0=quadt0.numpy(), traj_depth=depths.numpy(), traj_color=colors.numpy(), traj_cam=np.array(CAM, np.float32),
                     traj_px=np.stack(px), traj_py=np.stack(py), traj_rays_o0=np.stack(ro0), traj_rays_d0=np.stack(rd0),
                     traj_losses=np.array(losses, np.float64), traj_quadt=np.stack(leaves), traj_lr=np.array([NET_LR, GRID_LR, CAM_LR]))
    finally:
        tinycudann.Encoding, tinycudann.Network, torch.Tensor.get_device = old
    np.savez_compressed(os.path.join(HERE, "neus_ray_grad.npz"), bound=np.array(bound, np.float32), rt_bound=np.array(rt, np.float32),
                        weights_seed=9, **store)
    print("wrote neus_ray_grad")


if __name__ == "__main__":
    main()
