"""CPU oracle (TEST INFRASTRUCTURE — never imported by the product path) for camera refinement in mapping
(mapping.BA: src/mapping.py:173-194, 266-273; src/nerf_func.py:44-112):
  * pose_ray_backward — the float64 closed form goslam_mapping_pose_rays_backward implements (csrc/mapping.cu);
  * kernel_dirs — the f32 pinhole directions the ray kernels compute from pixel coordinates;
  * matrix_to_quaternion — Rt_to_quaternion's rotation part restated (Shepperd's method, w >= 0) without mathutils;
  * RefineSchedule — Mapper.__call__ with BA, as oracle/mapping_oracle.MapperSchedule restates it without;
  * StubRenderer / StubNet — a renderer and net whose outputs are smooth functions of rays_o, rays_d and five
    parameters, for pinning the driver (tests/golden/mapping_refine.npz) apart from the network.
The quaternion-to-rotation and ray construction are oracle/neus_ray_grad_oracle's quat_to_rotation and pose_rays.
"""
import numpy as np
import torch

from . import mapping_oracle as mo
from . import neus_ray_grad_oracle as nro

F32 = np.float32


# ----------------------------------------------------------------------------- pose rays
def kernel_dirs(px, py, fx, fy, cx, cy):
    """[N,3] f32 ((x - (f32)cx) * (f32)(1/fx), (y - (f32)cy) * (f32)(1/fy), 1): what torch's `(x - cx) / fx` and the
    ray kernels compute with Python-float intrinsics"""
    px, py = np.asarray(px, F32), np.asarray(py, F32)
    dx = (px - F32(cx)) * F32(1.0 / fx)
    dy = (py - F32(cy)) * F32(1.0 / fy)
    return np.stack([dx, dy, np.ones_like(dx)], -1).astype(F32)


def pose_ray_backward(quadt, dirs, rows, d_rays_o, d_rays_d):
    """d quadt [n,7] float64 for rays_d[r] = quat_to_rotation(q_e) dirs[r], rays_o[r] = t_e over entry e's `rows[e]`
    consecutive rows (0 allowed).  With R = I + s A(q), s = 2/|q|^2 (q need not be unit), G = sum_r g_d[r] dirs[r]^T:
      dL/dq_m = -s^2 q_m <G, A> + s <G, dA/dq_m>,   dL/dt = sum_r g_o[r]"""
    q = np.asarray(quadt, np.float64).reshape(-1, 7)
    dirs, go, gd = (np.asarray(a, np.float64).reshape(-1, 3) for a in (dirs, d_rays_o, d_rays_d))
    out = np.zeros_like(q)
    at = 0
    for e, n in enumerate(rows):
        G = gd[at:at + n].T @ dirs[at:at + n]
        out[e, 4:] = go[at:at + n].sum(0)
        at += n
        r, i, j, k = q[e, :4]
        s = 2.0 / (q[e, :4] ** 2).sum()
        A = np.array([[-(j * j + k * k), i * j - k * r, i * k + j * r],
                      [i * j + k * r, -(i * i + k * k), j * k - i * r],
                      [i * k - j * r, j * k + i * r, -(i * i + j * j)]])
        dA = [np.array([[0, -k, j], [k, 0, -i], [-j, i, 0]]),                 # d/dr
              np.array([[0, j, k], [j, -2 * i, -r], [k, r, -2 * i]]),          # d/di
              np.array([[-2 * j, i, r], [i, 0, k], [-r, k, -2 * j]]),          # d/dj
              np.array([[-2 * k, -r, i], [r, -2 * k, j], [i, j, 0]])]          # d/dk
        GA = (G * A).sum()
        for m in range(4):
            out[e, m] = -s * s * q[e, m] * GA + s * (G * dA[m]).sum()
    return out


def matrix_to_quaternion(R):
    """[...,3,3] -> [...,4] (w, x, y, z) float64 unit quaternions with quat_to_rotation(q) = R, w >= 0: Shepperd's
    method (the square root of the largest of 1 + trace and 1 + 2 R_aa - trace), then normalised"""
    R = np.asarray(R, np.float64)
    shape = R.shape[:-2]
    R = R.reshape(-1, 3, 3)
    out = np.empty((R.shape[0], 4))
    for b, m in enumerate(R):
        tr = m[0, 0] + m[1, 1] + m[2, 2]
        if tr >= m[0, 0] and tr >= m[1, 1] and tr >= m[2, 2]:
            h = np.sqrt(1.0 + tr); f = 0.5 / h
            q = [0.5 * h, (m[2, 1] - m[1, 2]) * f, (m[0, 2] - m[2, 0]) * f, (m[1, 0] - m[0, 1]) * f]
        elif m[0, 0] >= m[1, 1] and m[0, 0] >= m[2, 2]:
            h = np.sqrt(1.0 + m[0, 0] - m[1, 1] - m[2, 2]); f = 0.5 / h
            q = [(m[2, 1] - m[1, 2]) * f, 0.5 * h, (m[0, 1] + m[1, 0]) * f, (m[0, 2] + m[2, 0]) * f]
        elif m[1, 1] >= m[2, 2]:
            h = np.sqrt(1.0 - m[0, 0] + m[1, 1] - m[2, 2]); f = 0.5 / h
            q = [(m[0, 2] - m[2, 0]) * f, (m[0, 1] + m[1, 0]) * f, 0.5 * h, (m[1, 2] + m[2, 1]) * f]
        else:
            h = np.sqrt(1.0 - m[0, 0] - m[1, 1] + m[2, 2]); f = 0.5 / h
            q = [(m[1, 0] - m[0, 1]) * f, (m[0, 2] + m[2, 0]) * f, (m[1, 2] + m[2, 1]) * f, 0.5 * h]
        q = np.array(q)
        out[b] = q / np.linalg.norm(q) * (-1.0 if q[0] < 0 else 1.0)
    return out.reshape(shape + (4,))


def rt_to_quaternion(c2w):
    """Rt_to_quaternion(c2w, Tquad=False) with matrix_to_quaternion in place of mathutils: [7] f32 tensor"""
    m = c2w.detach().cpu().numpy()
    pose = np.concatenate([matrix_to_quaternion(m[:3, :3]), m[:3, 3]], axis=0)
    return torch.from_numpy(pose).float().to(c2w.device)


def quaternion_to_rt(quadt):
    """quaternion_to_Rt for one leaf [7] -> [4,4] (src/nerf_func.py:91-112), differentiable"""
    R = nro.quat_to_rotation(quadt[None, :4])[0]
    Rt = torch.cat([R, quadt[4:, None]], dim=1)
    return torch.cat([Rt, torch.tensor([[0, 0, 0, 1.0]], dtype=quadt.dtype, device=quadt.device)], dim=0)


# ----------------------------------------------------------------------------- the process with BA
class RefineSchedule(mo.MapperSchedule):
    """MapperSchedule with cfg['mapping']['BA'] (src/mapping.py:173-194, 266-273): enable_ba = BA and last_visit >= 10
    before the call moves last_visit; one leaf per visit-list entry from that entry's c2w; the optimizer's third group
    deleted, then the leaves added at BA_cam_lr; the visit batches from quaternion_to_Rt(leaf).  `calls` collects per
    call (number of groups, their learning rates, the leaves as created)."""

    def __init__(self, cfg, slam, SE3, optimize_map, optimizer=None):
        super().__init__(cfg, slam, SE3, optimize_map, optimizer)
        self.BA, self.BA_cam_lr = cfg['mapping']['BA'], cfg['mapping']['BA_cam_lr']
        self.calls = []

    def __call__(self, the_end=False):
        cur_idx = int(self.video.filtered_id.item())
        if cur_idx <= 1:
            return []
        num_joint_iters = self.num_joint_iters * 10 if the_end else self.num_joint_iters
        self.local_step = 0
        unvisit_list = list(range(self.last_visit, cur_idx))
        visit_list = [cur_idx - 1, cur_idx - 2]
        if self.last_visit > 0:
            _, indices = torch.sort(self.video.update_priority[:self.last_visit].detach(), dim=0, descending=True)
            visit_list += list(indices.cpu().numpy())[:10]
            visit_list += mo.random_select(self.last_visit, self.mapping_window_size - 12)
        enable_ba = self.BA and self.last_visit >= 10
        visit, leaves = {}, []
        for f in visit_list:
            visit[f] = mo.mapping_item(self.video, f, self.device, self.decay, self.SE3)
            if enable_ba:
                leaves.append(rt_to_quaternion(visit[f][2]).requires_grad_(True))
        unvisit = {f: mo.mapping_item(self.video, f, self.device, self.decay, self.SE3) for f in unvisit_list}
        opt = self.optimizer
        if enable_ba and len(opt.param_groups) > 2:
            del opt.param_groups[-1]
        if enable_ba and len(leaves) > 0:
            opt.add_param_group({'params': leaves, 'lr': self.BA_cam_lr})
        self.calls.append((len(opt.param_groups), [g['lr'] for g in opt.param_groups],
                           [q.detach().clone() for q in leaves]))
        self.mapping_net.update_bound(self.video.bound[0])
        self.log.append((list(unvisit_list), [int(f) for f in visit_list]))
        trained = []
        unvisit_factor = num_joint_iters * 10 if self.init else num_joint_iters
        if len(unvisit_list) > 2:
            self.last_visit = cur_idx
            for _ in range(unvisit_factor):
                sub = list(np.random.choice(unvisit_list, self.mapping_window_size))
                trained.append(self._train(sub, self.mapping_pixels // len(sub), unvisit))
        for _ in range(num_joint_iters):
            if len(visit_list) < 1:
                continue
            if enable_ba:
                items = [visit[f][:2] + (quaternion_to_rt(q),) + visit[f][3:] for f, q in zip(visit_list, leaves)]
                trained.append(self._train_entries(visit_list, self.mapping_pixels // len(visit_list), items))
            else:
                trained.append(self._train(visit_list, self.mapping_pixels // len(visit_list), visit))
        self.init = False
        return trained

    def _train_entries(self, frames, n_rays, items):
        """_train with one item per list entry (its own c2w) rather than per frame"""
        out = [[], [], [], []]
        for color, depth, c2w, _, mask in items:
            for acc, t in zip(out, mo.build_rays(n_rays, self.H, self.W, self.fx, self.fy, self.cx, self.cy, c2w, depth,
                                                 color, self.device, mask,
                                                 record=self.draws if self.record_draws else None)):
                acc.append(t.float())
        self.frame_lists.append(([int(f) for f in frames], n_rays))
        ro, rd, depth, color = [torch.cat(a, dim=0) for a in out]
        if len(ro) < 100:
            return False
        self._optimize_map(self, ro, rd, color, depth, self.optimizer, 1)
        return True


# ----------------------------------------------------------------------------- stand-ins
class StubNet(mo.StubNet):
    """mapping_oracle.StubNet (w [2] training, g [3] volume) with set values and the reference's compute_sdf_error
    signature: smooth losses of sdf against gt_depth - z_vals"""

    def __init__(self, device="cpu"):
        super().__init__(device)
        with torch.no_grad():
            self.w.copy_(torch.tensor([0.7, -0.4]))
            self.g.copy_(torch.tensor([0.1, -0.2, 0.3]))

    def compute_sdf_error(self, sdf, z_vals, gt_depth):
        tgt = (gt_depth - z_vals) * 0.1
        return ((sdf - tgt) ** 2).mean(), 0.01 * (sdf * sdf).mean()


class StubRenderer:
    """render_batch_ray's outputs (color [R,3], depth [R,1], sdf / z_vals [R,4], depth_variance [R,1], gradient_error)
    as smooth functions of rays_o, rays_d and the net's w, g"""

    def __init__(self, device="cpu"):
        g = torch.Generator().manual_seed(5)
        self.A = (0.5 * torch.randn(3, 3, generator=g)).to(device)
        self.B = (0.5 * torch.randn(3, 3, generator=g)).to(device)
        self.steps = torch.linspace(0.5, 1.5, 4).to(device)

    def render_batch_ray(self, rays_o, rays_d, net, render_params, device, gt_depth):
        h = torch.tanh(rays_o @ self.A + rays_d @ self.B)
        color = torch.sigmoid(h + net.w[0] * rays_d + net.g)
        depth = 1.0 + 0.5 * torch.tanh(net.w[1] * h.sum(-1, keepdim=True)) + 0.1 * (rays_o * rays_d).sum(-1, keepdim=True)
        z_vals = depth.detach() * self.steps
        sdf = (depth - z_vals) * (1.0 + 0.1 * h[:, :1])
        return {'color': color, 'depth': depth, 'sdf': sdf, 'z_vals': z_vals,
                'depth_variance': 0.1 + (h * h).sum(-1, keepdim=True),
                'gradient_error': ((net.g * net.g).sum() + ((rays_d * rays_d).sum(-1) - 1.0).pow(2).mean()).reshape(1)}


# ----------------------------------------------------------------------------- the golden scenario
# mapping_oracle's golden scene and config with BA on: calls before last_visit reaches 10 (no leaves), the first camera
# group (11, whose one visit batch is under 100 rays), replacements (12; 13 with an unvisit pass while leaves exist) and
# a the_end call (16)
REFINE_CALLS = [(1, False), (6, False), (10, False), (11, False), (12, False), (13, False), (16, True)]


def refine_cfg(device):
    S = mo.GOLDEN_SIZE
    cfg = mo.mapping_cfg(device, S["pixels"], S["window"], S["iters"])
    cfg['mapping']['BA'] = True
    return cfg
