"""Restatement of the reference's mapping process (TEST INFRASTRUCTURE — never imported by the product path).

`build_rays`, `build_all_rays` and `random_select` are src/nerf_func.py:28-40,115-221 and `mapping_item` is
DepthVideo.get_mapping_item (src/depth_video.py:153-173), with the same torch ops in the same order, so they run on
either device and match the reference there bit for bit.  `MapperSchedule.__call__` is Mapper.__call__
(src/mapping.py:151-300) with `optimize_map` injected, so a test can record the batches or train on them;
`reference_optimize_map` is the reference's training step (:60-148).  `build_rays(..., record=list)` also appends the
drawn indices.  The golden scenario (tests/golden/mapping.npz) is defined here for the generator and the tests.
"""
import types

import numpy as np
import torch


def random_select(l, k, start=0):
    m = (l - start) / k
    idx = np.linspace(start, l - 1 - m, k) + np.random.rand(k) * m
    idx = list(idx.clip(start, l - 1))
    return [int(i) for i in idx if i > 0]


def build_rays(n_rays, H, W, fx, fy, cx, cy, c2w, depth, color, device, mask, record=None):
    """build_rays(0, H, 0, W, n_rays, ..., nerf_coordinate=False, dir_normalize=False, mask=mask)"""
    x, y = torch.meshgrid(torch.linspace(0, W - 1, W).to(device), torch.linspace(0, H - 1, H).to(device),
                          indexing='ij')
    x, y = x.t().reshape(-1), y.t().reshape(-1)
    depth = depth.reshape(-1)
    color = color.reshape(-1, 3)
    keep = torch.masked_select(torch.arange(x.shape[0], dtype=torch.long, device=device), mask.reshape(-1).bool())
    x, y, depth, color = x[keep], y[keep], depth[keep], color[keep]
    N = x.shape[0]
    if 0 < n_rays < N // 2:
        idx = torch.randint(N, (n_rays,), device=device)
        if record is not None:
            record.append(idx.clone())
        idx = idx.clamp(0, N - 1)
        x, y, depth, color = x[idx], y[idx], depth[idx], color[idx]
    dirs = torch.stack([(x - cx) / fx, (y - cy) / fy, torch.ones_like(x)], dim=-1).to(device)
    rays_d = dirs @ c2w[:3, :3].t()
    rays_o = c2w[:3, 3].reshape(1, 3).repeat(x.shape[0], 1)
    return rays_o, rays_d, depth, color


def build_all_rays(H, W, fx, fy, cx, cy, c2w, device):
    """build_all_rays(..., nerf_coordinate=False, dir_normalize=False): rays_o, rays_d [H,W,3]"""
    if isinstance(c2w, np.ndarray):
        c2w = torch.from_numpy(c2w).to(device)
    x, y = torch.meshgrid(torch.linspace(0, W - 1, W).to(device), torch.linspace(0, H - 1, H).to(device),
                          indexing='ij')
    x, y = x.t(), y.t()
    dirs = torch.stack([(x - cx) / fx, (y - cy) / fy, torch.ones_like(x)], dim=-1).to(device)
    rays_d = dirs @ c2w[:3, :3].t()
    rays_o = c2w[:3, 3].reshape(1, 1, 3).repeat(H, W, 1)
    return rays_o, rays_d


def mapping_item(video, index, device, decay, SE3):
    """DepthVideo.get_mapping_item: image [H,W,3], depth, c2w [4,4], gt_c2w, mask"""
    with video.mapping.get_lock():
        image = video.images[index].clone().permute(1, 2, 0).contiguous().to(device)
        mask = video.mask_filtered[index].clone().to(device)
        depth = 1.0 / (video.disps_filtered[index].clone().to(device) + 1e-7)
        w2c = SE3(video.poses_filtered[index].clone().to(device))
        c2w = (SE3(video.pose_compensate[0].clone().to(device)) * w2c.inv()).matrix()
        gt_c2w = video.poses_gt[index].clone().to(device)
        video.update_priority[index] *= decay
        return image, depth, c2w, gt_c2w, mask


def render_img(renderer, net, c2w, device, gt_depth):
    """Renderer.render_img (src/render.py:177-237) on a renderer's render_batch_ray"""
    H, W = renderer.H, renderer.W
    rays_o, rays_d = build_all_rays(H, W, renderer.fx, renderer.fy, renderer.cx, renderer.cy, c2w, device)
    rays_o, rays_d = rays_o.reshape(-1, 3), rays_d.reshape(-1, 3)
    params = {'global_step': -1, 'gt_depth': None, 'stratified': False, 'update_state': False,
              'compute_sdf_smooth_error': False}
    out = {}
    gt_depth = gt_depth.reshape(-1)
    step = renderer.ray_batch_size
    for i in range(0, H * W, step):
        o = renderer.render_batch_ray(rays_o=rays_o[i:i + step], rays_d=rays_d[i:i + step], net=net,
                                      render_params=params, device=device, gt_depth=gt_depth[i:i + step])
        if not out:
            out = o
            continue
        for k, v in o.items():
            out[k] = torch.cat([out[k], v], dim=0) if torch.is_tensor(v) else v
    return out


def reference_optimize_map(mapper, rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters, losses=None):
    """src/mapping.py:60-148 (no BA, no log) on mapper's renderer / net; appends each total loss to `losses`"""
    for _ in range(num_joint_iters):
        mapper.local_step += 1
        mapper.global_step += 1
        optimizer.zero_grad()
        with torch.enable_grad():
            ret = mapper.renderer.render_batch_ray(rays_o=rays_o, rays_d=rays_d, net=mapper.mapping_net,
                                                   render_params={'global_step': mapper.global_step},
                                                   device=mapper.device, gt_depth=rays_depth)
        rays_depth = rays_depth.reshape(-1, 1)
        ok = (rays_depth > 0).reshape(-1)
        rays_depth, rays_color = rays_depth[ok], rays_color[ok]
        unc = 1.0 / torch.sqrt(ret['depth_variance'][ok].detach() + 1e-10)
        total = torch.abs(ret['color'][ok] - rays_color).mean() * mapper.w_color_loss
        total = total + (torch.abs(ret['depth'][ok] - rays_depth) * unc).mean()
        sl, spl = mapper.mapping_net.compute_sdf_error(sdf=ret['sdf'][ok], z_vals=ret['z_vals'][ok],
                                                       gt_depth=rays_depth)
        total = total + (sl + spl) * mapper.w_sdf_loss
        total = total + mapper.w_eikonal_loss * ret['gradient_error'].mean()
        total.backward()
        torch.nn.utils.clip_grad_norm_(mapper.train_params, max_norm=35.0)
        optimizer.step()
        optimizer.zero_grad()
        if losses is not None:
            losses.append(total.detach())


class MapperSchedule:
    """Mapper.__call__ with get_mapping_item -> mapping_item and optimize_map injected:
    optimize_map(schedule, rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters).
    `frame_lists` collects each iteration's frame list and n_rays, `draws` the randint outputs, `log` the log lines."""

    def __init__(self, cfg, slam, SE3, optimize_map, optimizer=None):
        m = cfg['mapping']
        self.video, self.mapping_net, self.renderer, self.SE3 = slam.video, slam.mapping_net, slam.renderer, SE3
        self.device = m['device']
        self.num_joint_iters, self.decay = m['iters'], float(m['decay'])
        self.w_color_loss, self.w_sdf_loss, self.w_eikonal_loss = m['w_color_loss'], m['w_sdf_loss'], m['w_eikonal_loss']
        self.mapping_pixels, self.mapping_window_size = m['pixels'], m['mapping_window_size']
        self.H, self.W, self.fx, self.fy, self.cx, self.cy = slam.H, slam.W, slam.fx, slam.fy, slam.cx, slam.cy
        self.local_step = self.global_step = self.last_visit = 0
        self.init = True
        self.optimizer = optimizer
        self.train_params = [p for g in optimizer.param_groups for p in g['params']] if optimizer is not None else []
        self._optimize_map = optimize_map
        self.frame_lists, self.draws, self.log = [], [], []
        self.record_draws = True

    def _batch(self, frames, n_rays, items):
        out = [[], [], [], []]
        for f in frames:
            color, depth, c2w, _, mask = items[f]
            for acc, t in zip(out, build_rays(n_rays, self.H, self.W, self.fx, self.fy, self.cx, self.cy, c2w, depth,
                                              color, self.device, mask,
                                              record=self.draws if self.record_draws else None)):
                acc.append(t.float())
        self.frame_lists.append(([int(f) for f in frames], n_rays))
        return [torch.cat(a, dim=0) for a in out]

    def _train(self, frames, n_rays, items):
        ro, rd, depth, color = self._batch(frames, n_rays, items)
        if len(ro) < 100:
            return False
        self._optimize_map(self, ro, rd, color, depth, self.optimizer, 1)
        return True

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
            visit_list += random_select(self.last_visit, self.mapping_window_size - 12)
        visit = {f: mapping_item(self.video, f, self.device, self.decay, self.SE3) for f in visit_list}
        unvisit = {f: mapping_item(self.video, f, self.device, self.decay, self.SE3) for f in unvisit_list}
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
            trained.append(self._train(visit_list, self.mapping_pixels // len(visit_list), visit))
        self.init = False
        return trained


# ----------------------------------------------------------------------------- stand-ins and scenes
def stub_video(n, ht, wd, device="cpu"):
    """the DepthVideo attributes the mapping process reads and writes, initialised as DepthVideo does"""
    from multiprocessing import Value
    ident = torch.tensor([[0, 0, 0, 0, 0, 0, 1.0]], device=device)
    v = types.SimpleNamespace(
        mapping=Value("i", 0), timestamp=torch.arange(n, dtype=torch.float, device=device),
        images=torch.zeros(n, 3, ht, wd, device=device), poses_filtered=ident.repeat(n, 1),
        poses_gt=torch.eye(4, device=device).repeat(n, 1, 1), disps_filtered=torch.zeros(n, ht, wd, device=device),
        mask_filtered=torch.zeros(n, ht, wd, device=device), update_priority=torch.zeros(n, device=device),
        filtered_id=torch.tensor([-1], dtype=torch.int, device=device), bound=torch.zeros(1, 3, 2, device=device),
        pose_compensate=ident.clone())
    v.get_bound = lambda: v.bound[0]
    return v


class StubNet(torch.nn.Module):
    """get_training_parameters / get_volume_parameters / update_bound / realtime_bound for the schedule alone"""

    def __init__(self, device="cpu"):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(2, device=device))
        self.g = torch.nn.Parameter(torch.zeros(3, device=device))
        self.register_buffer("realtime_bound", torch.zeros(3, 2, device=device))

    def get_training_parameters(self, ignore_keys=()):
        return [self.w]

    def get_volume_parameters(self):
        return [self.g]

    def update_bound(self, bound):
        self.realtime_bound[:] = bound.float().to(self.realtime_bound.device)


def stub_slam(video, net, renderer, intrinsics, output):
    fx, fy, cx, cy = intrinsics
    _, _, H, W = video.images.shape
    return types.SimpleNamespace(verbose=False, bound=video.bound, video=video, mapping_net=net, renderer=renderer,
                                 reload_map=torch.zeros(1).int(), output=output, H=H, W=W, fx=fx, fy=fy, cx=cx, cy=cy)


def mapping_cfg(device, pixels, window, iters, decay=0.8):
    return {'mapping': {'device': device, 'BA': False, 'BA_cam_lr': 0.001, 'net_lr': 0.001, 'grid_lr': 0.01,
                        'w_color_loss': 2.0, 'w_sdf_smooth_loss': 1.0, 'w_sdf_loss': 2.0, 'w_eikonal_loss': 0.1,
                        'uncertainty_weight_loss': True, 'mapping_window_size': window, 'pixels': pixels,
                        'iters': iters, 'post_processing_iters': 10, 'decay': decay}}


def random_pose(g, scale=1.0):
    q = torch.randn(4, generator=g)
    return torch.cat([scale * torch.randn(3, generator=g), q / q.norm()])


# unit quaternions (x, y, z, w) whose rotation matrices hold only 0 and +-1, and whose products stay in the set: with
# intrinsics that make (x - cx) / fx exact, every ray direction is exact whatever the order of its dot products
_EXACT_QUATS = [(0, 0, 0, 1.0), (1.0, 0, 0, 0), (0, 1.0, 0, 0), (0, 0, 1.0, 0), (0.5, 0.5, 0.5, 0.5),
                (-0.5, 0.5, 0.5, 0.5), (0.5, -0.5, 0.5, 0.5), (0.5, 0.5, -0.5, 0.5)]


def exact_pose(g, scale=1.0):
    q = _EXACT_QUATS[int(torch.randint(len(_EXACT_QUATS), (1,), generator=g))]
    return torch.cat([scale * torch.randn(3, generator=g), torch.tensor(q)])


def fill_frames(video, frames, g, mask_counts=None, density=0.7, zero_frac=0.02, trans=1.0, pose=None):
    """random images, disparities in [0.2, 2] (zero_frac of them 0), poses (translations ~ trans) and masks;
    mask_counts[f] = exact number of masked pixels, else a density fraction; pose = random_pose or exact_pose"""
    _, _, ht, wd = video.images.shape
    mask_counts = mask_counts or {}
    for f in frames:
        video.images[f] = torch.rand(3, ht, wd, generator=g)
        d = 0.2 + 1.8 * torch.rand(ht, wd, generator=g)
        d[torch.rand(ht, wd, generator=g) < zero_frac] = 0.0
        video.disps_filtered[f] = d
        if f in mask_counts:
            m = torch.zeros(ht * wd)
            m[torch.randperm(ht * wd, generator=g)[:mask_counts[f]]] = 1.0
            video.mask_filtered[f] = m.reshape(ht, wd)
        else:
            video.mask_filtered[f] = (torch.rand(ht, wd, generator=g) < density).float()
        video.poses_filtered[f] = (pose or random_pose)(g, trans)
        video.update_priority[f] = torch.rand((), generator=g) * 4.0


# golden scene: 16 x 24 frames, window 14, 140 pixels (10 rays per unvisit frame), iters 1
GOLDEN_SIZE = dict(buffer=16, ht=16, wd=24, pixels=140, window=14, iters=1, seed=11)
GOLDEN_INTR = (20.5, 19.25, 11.3, 7.6)
# (filtered_id, the_end, {frame: exact mask count}) per call; frames first seen in a call are filled before it
GOLDEN_CALLS = [                  # (filtered_id, the_end)
    (1, False),                   # cur_idx <= 1: no-op
    (6, False),                   # init: unvisit_factor x10; empty mask, N < 2n, N == 2n; the visit batch is < 100 rays
    (10, False),                  # last_visit > 0; every unvisit batch is < 100 rays
    (11, False),                  # one unvisit frame: snapshotted and decayed, not trained
    (14, True),                   # the_end: num_joint_iters x10
]
GOLDEN_MASK_COUNTS = {2: 0, 3: 15, 4: 20, 6: 3, 7: 4, 8: 0, 9: 5}


def golden_video():
    """the golden's inputs (every frame filled up front: a call reads no frame at or beyond its filtered_id)"""
    S = GOLDEN_SIZE
    video = stub_video(S["buffer"], S["ht"], S["wd"])
    g = torch.Generator().manual_seed(S["seed"])
    video.pose_compensate[0] = random_pose(g, 0.3)
    video.bound[0] = torch.tensor([[-2.0, 2.5], [-1.5, 1.0], [-3.0, 0.5]])
    fill_frames(video, range(S["buffer"]), g, GOLDEN_MASK_COUNTS)
    return video


INPUTS = ("images", "disps_filtered", "mask_filtered", "poses_filtered", "update_priority", "pose_compensate", "bound")


def golden_inputs(video):
    return {k: getattr(video, k).detach().cpu().numpy().copy() for k in INPUTS}


def video_from_golden(g, device="cpu"):
    S = GOLDEN_SIZE
    video = stub_video(S["buffer"], S["ht"], S["wd"], device)
    for k in INPUTS:
        getattr(video, k).copy_(torch.from_numpy(np.asarray(g["in_" + k])).to(device))
    return video
