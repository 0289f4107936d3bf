"""`Mapper` — the reference's mapping process (src/mapping.py:11-300) with its constructor, config keys, attributes and
call schedule, with the frame hand-over and the ray batches on the sm_90a kernels of csrc/mapping.cu.

Per call the reference runs DepthVideo.get_mapping_item once per entry of the visit and unvisit lists (clones, the
depth reciprocal, an SE3 chain and a priority decay: ~50 small launches per frame), and per training iteration
build_rays once per listed frame (~25 launches, two pageable copies and a masked_select sync each) plus four
torch.cat.  Here:
    snapshot_frames   one lock, three launches: every touched frame's masked pixels as compact records and the
                      priority decays; the c2w of all frames in one batched lietorch call; ONE host read (the N_f)
    build_ray_batch   the reference's torch.randint draws into slices of one buffer, then one launch for the batch
The training step (`optimize_map`) is the reference's, on this library's renderer and InstantNeuS.

Documented differences:
  - cfg['mapping']['BA'] true raises NotImplementedError at construction; `RefiningMapper` (below) is the same process
    with the reference's camera refinement.  Every shipped config sets it false.
  - importing this module does not turn on torch.autograd.set_detect_anomaly(True) process-wide.
  - the snapshot takes the video's mapping lock once per call, where the reference takes it once per frame.
There is no CPU path: the video buffers must live on a CUDA device.
"""
import ctypes
import os
from collections import namedtuple
from time import gmtime, strftime

import numpy as np
import torch

from . import _lib
from . import lietorch

try:
    from colorama import Fore as _Fore, Style as _Style
    _MAGENTA, _RESET = _Fore.MAGENTA, _Style.RESET_ALL
except ImportError:                              # colorama is optional: the same escape codes
    _MAGENTA, _RESET = "\x1b[35m", "\x1b[0m"


# ----------------------------------------------------------------------------- host planning (no device)
def random_select(l, k, start=0):
    """up to k frame ids in [start, l): one uniform draw in each of k equal strata (np.random.rand(k)), truncated,
    ids <= 0 dropped — src/nerf_func.py:28-40 (same numpy calls in the same order)"""
    width = (l - start) / k
    picks = np.linspace(start, l - 1 - width, k) + np.random.rand(k) * width
    return [int(v) for v in list(picks.clip(start, l - 1)) if v > 0]


def distinct_frames(frames):
    """(distinct frame ids in order of first occurrence, occurrence count of each)"""
    order, occ = [], {}
    for f in frames:
        f = int(f)
        if f not in occ:
            order.append(f)
            occ[f] = 0
        occ[f] += 1
    return order, [occ[f] for f in order]


def visit_frames(cur_idx, last_visit, priority_order, window):
    """the visit list of one call: the two newest filtered keyframes, then (once something has been visited) the ten
    of highest update priority (`priority_order` = torch.sort(..., descending=True) indices as numpy) and
    random_select(last_visit, window - 12)"""
    visit = [cur_idx - 1, cur_idx - 2]
    if last_visit > 0:
        visit += list(priority_order)[:10]
        visit += random_select(last_visit, window - 12)
    return visit


BatchPlan = namedtuple("BatchPlan", "draw rows offsets R n_draws")


def plan_batch(counts, n_rays):
    """the reference's per-frame rule `0 < n_rays < N // 2`: draw n_rays random records, else take all N (none when
    N == 0).  counts: N_f of each list entry in list order.  Returns per entry the draw size (0 = all records), its row
    count and first row, the batch size R and the total number of draws."""
    draw = [n_rays if 0 < n_rays < n // 2 else 0 for n in counts]
    rows = [d if d > 0 else n for d, n in zip(draw, counts)]
    offsets = [0] * len(rows)
    for i in range(1, len(rows)):
        offsets[i] = offsets[i - 1] + rows[i - 1]
    return BatchPlan(draw, rows, offsets, sum(rows), sum(draw))


# ----------------------------------------------------------------------------- device helpers
class Snapshot:
    """records of the frames one Mapper call touches (csrc/mapping.cu), read by build_ray_batch.
    frames: distinct ids (slot order); counts: N_f per slot; c2w [F,4,4] f32."""

    def __init__(self, frames, counts, c2w, workspace, H, W):
        self.frames, self.counts, self.c2w, self.workspace, self.H, self.W = frames, counts, c2w, workspace, H, W
        self.slot = {f: s for s, f in enumerate(frames)}

    def count(self, frame):
        return self.counts[self.slot[int(frame)]]


def _check_buffer(t, name):
    if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
        raise RuntimeError("snapshot_frames: video.%s must be a contiguous f32 CUDA tensor (no CPU fallback)" % name)


def snapshot_frames(video, frames, decay):
    """DepthVideo.get_mapping_item for every entry of `frames` (repeats allowed, in call order) under ONE hold of the
    video's mapping lock: the masked pixels of each distinct frame, its depth 1/(disp+1e-7) and rgb, and
    update_priority[f] *= decay once per occurrence.  The N_f are read back before the lock is released (the one host
    synchronisation), so nothing reads the live buffers afterwards.  c2w = (SE3(pose_compensate[0]) *
    SE3(poses_filtered[f]).inv()).matrix() for all frames in one batched call."""
    order, occ = distinct_frames(frames)
    for name in ("images", "mask_filtered", "disps_filtered", "update_priority", "poses_filtered"):
        _check_buffer(getattr(video, name), name)
    dev = video.images.device
    buffer, _, H, W = video.images.shape
    if any(f < 0 or f >= buffer for f in order):
        raise IndexError("snapshot_frames: frame id outside the video buffer [0, %d)" % buffer)
    F = len(order)
    if F == 0:
        return Snapshot([], [], torch.empty((0, 4, 4), device=dev), None, H, W)
    nbytes = int(_lib.load().goslam_mapping_snapshot_workspace_bytes(F, H, W))
    if nbytes == 0:
        raise RuntimeError("snapshot_frames: invalid size (%d frames of %d x %d)" % (F, H, W))
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    counts = torch.empty((F,), dtype=torch.int32, device=dev)
    ids = torch.tensor([order, occ], dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
    with video.mapping.get_lock():
        _lib.call("mapping_snapshot", video.images, video.mask_filtered, video.disps_filtered, video.update_priority,
                  buffer, H, W, ids[0], ids[1], F, float(decay), ws, nbytes, counts)
        poses = video.poses_filtered.index_select(0, ids[0].long())
        comp = video.pose_compensate[0:1].clone()
        n_f = counts.tolist()
    c2w = (lietorch.SE3(comp) * lietorch.SE3(poses).inv()).matrix().contiguous()
    return Snapshot(order, n_f, c2w, ws, H, W)


RayBatch = namedtuple("RayBatch", "rays_o rays_d depth color draws")


def _draw_batch(snapshot, frame_list, n_rays):
    """(slots, counts, plan, draws) of one batch: the reference's torch.randint(N_f, (n_rays,)) per random-branch entry
    in list order on the current CUDA generator, into slices of one buffer"""
    slots = [snapshot.slot[int(f)] for f in frame_list]
    counts = [snapshot.counts[s] for s in slots]
    plan = plan_batch(counts, n_rays)
    draws = torch.empty((plan.n_draws,), dtype=torch.int64, device=snapshot.c2w.device)
    at = 0
    for n, d in zip(counts, plan.draw):
        if d > 0:
            draws[at:at + d].random_(0, n)                     # == torch.randint(n, (d,)): the same Philox consumption
            at += d
    return slots, counts, plan, draws


def build_ray_batch(snapshot, frame_list, n_rays, intrinsics):
    """build_rays(0, H, 0, W, n_rays, ..., nerf_coordinate=False, mask=mask) for every entry of frame_list (repeats
    allowed), concatenated: rays_o, rays_d, color [R,3], depth [R] f32 and the drawn record indices `draws`.
    intrinsics = (fx, fy, cx, cy).  The random draws are the reference's torch.randint(N_f, (n_rays,)) per
    random-branch entry in list order on the current CUDA generator; no host synchronisation."""
    fx, fy, cx, cy = [float(v) for v in intrinsics]
    slots, counts, plan, draws = _draw_batch(snapshot, frame_list, n_rays)
    dev = snapshot.c2w.device
    rays_o = torch.empty((plan.R, 3), dtype=torch.float32, device=dev)
    rays_d = torch.empty((plan.R, 3), dtype=torch.float32, device=dev)
    color = torch.empty((plan.R, 3), dtype=torch.float32, device=dev)
    depth = torch.empty((plan.R,), dtype=torch.float32, device=dev)
    if plan.R > 0:
        n = len(slots)
        arr = ctypes.c_int * n
        _lib.call("mapping_rays", snapshot.workspace, snapshot.workspace.numel(), len(snapshot.frames), snapshot.H,
                  snapshot.W, snapshot.c2w, draws, plan.n_draws, n, arr(*slots), arr(*counts), arr(*plan.draw), fx, fy,
                  cx, cy, rays_o, rays_d, depth, color, plan.R)
    return RayBatch(rays_o, rays_d, depth, color, draws)


def c2w_to_quadt(c2w):
    """Rt_to_quaternion(c2w, Tquad=False) (src/nerf_func.py:69-88) for c2w [n,4,4] or [4,4] on the device, one launch:
    (w, x, y, z, tx, ty, tz) f32, the unit quaternion by Shepperd's method in double with w >= 0.  The reference's sign
    comes from mathutils; either sign gives the same rotation and, under AdamW, the negated trajectory."""
    _lib.need_cuda("c2w_to_quadt", c2w)
    m = c2w.detach().to(torch.float32).contiguous()
    out = torch.empty(m.shape[:-2] + (7,), dtype=torch.float32, device=m.device)
    n = out.numel() // 7
    if n > 0:
        _lib.call("mapping_c2w_to_quadt", m, n, out)
    return out


class _PoseRays(torch.autograd.Function):
    """rays_o, rays_d of one batch from per-entry leaves quadt [n,7]; backward: d quadt (csrc/mapping.cu)"""

    @staticmethod
    def forward(ctx, quadt, snapshot, table, draws, intrinsics, R):
        q = quadt.detach().to(torch.float32).contiguous()
        dev = q.device
        rays_o = torch.empty((R, 3), dtype=torch.float32, device=dev)
        rays_d = torch.empty((R, 3), dtype=torch.float32, device=dev)
        color = torch.empty((R, 3), dtype=torch.float32, device=dev)
        depth = torch.empty((R,), dtype=torch.float32, device=dev)
        if R > 0:
            _lib.call("mapping_pose_rays", snapshot.workspace, snapshot.workspace.numel(), len(snapshot.frames),
                      snapshot.H, snapshot.W, q, draws, draws.numel(), *table, *intrinsics, rays_o, rays_d, depth,
                      color, R)
        ctx.args = (q, quadt.dtype, snapshot, table, draws, intrinsics, R)
        ctx.mark_non_differentiable(depth, color)
        return rays_o, rays_d, depth, color

    @staticmethod
    def backward(ctx, g_o, g_d, _g_depth, _g_color):
        q, dtype, snapshot, table, draws, intrinsics, R = ctx.args
        z = None if g_o is not None and g_d is not None else torch.zeros((R, 3), dtype=torch.float32, device=q.device)
        g_o = z if g_o is None else g_o.to(torch.float32).contiguous()
        g_d = z if g_d is None else g_d.to(torch.float32).contiguous()
        d_q = torch.empty_like(q)
        _lib.call("mapping_pose_rays_backward", snapshot.workspace, snapshot.workspace.numel(), len(snapshot.frames),
                  snapshot.H, snapshot.W, q, draws, draws.numel(), *table, *intrinsics, g_o, g_d, R, d_q)
        return d_q.to(dtype), None, None, None, None, None


def build_pose_ray_batch(snapshot, frame_list, n_rays, intrinsics, quadt):
    """build_ray_batch with entry e's pose quaternion_to_Rt(quadt[e]) (src/nerf_func.py:44-112) in place of its
    frame's c2w: quadt [len(frame_list),7], one row per entry (a frame listed twice has two rows).  rays_o and rays_d
    are differentiable with respect to quadt (goslam_mapping_pose_rays_backward); depth, color and the draws are
    build_ray_batch's, on the same generator, so the random stream does not depend on refinement."""
    if quadt.dim() != 2 or quadt.shape != (len(frame_list), 7):
        raise ValueError("build_pose_ray_batch: quadt must be [%d, 7], got %s" % (len(frame_list), tuple(quadt.shape)))
    _lib.need_cuda("build_pose_ray_batch", quadt)
    intr = tuple(float(v) for v in intrinsics)
    slots, counts, plan, draws = _draw_batch(snapshot, frame_list, n_rays)
    n = len(slots)
    arr = ctypes.c_int * n
    table = (n, arr(*slots), arr(*counts), arr(*plan.draw))
    rays_o, rays_d, depth, color = _PoseRays.apply(quadt, snapshot, table, draws, intr, plan.R)
    return RayBatch(rays_o, rays_d, depth, color, draws)


def all_rays(H, W, intrinsics, c2w):
    """build_all_rays(H, W, fx, fy, cx, cy, c2w, nerf_coordinate=False) flattened: rays_o, rays_d [H*W,3]"""
    fx, fy, cx, cy = [float(v) for v in intrinsics]
    _lib.need_cuda("all_rays", c2w)
    m = c2w.detach().to(torch.float32).contiguous()
    rays_o = torch.empty((H * W, 3), dtype=torch.float32, device=m.device)
    rays_d = torch.empty((H * W, 3), dtype=torch.float32, device=m.device)
    _lib.call("mapping_all_rays", m, int(H), int(W), fx, fy, cx, cy, rays_o, rays_d)
    return rays_o, rays_d


# ----------------------------------------------------------------------------- the process
class _TextLogger:
    """the reference's TextLogger (src/Logger.py): 'Start recording...' header, '<UTC time> - msg' lines, echoed"""

    def __init__(self, log_file):
        self.log_file = log_file
        with open(log_file, 'w') as fp:
            fp.write('Start recording...\n')

    def info(self, msg):
        msg = strftime("%Y-%m-%d %H:%M:%S", gmtime()) + ' - ' + msg
        print(msg)
        with open(self.log_file, 'a') as fp:
            fp.write(msg + '\n')


class Mapper(object):
    _refines_cameras = False          # RefiningMapper: mapping.BA is accepted

    def __init__(self, cfg, args, slam):
        self.cfg = cfg
        self.args = args
        self.verbose = slam.verbose
        self.bound = slam.bound
        self.video = slam.video
        self.mapping_net = slam.mapping_net
        self.renderer = slam.renderer
        self.reload_map = slam.reload_map
        self.output = slam.output

        m = cfg['mapping']
        self.device = m['device']
        if torch.device(self.device).type != "cuda":
            raise RuntimeError("goslam_b200.Mapper: a CUDA device is required (no CPU fallback)")
        self.num_joint_iters = m['iters']
        self.decay = float(m['decay'])
        self.w_color_loss = m['w_color_loss']
        self.w_sdf_loss = m['w_sdf_loss']
        self.w_eikonal_loss = m['w_eikonal_loss']
        self.uncertainty_based = m['uncertainty_weight_loss']
        self.BA = m['BA']
        if self.BA and not self._refines_cameras:
            raise NotImplementedError("goslam_b200.Mapper: mapping-side camera refinement (mapping.BA: True) is not "
                                      "supported")
        self.BA_cam_lr = m['BA_cam_lr']
        self.mapping_pixels = m['pixels']
        self.mapping_window_size = m['mapping_window_size']

        self.H, self.W, self.fx, self.fy, self.cx, self.cy = slam.H, slam.W, slam.fx, slam.fy, slam.cx, slam.cy
        self.local_step = 0
        self.global_step = 0
        self.last_visit = 0
        self.init = True

        os.makedirs(f'{self.output}/logs/mapping/', exist_ok=True)
        self.txt = _TextLogger(f'{self.output}/logs/mapping/log.txt')

        net_param = self.mapping_net.get_training_parameters(ignore_keys=())
        grid_param = self.mapping_net.get_volume_parameters()
        self.train_params = list(net_param) + list(grid_param)
        self.optimizer = torch.optim.AdamW([
            {'params': net_param, 'lr': m['net_lr']},
            {'params': grid_param, 'lr': m['grid_lr']},
        ], betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)

    def optimize_map(self, rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters):
        """num_joint_iters AdamW steps on one ray batch with the reference's loss (src/mapping.py:60-148)"""
        device = self.device
        for _ in range(num_joint_iters):
            self.local_step += 1
            self.global_step += 1
            optimizer.zero_grad()
            with torch.enable_grad():
                ret = self.renderer.render_batch_ray(rays_o=rays_o, rays_d=rays_d, net=self.mapping_net.to(device),
                                                     render_params={'global_step': self.global_step}, device=device,
                                                     gt_depth=rays_depth)
            rays_depth = rays_depth.reshape(-1, 1)
            valid = (rays_depth > 0).reshape(-1)
            rays_depth = rays_depth[valid]
            rays_color = rays_color[valid]
            est_color = ret['color'][valid]
            est_depth = ret['depth'][valid]
            sdf = ret['sdf'][valid]
            z_vals = ret['z_vals'][valid]
            depth_variance = ret['depth_variance'][valid]
            uncertainty_weight = 1.0 / torch.sqrt(depth_variance.detach() + 1e-10)
            if not self.uncertainty_based:
                uncertainty_weight = torch.ones_like(uncertainty_weight)
            assert rays_depth.shape == est_depth.shape, f'{rays_depth.shape}, {est_depth.shape}!'

            total_loss = 0.0
            color_loss = torch.abs(est_color - rays_color).mean()
            total_loss = total_loss + color_loss * self.w_color_loss
            depth_loss = (torch.abs(est_depth - rays_depth) * uncertainty_weight).mean()
            total_loss = total_loss + depth_loss * 1.0
            sdf_loss = 0.0
            if self.w_sdf_loss > 0:
                sdf_loss, sparse_loss = self.mapping_net.compute_sdf_error(sdf=sdf, z_vals=z_vals, gt_depth=rays_depth)
                total_loss = total_loss + (sdf_loss + sparse_loss) * self.w_sdf_loss
            if self.w_eikonal_loss > 0:
                total_loss = total_loss + self.w_eikonal_loss * ret['gradient_error'].mean()

            total_loss.backward(retain_graph=False)
            torch.nn.utils.clip_grad_norm_(self.train_params, max_norm=35.0)
            optimizer.step()
            optimizer.zero_grad()

            if (self.local_step % self.num_joint_iters == 0) and self.verbose:
                list_lr = [round(g['lr'], 6) for g in optimizer.param_groups]
                self.txt.info('Lr : {}'.format(list_lr) +
                              f' | Loss of total: {total_loss.detach():.4f}, depth: {depth_loss:.4f}, '
                              f'color: {color_loss:.4f}, sdf: {sdf_loss:.4f}, n_rays: {rays_o.shape}!')

    def _camera_leaves(self, snapshot, visit_list, optimizer):
        """the per-entry pose leaves of this call's visit iterations: none (RefiningMapper makes them)"""
        return None

    def _batch(self, snapshot, frame_list, n_rays, leaves):
        return build_ray_batch(snapshot, frame_list, n_rays, (self.fx, self.fy, self.cx, self.cy))

    def _train(self, snapshot, frame_list, n_rays, optimizer, leaves=None):
        batch = self._batch(snapshot, frame_list, n_rays, leaves)
        if len(batch.rays_o) < 100:
            return
        self.optimize_map(rays_o=batch.rays_o, rays_d=batch.rays_d, rays_color=batch.color, rays_depth=batch.depth,
                          optimizer=optimizer, num_joint_iters=1)

    def __call__(self, the_end=False):
        cur_idx = int(self.video.filtered_id.item())
        if cur_idx <= 1:
            return
        timestamp = self.video.timestamp[cur_idx - 1]
        num_joint_iters = self.num_joint_iters * 10 if the_end else self.num_joint_iters
        self.local_step = 0

        unvisit_list = list(range(self.last_visit, cur_idx))
        order = None
        if self.last_visit > 0:
            priority = self.video.update_priority[:self.last_visit].detach()
            _, indices = torch.sort(priority, dim=0, descending=True)
            order = indices.cpu().numpy()
        visit_list = visit_frames(cur_idx, self.last_visit, order, self.mapping_window_size)

        snapshot = snapshot_frames(self.video, visit_list + unvisit_list, self.decay)
        optimizer = self.optimizer
        leaves = self._camera_leaves(snapshot, visit_list, optimizer)      # before last_visit moves

        bd = self.video.get_bound()
        with self.video.mapping.get_lock():
            self.mapping_net.update_bound(bd)
        bd = self.mapping_net.realtime_bound.tolist()
        prefix = "Bound: ["
        prefix += f'[{bd[0][0]:.1f}, {bd[0][1]:.1f}], '
        prefix += f'[{bd[1][0]:.1f}, {bd[1][1]:.1f}], '
        prefix += f'[{bd[2][0]:.1f}, {bd[2][1]:.1f}]]; '
        print(_MAGENTA)
        if self.verbose:
            self.txt.info(prefix + 'Mapping Frame {}, unvisit {}, has visited {}'.format(
                timestamp.item(), unvisit_list, visit_list))
        elif len(unvisit_list) > 2:
            self.txt.info(prefix + 'Mapping Frame {}, unvisit kf are: {}!'.format(timestamp.item(), unvisit_list))
        print(_RESET)

        unvisit_factor = num_joint_iters * 10 if self.init else num_joint_iters
        if len(unvisit_list) > 2:
            self.last_visit = cur_idx
            for _ in range(unvisit_factor):
                sub_unvisit_list = list(np.random.choice(unvisit_list, self.mapping_window_size))
                self._train(snapshot, sub_unvisit_list, self.mapping_pixels // len(sub_unvisit_list), optimizer)
        torch.cuda.empty_cache()

        for _ in range(num_joint_iters):
            if len(visit_list) < 1:
                continue
            self._train(snapshot, visit_list, self.mapping_pixels // len(visit_list), optimizer, leaves)

        self.reload_map += 1
        self.init = False
        del snapshot
        torch.cuda.empty_cache()


class RefiningMapper(Mapper):
    """Mapper with the reference's camera refinement in mapping (cfg['mapping']['BA'], src/mapping.py:173-194, 266-273):
    once last_visit >= 10 (tested before this call moves it), every entry of the visit list — a frame listed twice
    gets two — has a quaternion-translation leaf from its snapshot c2w (c2w_to_quadt, one launch); the leaves replace
    the optimizer's previous camera group (kept while it has more than the two network groups) as one group at
    BA_cam_lr with the optimizer's other defaults; every visit iteration builds its rays from the current leaves
    (build_pose_ray_batch), so AdamW moves the map and the cameras together.  The unvisit iterations use the snapshot
    c2w: the leaves have no gradient there and AdamW skips them.  clip_grad_norm_ covers the network parameters only,
    and the refined poses are not written back to the video, as in the reference.  With BA false, or before
    last_visit reaches 10, it is Mapper.

    Documented difference: the AdamW state of a camera group that is replaced is dropped from optimizer.state (the
    reference keeps it, unread, for the life of the optimizer)."""
    _refines_cameras = True

    def _camera_leaves(self, snapshot, visit_list, optimizer):
        if not (self.BA and self.last_visit >= 10):
            return None
        dev = snapshot.c2w.device
        slots = torch.tensor([snapshot.slot[int(f)] for f in visit_list], dtype=torch.int64).pin_memory()
        quadt = c2w_to_quadt(snapshot.c2w.index_select(0, slots.to(dev, non_blocking=True)))
        leaves = [q.detach().requires_grad_(True) for q in quadt]          # rows of one buffer, each its own leaf
        if len(optimizer.param_groups) > 2:
            for p in optimizer.param_groups.pop()['params']:
                optimizer.state.pop(p, None)
        if len(leaves) > 0:
            optimizer.add_param_group({'params': leaves, 'lr': self.BA_cam_lr})
        return leaves

    def _batch(self, snapshot, frame_list, n_rays, leaves):
        if leaves is None:
            return build_ray_batch(snapshot, frame_list, n_rays, (self.fx, self.fy, self.cx, self.cy))
        return build_pose_ray_batch(snapshot, frame_list, n_rays, (self.fx, self.fy, self.cx, self.cy),
                                    torch.stack(leaves))
