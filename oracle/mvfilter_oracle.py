"""Twin of the reference's multiview filter (TEST INFRASTRUCTURE — never imported by the product path) and the
analytic scenes its tests run on.

`MultiviewFilterTwin.forward` is src/multiview_filter.py:98-170 restated line for line with the same torch ops,
including the `.cpu()` round trips and the host-side mask / bound work; `iproj`, `depth_filter` and the SE3 class
are injected.  With this library's droid_backends and lietorch it is what the reference runs today after
`goslam_b200.install()`; with oracle.geom_oracle on the CPU it reproduces the reference's own class bit for bit
(tests/golden/multiview_filter.npz).  Only difference to the reference: no colorama, the same escape codes.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

_CYAN, _RESET = "\x1b[36m", "\x1b[0m"


class MultiviewFilterTwin:
    def __init__(self, cfg, args, slam, iproj, depth_filter, SE3, log=print):
        self.args = args
        self.cfg = cfg
        self.device = args.device
        self.warmup = cfg['tracking']['warmup']
        self.filter_thresh = cfg['tracking']['multiview_filter']['thresh']
        self.filter_visible_num = cfg['tracking']['multiview_filter']['visible_num']
        self.kernel_size = cfg['tracking']['multiview_filter']['kernel_size']
        self.bound_enlarge_scale = cfg['tracking']['multiview_filter']['bound_enlarge_scale']
        self.video = slam.video
        self.iproj, self.depth_filter, self.SE3, self.log = iproj, depth_filter, SE3, log

    def pose_dist(self, Tquad0, Tquad1):
        def quat_to_euler(Tquad):
            tx, ty, tz, x, y, z, w = torch.unbind(Tquad, dim=-1)
            t0 = 2.0 * (w * x + y * z)
            t1 = 1.0 - 2.0 * (x * x + y * y)
            roll_x = torch.atan2(t0, t1)

            t2 = 2.0 * (w * y - z * x)
            t2 = torch.clamp(t2, min=-1.0, max=1.0)
            pitch_y = torch.asin(t2)

            t3 = 2.0 * (w * z + x * y)
            t4 = 1.0 - 2.0 * (y * y + z * z)
            yaw_z = torch.atan2(t3, t4)

            return torch.stack([tx, ty, tz, roll_x, pitch_y, yaw_z], dim=-1)

        Teuler0 = quat_to_euler(Tquad0)
        Teuler1 = quat_to_euler(Tquad1)
        dist = (Teuler0 - Teuler1).abs()
        return 1.0 * dist[:, :3].sum(dim=-1) + 2.0 * dist[:, 3:].sum(dim=-1)

    @torch.no_grad()
    def in_bound(self, pts, bound):
        bound = bound.to(pts.device)
        mask_x = (pts[:, 0] < bound[0, 1]) & (pts[:, 0] > bound[0, 0])
        mask_y = (pts[:, 1] < bound[1, 1]) & (pts[:, 1] > bound[1, 0])
        mask_z = (pts[:, 2] < bound[2, 1]) & (pts[:, 2] > bound[2, 0])
        return (mask_x & mask_y & mask_z).bool()

    @torch.no_grad()
    def get_bound_from_pointcloud(self, pts, enlarge_scale=1.0):
        bound = torch.stack([
            torch.min(pts, dim=0, keepdim=False).values,
            torch.max(pts, dim=0, keepdim=False).values,
        ], dim=-1)
        enlarge_bound_length = (bound[:, 1] - bound[:, 0]) * (enlarge_scale - 1.0)
        bound_edge = torch.stack([
            -enlarge_bound_length / 2.0,
            enlarge_bound_length / 2.0,
        ], dim=-1)
        return bound + bound_edge

    def forward(self):
        SE3 = self.SE3
        cur_t = self.video.counter.value
        filtered_t = int(self.video.filtered_id.item())
        if filtered_t < cur_t and cur_t > self.warmup:
            with self.video.get_lock():
                dirty_index = torch.arange(0, cur_t).long().to(self.device)
                poses = torch.index_select(self.video.poses.detach(), dim=0, index=dirty_index)
                disps = torch.index_select(self.video.disps_up.detach(), dim=0, index=dirty_index)
                common_intrinsic_id = 0
                intrinsic = self.video.intrinsics[common_intrinsic_id].detach() * self.video.scale_factor
                w2w = SE3(self.video.pose_compensate[0].clone().unsqueeze(dim=0)).to(self.device)

            points = self.iproj((w2w * SE3(poses).inv()).data, disps, intrinsic).cpu()
            thresh = self.filter_thresh * torch.ones_like(disps.mean(dim=[1, 2]))
            count = self.depth_filter(poses, disps, intrinsic, dirty_index, thresh)

            count = count.cpu()
            disps = disps.cpu()

            masks = (count >= self.filter_visible_num)
            masks = masks & (disps > 0.01 * disps.mean(dim=[1, 2], keepdim=True))
            if masks.sum() < 100:
                return
            sel_points = points.reshape(-1, 3)[masks.reshape(-1)]
            bound = self.get_bound_from_pointcloud(sel_points)

            if isinstance(self.kernel_size, str) and self.kernel_size == 'inf':
                extended_masks = torch.ones_like(masks).bool()
            elif int(self.kernel_size) < 2:
                extended_masks = masks
            else:
                kernel = int(self.kernel_size)
                kernel = (kernel // 2) * 2 + 1
                extended_masks = F.conv2d(
                    masks.unsqueeze(dim=1).float(),
                    weight=torch.ones(1, 1, kernel, kernel, dtype=torch.float, device=masks.device),
                    stride=1,
                    padding=kernel // 2,
                    bias=None,
                ).bool().squeeze(dim=1)

            if extended_masks.sum() < 100:
                return
            sel_points = points.reshape(-1, 3)[extended_masks.reshape(-1)]
            in_bound_mask = self.in_bound(sel_points, bound)
            extended_masks[extended_masks.clone()] = in_bound_mask

            sel_points = points.reshape(-1, 3)[extended_masks.reshape(-1)]
            bound = self.get_bound_from_pointcloud(sel_points)

            priority = self.pose_dist(self.video.poses_filtered[:cur_t].detach(), poses)

            with self.video.mapping.get_lock():
                self.video.update_priority[:cur_t] += priority.detach()
                self.video.mask_filtered[:cur_t] = extended_masks.detach()
                self.video.disps_filtered[:cur_t] = disps.detach()
                self.video.poses_filtered[:cur_t] = poses.detach()
                self.video.filtered_id[0] = cur_t
                self.video.bound[0] = bound

            prefix = "Bound: ["
            bd = bound.tolist()
            prefix += f'[{bd[0][0]:.1f}, {bd[0][1]:.1f}], '
            prefix += f'[{bd[1][0]:.1f}, {bd[1][1]:.1f}], '
            prefix += f'[{bd[2][0]:.1f}, {bd[2][1]:.1f}]]!'
            self.log(_CYAN)
            self.log(f'\n\n Multiview filtering: previous at {filtered_t}, now at {cur_t}, {masks.sum()} valid points found! {prefix}\n')
            self.log(_RESET)
            del points, masks, poses, disps


# ----------------------------------------------------------------------------- scenes
def _quat(axis_angle):
    """unit quaternion (x, y, z, w) of a rotation vector, float64 [..., 3] -> [..., 4]"""
    th = axis_angle.norm(dim=-1, keepdim=True)
    s = torch.where(th > 0, torch.sin(0.5 * th) / th.clamp_min(1e-300), torch.full_like(th, 0.5))
    return torch.cat([s * axis_angle, torch.cos(0.5 * th)], dim=-1)


def _qrot(q, v):
    qv, qw = q[..., :3], q[..., 3:]
    uv = 2.0 * torch.linalg.cross(qv.expand_as(v), v, dim=-1)
    return v + qw * uv + torch.linalg.cross(qv.expand_as(v), uv, dim=-1)


def surface_z(x, y):
    """world height field the cameras look at: tilted and wavy, so no extreme of a point set lies on a plane"""
    return 3.0 + 0.25 * torch.sin(1.7 * x + 0.3) * torch.cos(1.3 * y) + 0.2 * x - 0.15 * y


def _surface_dz(x, y):
    dx = 0.25 * 1.7 * torch.cos(1.7 * x + 0.3) * torch.cos(1.3 * y) + 0.2
    dy = -0.25 * 1.3 * torch.sin(1.7 * x + 0.3) * torch.sin(1.3 * y) - 0.15
    return dx, dy


def trajectory(T, seed):
    """c2w (t, q) in float64 and the w2c poses [T, 7] float32 the video stores"""
    g = torch.Generator().manual_seed(seed)
    i = torch.arange(T, dtype=torch.float64)
    pos = torch.stack([0.04 * i, 0.03 * torch.sin(0.7 * i), 0.05 * torch.cos(0.3 * i)], -1)
    rv = torch.stack([0.02 * torch.sin(0.5 * i), 0.015 * torch.cos(0.4 * i), 0.01 * i / max(T, 1)], -1)
    pos = pos + 0.002 * torch.randn(T, 3, generator=g, dtype=torch.float64)
    q = _quat(rv)
    qi = torch.cat([-q[:, :3], q[:, 3:]], -1)
    w2c = torch.cat([-_qrot(qi, pos), qi], -1).float()
    # re-derive c2w from the stored float32 w2c so the rays match what the kernels see
    qs = w2c[:, 3:].double()
    qc = torch.cat([-qs[:, :3], qs[:, 3:]], -1)
    tc = -_qrot(qc, w2c[:, :3].double())
    return tc, qc, w2c


def raycast(tc, qc, intr_full, ht, wd, device="cpu"):
    """inverse depth [T, ht, wd] float64 of the height field seen from c2w (tc, qc), Newton along each ray"""
    fx, fy, cx, cy = intr_full
    v, u = torch.meshgrid(torch.arange(ht, dtype=torch.float64, device=device),
                          torch.arange(wd, dtype=torch.float64, device=device), indexing="ij")
    rc = torch.stack([(u - cx) / fx, (v - cy) / fy, torch.ones_like(u)], -1)         # [ht, wd, 3]
    out = torch.empty((tc.shape[0], ht, wd), dtype=torch.float64, device=device)
    for f in range(tc.shape[0]):
        q = qc[f].to(device)
        o = tc[f].to(device)
        r = _qrot(q.view(1, 1, 4), rc)
        t = (3.0 - o[2]) / r[..., 2]
        for _ in range(12):
            x, y = o[0] + t * r[..., 0], o[1] + t * r[..., 1]
            h = o[2] + t * r[..., 2] - surface_z(x, y)
            dx, dy = _surface_dz(x, y)
            t = t - h / (r[..., 2] - dx * r[..., 0] - dy * r[..., 1])
        out[f] = 1.0 / t
    return out


def threshold_margin_ok(disps, ulps=8):
    """no pixel within `ulps` float32 ulp of its frame's 0.01 * mean threshold (fp32 mean and fp64 mean both)"""
    d = disps.float()
    for mean in (d.mean(dim=[1, 2]), d.double().mean(dim=[1, 2]).float()):
        thr = 0.01 * mean
        gap = torch.nextafter(thr, torch.full_like(thr, math.inf)) - thr
        if ((d - thr[:, None, None]).abs() <= ulps * gap[:, None, None]).any():
            return False
    return True


def make_disps(tc, qc, intr_full, ht, wd, seed, noise=0.002, hole_frac=0.02, far_frac=0.01, device="cpu",
               fp16_exact=False):
    """float32 inverse depth with multiplicative noise, holes (d = 0) and far pixels (d below 0.01 * mean);
    fp16_exact rounds every value to one a float16 holds, so a fixture can store it in half the bytes"""
    g = torch.Generator(device=device).manual_seed(seed)
    d = raycast(tc, qc, intr_full, ht, wd, device=device)
    T = d.shape[0]
    d = d * (1.0 + noise * torch.randn(d.shape, generator=g, dtype=torch.float64, device=device))
    r = torch.rand(d.shape, generator=g, dtype=torch.float64, device=device)
    d = torch.where(r < hole_frac, torch.zeros_like(d), d)
    far = (r >= hole_frac) & (r < hole_frac + far_frac)
    d = torch.where(far, 0.003 * d.mean(dim=[1, 2], keepdim=True) * (1.0 + r), d)
    d = d.half().float() if fp16_exact else d.float()
    assert T == 0 or threshold_margin_ok(d)
    return d


def full_intrinsics(ht, wd):
    """full-resolution (fx, fy, cx, cy): multiples of 1/8, so intrinsics[0] = these / 8 is exact"""
    f = round(0.8 * wd * 8) / 8.0
    return (f, f, (wd - 1) / 2.0, (ht - 1) / 2.0)


def compensate_pose():
    """a non-identity pose_compensate (w2w), float32 [1, 7]"""
    q = _quat(torch.tensor([[0.05, -0.03, 0.08]], dtype=torch.float64))
    return torch.cat([torch.tensor([[0.3, -0.2, 0.1]], dtype=torch.float64), q], -1).float()


def stub_video(n, ht, wd, device="cpu"):
    """the DepthVideo attributes the filter reads and writes, initialised as DepthVideo does"""
    from multiprocessing import Value
    import types
    ident = torch.tensor([[0, 0, 0, 0, 0, 0, 1.0]], device=device)
    video = types.SimpleNamespace(
        counter=Value("i", 0), mapping=Value("i", 0), scale_factor=8, poses=ident.repeat(n, 1),
        disps_up=torch.zeros(n, ht, wd, device=device), intrinsics=torch.zeros(n, 4, device=device),
        pose_compensate=ident.clone(), poses_filtered=ident.repeat(n, 1),
        disps_filtered=torch.zeros(n, ht, wd, device=device), mask_filtered=torch.zeros(n, ht, wd, device=device),
        update_priority=torch.zeros(n, device=device), filtered_id=torch.tensor([-1], dtype=torch.int, device=device),
        bound=torch.zeros(1, 3, 2, device=device))
    video.get_lock = video.counter.get_lock
    return video


def stub_slam(video, device):
    import types
    n, ht, wd = video.disps_up.shape
    fx, fy, cx, cy = (video.intrinsics[0] * 8).tolist()
    return (types.SimpleNamespace(device=device),
            types.SimpleNamespace(net=None, video=video, verbose=False, mode="mono", H=ht, W=wd, fx=fx, fy=fy, cx=cx,
                                  cy=cy))


def filter_cfg(kernel_size, warmup, thresh=0.01, visible_num=2):
    return {"tracking": {"warmup": warmup, "multiview_filter": {
        "thresh": thresh, "visible_num": visible_num, "kernel_size": kernel_size, "bound_enlarge_scale": 1.2}}}


def numpy_state(video, names=("poses_filtered", "disps_filtered", "mask_filtered", "update_priority",
                              "filtered_id", "bound")):
    return {n: getattr(video, n).detach().cpu().numpy().copy() for n in names}



# ----------------------------------------------------------------------------- golden scenario
GOLDEN_SIZE = dict(buffer=14, ht=40, wd=56, warmup=8)
# (counter, kernel_size, what changes in the video before the pass)
GOLDEN_PASSES = [
    (8, 1, "base"),          # cur_t <= warmup: no-op
    (10, 1, None),           # first commit
    (10, 1, None),           # filtered_t >= cur_t: no-op
    (12, 2, "perturb"),      # kernel 2 -> 3x3 dilation; priority accumulates
    (13, 1, "scramble"),     # poses scrambled: fewer than 100 mask points, early return
    (13, 1, "flat"),         # constant inverse depth, identity poses: every z equal, empty in-bound set (raises)
    (14, "inf", "perturb"),  # every pixel extended
]



# ----------------------------------------------------------------------------- golden file layout
# Stored compactly: the distinct inverse-depth inputs once, as float16 (the scenes are fp16-exact); masks as bits;
# disps_filtered not at all — after every pass it is rows [:filtered_id] of the inputs of the last committing pass
# (zeros before the first commit), which the generator asserts before it drops them.
_SMALL_STATE = ("poses_filtered", "update_priority", "filtered_id", "bound")


def golden_pack(passes, init, intrinsics, size):
    """passes: list of dicts with counter, kernel_size, raised, log, inputs (poses, disps, compensate) and the
    state after the pass (numpy_state)"""
    sets, idx, src, last = [], [], [], -1
    for p, r in enumerate(passes):
        d = r["disps"]
        assert np.array_equal(d.astype(np.float16).astype(np.float32), d)
        for i, s in enumerate(sets):
            if np.array_equal(s, d):
                break
        else:
            sets.append(d)
            i = len(sets) - 1
        idx.append(i)
        fid = int(r["state"]["filtered_id"][0])
        if fid != (int(passes[p - 1]["state"]["filtered_id"][0]) if p else -1):
            last = p
        src.append(last)
        want = np.zeros_like(d)
        if last >= 0:
            want[:fid] = passes[last]["disps"][:fid]
        assert np.array_equal(want.view(np.uint32), r["state"]["disps_filtered"].view(np.uint32)), p
        m = r["state"]["mask_filtered"]
        assert np.array_equal(m, (m != 0).astype(m.dtype))
    out = {
        "size": np.array(size), "intrinsics": intrinsics,
        "counter": np.array([r["counter"] for r in passes]),
        "kernel_size": np.array([r["kernel_size"] for r in passes]),
        "raised": np.array([r["raised"] for r in passes]), "log": np.array([r["log"] for r in passes]),
        "in_poses": np.stack([r["poses"] for r in passes]),
        "in_compensate": np.stack([r["compensate"] for r in passes]),
        "in_disps_set": np.stack(sets).astype(np.float16), "in_disps_idx": np.array(idx),
        "out_disps_src": np.array(src),
        "out_mask_bits": np.stack([np.packbits(r["state"]["mask_filtered"].reshape(-1) != 0) for r in passes]),
    }
    for k in _SMALL_STATE:
        out["out_" + k] = np.stack([r["state"][k] for r in passes])
        out["init_" + k] = init[k]
    return out


def golden_unpack(g):
    """the stored golden as full arrays: in_disps, out_<state> for every pass, init_<state>"""
    n, ht, wd = [int(x) for x in g["size"][:3]]
    sets = g["in_disps_set"].astype(np.float32)
    in_disps = sets[g["in_disps_idx"]]
    P = len(g["counter"])
    out = {k: g[k] for k in g.files}
    out["in_disps"] = in_disps
    dfilt = np.zeros((P, n, ht, wd), np.float32)
    for p in range(P):
        src = int(g["out_disps_src"][p])
        if src >= 0:
            fid = int(g["out_filtered_id"][p][0])
            dfilt[p, :fid] = in_disps[src, :fid]
    out["out_disps_filtered"] = dfilt
    out["out_mask_filtered"] = np.unpackbits(g["out_mask_bits"], axis=1, count=n * ht * wd).reshape(
        P, n, ht, wd).astype(np.float32)
    out["init_disps_filtered"] = np.zeros((n, ht, wd), np.float32)
    out["init_mask_filtered"] = np.zeros((n, ht, wd), np.float32)
    return out
