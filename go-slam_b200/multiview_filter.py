"""`MultiviewFilter` — the reference's multiview-filter process (src/multiview_filter.py:9-170) with its constructor,
config keys and attributes, on top of the sm_90a kernels of csrc/geom.cu.

One pass of the reference runs iproj + depth_filter on the GPU, copies points / counts / disps to the host, builds
the masks and bounds there and copies the results back into the shared video buffers.  Here the pass is two C calls
on one stream and nothing leaves the device:
    goslam_mvfilter_compute  frame means, votes, mask1 + first bound, extended mask + in-bound test + second bound
    goslam_mvfilter_commit   gated on the device: priority, poses / disps / mask / bound / filtered_id, status
The only host reads are the ones the reference also makes (counter, filtered_id) and the 4-entry status record
after the stream has been synchronised.

One documented difference: when the in-bound point set is empty the reference's torch.min raises an IndexError;
here the pass raises RuntimeError.  In both cases nothing is committed.
"""
import torch

from . import _lib
from . import lietorch

_CYAN, _RESET = "\x1b[36m", "\x1b[0m"          # colorama's Fore.CYAN / Style.RESET_ALL


class MultiviewFilter(torch.nn.Module):
    def __init__(self, cfg, args, slam):
        super().__init__()
        self.args = args
        self.cfg = cfg
        self.device = args.device
        if torch.device(self.device).type != "cuda":
            raise RuntimeError("goslam_b200.MultiviewFilter: a CUDA device is required (no CPU fallback)")
        self.warmup = cfg['tracking']['warmup']
        self.filter_thresh = cfg['tracking']['multiview_filter']['thresh']
        self.filter_visible_num = cfg['tracking']['multiview_filter']['visible_num']
        self.kernel_size = cfg['tracking']['multiview_filter']['kernel_size']
        self.bound_enlarge_scale = cfg['tracking']['multiview_filter']['bound_enlarge_scale']
        self.net = slam.net
        self.video = slam.video
        self.verbose = slam.verbose
        self.mode = slam.mode

        self.H, self.W, self.fx, self.fy, self.cx, self.cy = slam.H, slam.W, slam.fx, slam.fy, slam.cx, slam.cy
        self._snap = None
        self._ws = None

    # 0 = every pixel ('inf'), 1 = mask1, k >= 2 = box dilation (src/multiview_filter.py:126-140)
    def _kernel_code(self):
        if isinstance(self.kernel_size, str) and self.kernel_size == 'inf':
            return 0
        k = int(self.kernel_size)
        return 1 if k < 2 else k

    def _snapshot(self):
        """snapshot buffers sized for the whole video, allocated once"""
        if self._snap is None:
            v = self.video
            dev = v.poses.device
            n, ht, wd = v.disps_up.shape
            self._snap = {
                "poses": torch.empty((n, 7), dtype=torch.float32, device=dev),
                "disps": torch.empty((n, ht, wd), dtype=torch.float32, device=dev),
                "intrinsic": torch.empty((4,), dtype=torch.float32, device=dev),
                "w2w": torch.empty((1, 7), dtype=torch.float32, device=dev),
                "status": torch.zeros((4,), dtype=torch.int64, device=dev),
            }
            nbytes = _lib.load().goslam_mvfilter_workspace_bytes(n, ht, wd)
            if nbytes == 0:
                raise RuntimeError("MultiviewFilter: invalid video size (%d, %d, %d)" % (n, ht, wd))
            self._ws = torch.empty((int(nbytes),), dtype=torch.uint8, device=dev)
        return self._snap

    @torch.no_grad()
    def forward(self):
        v = self.video
        cur_t = v.counter.value
        filtered_t = int(v.filtered_id.item())
        if not (filtered_t < cur_t and cur_t > self.warmup):
            return
        b = self._snapshot()
        T = cur_t
        n, ht, wd = v.disps_up.shape
        if T > n:
            raise RuntimeError("MultiviewFilter: counter %d exceeds the video buffer %d" % (T, n))
        dev = b["poses"].device
        with torch.cuda.device(dev):
            with v.get_lock():
                b["poses"][:T].copy_(v.poses[:T])
                b["disps"][:T].copy_(v.disps_up[:T])
                torch.mul(v.intrinsics[0], v.scale_factor, out=b["intrinsic"])
                b["w2w"].copy_(v.pose_compensate[0:1])
            poses, disps = b["poses"][:T], b["disps"][:T]
            # the reference's iproj argument, with the same SE3 algebra
            poses_world = (lietorch.SE3(b["w2w"]) * lietorch.SE3(poses).inv()).data.contiguous()
        _lib.call("mvfilter_compute", poses, poses_world, disps, b["intrinsic"], float(self.filter_thresh),
                  int(self.filter_visible_num), self._kernel_code(), T, ht, wd, self._ws, self._ws.numel())
        with v.mapping.get_lock():
            _lib.call("mvfilter_commit", poses, disps, self._ws, self._ws.numel(), T, ht, wd, v.poses_filtered,
                      v.disps_filtered, v.mask_filtered, v.update_priority, v.filtered_id, v.bound, b["status"])
            # mapping reads these buffers from another process as soon as the lock is released
            torch.cuda.current_stream(dev).synchronize()
            n_mask, _, n_final, committed = b["status"].tolist()
            bd = v.bound[0].tolist()
        if n_mask < 100:
            return
        if not committed:
            raise RuntimeError("MultiviewFilter: no filtered point lies strictly inside the bound of the %d "
                               "mask points (n_final = %d); nothing committed" % (n_mask, n_final))
        # with kernel_size < 2 the reference's extended_masks IS masks, so its in-place in-bound assignment
        # (src/multiview_filter.py:146) also rewrites masks and the count it prints is the final one
        shown = n_final if self._kernel_code() == 1 else n_mask
        prefix = "Bound: ["
        prefix += f'[{bd[0][0]:.1f}, {bd[0][1]:.1f}], '
        prefix += f'[{bd[1][0]:.1f}, {bd[1][1]:.1f}], '
        prefix += f'[{bd[2][0]:.1f}, {bd[2][1]:.1f}]]!'
        print(_CYAN)
        print(f'\n\n Multiview filtering: previous at {filtered_t}, now at {cur_t}, {shown} valid points '
              f'found! {prefix}\n')
        print(_RESET)
