"""Renderer with the reference's call signature (src/render.py:6-175): near/far from the scene
AABB, stratified + surface-guided z sampling, then ONE call of the fused marcher for the whole
ray batch (the reference splits into 10,000-ray chunks of ~60 eager kernels each, :53-59).

The z-sampling is ONE kernel launch (goslam_sample_z, csrc/zsample.cu; the reference issues ~25
eager [R,S] kernels and a torch.sort).  The two linspace tables and the shared
`perturb_rand[N_samples]` (src/render.py:159) still come from torch, so the RNG stream advances
exactly as in the reference and z_vals are bit-identical to it for the same RNG state.
"""
import torch

from . import _lib
from .mapping import all_rays

_tables = {}


def _linspace_tables(n_samples, n_surface, device):
    key = (n_samples, n_surface, str(device))
    if key not in _tables:
        tv = torch.linspace(0, 1, steps=n_samples, device=device)                       # src/render.py:143
        ts = torch.linspace(0, 1, steps=n_surface).float().to(device) if n_surface > 0 else None   # :134
        _tables[key] = (tv, ts)
    return _tables[key]


def sample_z(rays_o, rays_d, bound, gt_depth, n_samples, n_surface, perturb=1.0, lindisp=False):
    """Returns z_vals [R, S], dists [R, S] with S = n_samples (+ n_surface when gt_depth is given)."""
    device = rays_o.device
    _lib.need_cuda("sample_z", rays_o)
    R = int(rays_o.shape[0])
    if gt_depth is None:
        n_surface = 0
    S = n_samples + n_surface
    tv, ts = _linspace_tables(n_samples, n_surface, device)
    rand = torch.rand(n_samples, device=device) if perturb > 0 else None                # src/render.py:159
    ro = rays_o.detach().float().contiguous()
    rd = rays_d.detach().float().contiguous()
    bd = bound.to(device=device, dtype=torch.float32).contiguous()
    gd = gt_depth.reshape(-1).float().contiguous() if gt_depth is not None else None
    z_vals = torch.empty((R, S), dtype=torch.float32, device=device)
    dists = torch.empty((R, S), dtype=torch.float32, device=device)
    ws = _lib.workspace(256, device)
    _lib.call("sample_z", ro, rd, bd, gd, tv, ts, rand, R, n_samples, n_surface, int(bool(lindisp)), z_vals, dists, ws,
              ws.numel())
    return z_vals, dists


class Renderer(object):
    def __init__(self, cfg, args, slam, points_batch_size=1e4, ray_batch_size=5e3):
        self.ray_batch_size = int(ray_batch_size)
        self.points_batch_size = int(points_batch_size)     # kept for API parity; not needed
        r = cfg['rendering']
        self.lindisp, self.perturb = r['lindisp'], r['perturb']
        self.N_samples, self.N_surface = r['N_samples'], r['N_surface']
        self.H, self.W, self.fx, self.fy, self.cx, self.cy = slam.H, slam.W, slam.fx, slam.fy, slam.cx, slam.cy

    def eval_points(self, rays_o, rays_d, z_vals, dists, net, render_params):
        return net(rays_o, rays_d, z_vals, dists, render_params=render_params)

    def render_batch_ray(self, rays_o, rays_d, net, render_params, device='cuda:0', gt_depth=None):
        z_vals, dists = sample_z(rays_o, rays_d, net.bound, gt_depth, self.N_samples, self.N_surface,
                                 self.perturb, self.lindisp)
        return self.eval_points(rays_o, rays_d, z_vals, dists, net, render_params)

    def render_img(self, net, c2w, device, gt_depth=None):
        """the reference's render_img (src/render.py:177-237): the whole image's rays in one launch
        (goslam_mapping_all_rays), then one sample_z + forward per ray_batch_size chunk.  The chunking is kept
        because it shows in the result: the far clamp uses each chunk's own gt_depth.max(), each chunk draws its own
        perturb_rand, the forward's mask fix-up is per chunk, and gradient_error comes out as [n_chunks].
        c2w: [4,4] tensor or ndarray."""
        with torch.no_grad():
            H, W = self.H, self.W
            if not torch.is_tensor(c2w):
                c2w = torch.from_numpy(c2w)
            rays_o, rays_d = all_rays(H, W, (self.fx, self.fy, self.cx, self.cy), c2w.to(device))
            render_params = {
                'global_step': -1,
                'gt_depth': None,
                'stratified': False,
                'update_state': False,
                'compute_sdf_smooth_error': False,
            }
            render_out = {}
            step = self.ray_batch_size
            gt_depth = gt_depth.reshape(-1)        # the reference requires gt_depth here too
            for i in range(0, H * W, step):
                out = self.render_batch_ray(rays_o=rays_o[i:i + step], rays_d=rays_d[i:i + step], net=net,
                                            render_params=render_params, device=device,
                                            gt_depth=gt_depth[i:i + step])
                if len(render_out) == 0:
                    render_out = out
                    continue
                for k, v in out.items():
                    if torch.is_tensor(v):
                        render_out[k] = torch.cat([render_out[k], v], dim=0)
                    else:
                        assert v is None, type(v)
                        render_out[k] = v
            return render_out
