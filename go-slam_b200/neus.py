"""InstantNeuS with the reference's constructor / forward signature (src/InstantNeuS.py:219-370),
backed by the fused sm_90a ray marcher (goslam_neus_forward) instead of tiny-cuda-nn + ~60
eager torch kernels.

    net = InstantNeuS(cfg, bound, device)               # cfg = cfg['mapping']['model']
    out = net(rays_o, rays_d, z_vals, dists, render_params=None)   # dict with the 9 reference keys

Parameters keep the reference's names so `state_dict()` round-trips through the same keys the
reference checkpoint (go.ckpt 'mapping_net') holds:
    sdf_network.encoding.encoding.params   tcnn HashGrid params (fp32 master, 16 lvl x 2 feat)
    sdf_network.encoding._B                (unused by the non-directional encoding, kept)
    sdf_network.sdf_layer.{weight,bias}    nn.Linear(35, 32)
    color_network._B                       [3, 33]
    color_network.network.params           tcnn FullyFusedMLP params (fp32 master) 64x80|64x64|16x64
    variance_network.variance
Under `torch.no_grad()` the forward pass is the inference path.  With grad enabled (what
Mapper.optimize_map does, src/mapping.py:89-91) the same fused kernel keeps its per-sample intermediates and the
returned tensors carry a grad_fn: `loss.backward()` runs goslam_neus_composite_backward, goslam_neus_mlp_backward, the
weight-gradient GEMMs (cuBLAS) and goslam_neus_grid_backward, and fills `.grad` of the hash grid, sdf_layer, colour `_B`, colour
network and variance parameters (SURVEY 8f-3).  Differentiable outputs: color, depth, sdf, gradient_error; the other
keys are returned detached (the reference's losses use depth_variance detached and never read normal / weight_sum).
When rays_o or rays_d requires grad (camera refinement: rays built from a pose leaf), the backward also runs
goslam_neus_ray_backward and returns dL/d rays_o, dL/d rays_d in the rays' dtype; the parameter gradients are the same.
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import _lib
from .mesher import keep_box

N_LEVELS, N_FEAT = 16, 2
MLP_IN, MLP_IN_PAD, MLP_HID, MLP_OUT_PAD = 67, 80, 64, 16
MLP_PARAMS = MLP_HID * MLP_IN_PAD + MLP_HID * MLP_HID + MLP_OUT_PAD * MLP_HID


def hashgrid_layout():
    """(offsets[17] in params, resolutions[16], scales[16], total_params) from the C-ABI helper."""
    lib = _lib.load()
    off = (ctypes.c_int64 * (N_LEVELS + 1))()
    res = (ctypes.c_int * N_LEVELS)()
    sc = (ctypes.c_float * N_LEVELS)()
    total = lib.goslam_hashgrid_layout(off, res, sc)
    return list(off), list(res), list(sc), int(total)


class _TcnnParams(nn.Module):
    """stands in for a tcnn module: a flat fp32 `params` tensor (tcnn keeps fp32 masters and
    uses fp16 copies on the device, which is what we hand to the kernel)."""

    def __init__(self, n, init):
        super().__init__()
        self.params = nn.Parameter(init(n))
        self.n_output_dims = None


class Encoding(nn.Module):
    def __init__(self, n_input_dims=3, device='cuda:0', direction=False):
        super().__init__()
        if direction:
            raise NotImplementedError("directional (SH) encoding is unused by the reference model")
        self.n_input_dims = n_input_dims
        self.include_xyz = True
        _, _, _, total = hashgrid_layout()
        # tcnn initialises grid params U(-1e-4, 1e-4)
        self.encoding = _TcnnParams(total, lambda n: (torch.rand(n) * 2 - 1) * 1e-4)
        self.encoding.n_output_dims = N_LEVELS * N_FEAT
        self._B = nn.Parameter(torch.randn(n_input_dims, 3) * 25.0)
        self.n_output_dims = 3 + N_LEVELS * N_FEAT


class SDFNetwork(nn.Module):
    def __init__(self, d_in=3, d_out=32, device='cuda:0'):
        super().__init__()
        if d_out != 32:
            raise ValueError("fused marcher is specialised for d_out = 32 (reference default)")
        self.d_in, self.d_out = d_in, d_out
        self.encoding = Encoding(n_input_dims=d_in, device=device)
        self.sdf_layer = nn.Linear(self.encoding.n_output_dims, d_out)
        torch.nn.init.constant_(self.sdf_layer.bias, 0.0)
        torch.nn.init.constant_(self.sdf_layer.weight[:, 3:], 0.0)
        torch.nn.init.normal_(self.sdf_layer.weight[:, :3], mean=0.0, std=math.sqrt(2) / math.sqrt(d_out))

    def get_training_parameters(self, ignore_keys=()):
        return {'network': list(self.sdf_layer.parameters()) + [self.encoding._B],
                'volume': list(self.encoding.encoding.parameters())}


class ColorNetwork(nn.Module):
    def __init__(self, d_in=3, d_feat=31, d_hidden=64, n_layers=2, device='cuda:0'):
        super().__init__()
        if (d_feat, d_hidden, n_layers) != (31, 64, 2):
            raise ValueError("fused marcher is specialised for d_feat=31, d_hidden=64, n_layers=2")
        self._B = nn.Parameter(torch.randn(3, 33) * 25.0)
        # tcnn default init: xavier-uniform per matrix
        def init(n):
            mats = []
            for fo, fi in ((MLP_HID, MLP_IN_PAD), (MLP_HID, MLP_HID), (MLP_OUT_PAD, MLP_HID)):
                lim = math.sqrt(6.0 / (fi + fo))
                mats.append(((torch.rand(fo * fi) * 2 - 1) * lim))
            return torch.cat(mats)
        self.network = _TcnnParams(MLP_PARAMS, init)


class SingleVarianceNetwork(nn.Module):
    def __init__(self, init_val=0.2, scale_factor=10.0):
        super().__init__()
        self.scale_factor = scale_factor
        self.register_parameter('variance', nn.Parameter(torch.tensor(init_val)))

    def forward(self, x):
        return torch.ones(size=[x.shape[0], 1], device=x.device) * torch.exp(self.variance * self.scale_factor)


class InstantNeuS(nn.Module):
    def __init__(self, cfg, bound, device='cuda:0'):
        super().__init__()
        self.cfg = cfg
        self.register_buffer('bound', torch.tensor(bound).float())
        self.register_buffer('realtime_bound', torch.tensor(bound).float())
        self.device = device
        self.sdf_network = SDFNetwork(**cfg['sdf_network'], device=device)
        self.color_network = ColorNetwork(**cfg['color_network'], device=device)
        self.variance_network = SingleVarianceNetwork(**cfg['variance_network'])
        self.sdf_smooth_std = cfg.get('sdf_smooth_std')
        self.sdf_sparse_factor = cfg.get('sdf_sparse_factor')
        self.sdf_truncation = cfg.get('sdf_truncation')
        self.sdf_random_weight = cfg.get('sdf_random_weight')
        self.cos_anneal_ratio = 1.0
        self._half_cache = None

    # ---- reference helper API -------------------------------------------------------------
    def get_training_parameters(self, ignore_keys=()):
        all_params = {
            'sdf_network': list(self.sdf_network.get_training_parameters()['network']),
            'color_network': list(self.color_network.parameters()),
            'variance_network': list(self.variance_network.parameters()),
        }
        params = []
        for k, v in all_params.items():
            if k not in ignore_keys:
                params += v
        return params

    def get_volume_parameters(self):
        return list(self.sdf_network.get_training_parameters()['volume'])

    @torch.no_grad()
    def update_bound(self, bound):
        self.realtime_bound[:] = bound.float().to(self.realtime_bound.device)

    def compute_sdf_error(self, sdf, z_vals, gt_depth):
        """the SDF supervision of the mapping step (src/InstantNeuS.py:372-400): returns (sdf_error, front_error).
        Samples within +-truncation of the sensor depth are pulled to `depth - z`; samples in front of that band pay
        max(exp(-sparse_factor * sdf) - 1, sdf - (depth - z)) clamped at 0; both averaged per ray over the ray's
        supervised samples, then over the valid rays.  Plain elementwise torch on [n_rays, n_samples] (autograd
        hands d_sdf to the renderer backward)."""
        n_rays = z_vals.shape[0]
        pred = sdf.reshape(n_rays, -1)
        depth = gt_depth.reshape(n_rays, 1)
        ok = (depth > 0).reshape(-1)
        depth, z, pred = depth[ok], z_vals[ok], pred[ok]
        to_surface = depth - z
        in_front = z < (depth - self.sdf_truncation)
        in_band = to_surface.abs() <= self.sdf_truncation
        per_ray = in_front.sum(dim=1) + in_band.sum(dim=1) + 1e-8
        n_ok = ok.sum()
        sparse = torch.exp((-self.sdf_sparse_factor * pred).clamp(max=10.0)) - 1.0
        front = torch.maximum(sparse, pred - to_surface).clamp(min=0.0) * in_front
        front_error = (front.sum(dim=1) / per_ray).sum() / n_ok
        band_error = (((pred - to_surface).abs() * in_band).sum(dim=1) / per_ray).sum() / n_ok
        return band_error, front_error

    # ---- kernel-side parameter staging ------------------------------------------------------
    def refresh_device_params(self):
        """fp16 copies of the tcnn-style params (call after loading / changing weights)."""
        g = self.sdf_network.encoding.encoding.params
        m = self.color_network.network.params
        self._half_cache = (g.detach().half().contiguous(), m.detach().half().contiguous(),
                            g._version, m._version)

    def _params_struct(self):
        g = self.sdf_network.encoding.encoding.params
        m = self.color_network.network.params
        if (self._half_cache is None or self._half_cache[2] != g._version
                or self._half_cache[3] != m._version or self._half_cache[0].device != g.device):
            self.refresh_device_params()
        grid_h, mlp_h = self._half_cache[0], self._half_cache[1]
        p = _lib.NeusParams()
        keep = [grid_h, mlp_h,
                self.sdf_network.sdf_layer.weight.detach().float().contiguous(),
                self.sdf_network.sdf_layer.bias.detach().float().contiguous(),
                self.color_network._B.detach().float().contiguous()]
        p.grid = grid_h.data_ptr()
        p.mlp_w = mlp_h.data_ptr()
        p.sdf_w = keep[2].data_ptr()
        p.sdf_b = keep[3].data_ptr()
        p.color_B = keep[4].data_ptr()
        key = (self.bound._version, self.realtime_bound._version,
               self.variance_network.variance._version)
        if getattr(self, '_host_cache', None) is None or self._host_cache[0] != key:
            # one D2H sync per parameter change, not per call
            b = self.bound.detach().float().cpu().reshape(-1).tolist()
            rb = self.realtime_bound.detach().float().cpu().reshape(-1).tolist()
            inv_s = float(torch.exp(self.variance_network.variance.detach().float().cpu()
                                    * self.variance_network.scale_factor).clip(1e-6, 1e6))
            self._host_cache = (key, b, rb, inv_s)
        _, b, rb, inv_s = self._host_cache
        for i in range(6):
            p.bound[i] = b[i]
            p.rt_bound[i] = rb[i]
        p.inv_s = inv_s
        p.cos_anneal_ratio = float(self.cos_anneal_ratio)
        return p, keep, inv_s

    # ---- forward ------------------------------------------------------------------------------
    def trainable_tensors(self):
        """the parameters the renderer backward produces gradients for, in the order _NeusFunction takes them"""
        return (self.sdf_network.encoding.encoding.params, self.color_network.network.params,
                self.sdf_network.sdf_layer.weight, self.sdf_network.sdf_layer.bias, self.color_network._B,
                self.variance_network.variance)

    def forward(self, rays_o, rays_d, z_vals, dists, render_params: dict = None, debug=False):
        """debug=True (tests only): additionally keeps the per-sample NeuS alpha [R,S] and SDF normal [R,S,3]
        in `self.last_debug`.  With grad enabled and any trainable parameter, rays_o or rays_d requiring grad:
        differentiable, also w.r.t. the rays (camera refinement, src/mapping.py:173-194).  z_vals and dists are sampled
        from detached rays and carry no gradient."""
        params = self.trainable_tensors()
        if torch.is_grad_enabled() and not debug and any(t.requires_grad for t in params + (rays_o, rays_d)):
            if z_vals.requires_grad or dists.requires_grad:
                raise RuntimeError("InstantNeuS.forward: gradients w.r.t. z_vals / dists are not implemented "
                                   "(the renderer samples them from detached rays)")
            vals = _NeusFunction.apply(self, rays_o, rays_d, z_vals, dists, *params)
            return dict(zip(_NeusFunction.KEYS, vals))
        return self._forward_impl(rays_o, rays_d, z_vals, dists, debug=debug)

    @torch.no_grad()
    def _forward_impl(self, rays_o, rays_d, z_vals, dists, debug=False, train=False):
        """the fused marcher; train=True keeps what the backward needs in `self.last_debug`"""
        _lib.need_cuda("InstantNeuS.forward", z_vals)
        dev = z_vals.device
        R, S = z_vals.shape
        rays_o = rays_o.detach().float().contiguous()
        rays_d = rays_d.detach().float().contiguous()
        z_vals = z_vals.detach().float().contiguous()
        dists = dists.detach().float().contiguous()
        p, keep, inv_s = self._params_struct()
        f32 = dict(dtype=torch.float32, device=dev)
        out = {
            'color': torch.empty((R, 3), **f32), 'depth': torch.empty((R, 1), **f32),
            'depth_variance': torch.empty((R, 1), **f32), 'normal': torch.empty((R, 3), **f32),
            'weight_sum': torch.empty((R, 1), **f32), 'sdf': torch.empty((R, S), **f32),
            'z_vals': torch.empty((R, S), **f32), 'gradient_error': torch.zeros((1,), **f32),
        }
        o = _lib.NeusOut()
        o.color = out['color'].data_ptr(); o.depth = out['depth'].data_ptr()
        o.depth_variance = out['depth_variance'].data_ptr(); o.normal = out['normal'].data_ptr()
        o.weight_sum = out['weight_sum'].data_ptr(); o.sdf = out['sdf'].data_ptr()
        o.z_mid = out['z_vals'].data_ptr(); o.gradient_error = out['gradient_error'].data_ptr()
        self.last_debug = None
        if debug or train:
            self.last_debug = {'alpha': torch.empty((R, S), **f32), 'grad': torch.empty((R, S, 3), **f32)}
            o.alpha = self.last_debug['alpha'].data_ptr()
            o.grad = self.last_debug['grad'].data_ptr()
            self.last_debug['pos'] = torch.empty((R, S, 3), **f32)
            o.pos = self.last_debug['pos'].data_ptr()
        if train:
            f16 = dict(dtype=torch.float16, device=dev)
            self.last_debug.update(rgb=torch.empty((R, S, 3), **f32), mlp_in=torch.empty((R, S, MLP_IN_PAD), **f16),
                                   enc=torch.empty((R, S, N_LEVELS * N_FEAT), **f16),
                                   fallback=torch.empty((1,), dtype=torch.int32, device=dev))
            o.rgb = self.last_debug['rgb'].data_ptr()
            o.mlp_in = self.last_debug['mlp_in'].data_ptr()
            o.enc = self.last_debug['enc'].data_ptr()
            o.fallback = self.last_debug['fallback'].data_ptr()
        ws = _lib.workspace(_lib.load().goslam_neus_workspace_bytes(R, S), dev)
        _lib.call("neus_forward", ctypes.byref(p), rays_o, rays_d, z_vals, dists, R, S, ctypes.byref(o), ws, ws.numel())
        out['sdf_variance'] = torch.full((R, 1), 1.0 / inv_s, **f32)
        return out

    # ---- mesh extraction (src/InstantNeuS.py:258-274, 402-492) ------------------------------------------------
    @torch.no_grad()
    def in_bound(self, pts, bound):
        """strict per-axis test of pts [n,3] against bound [3,2] (src/InstantNeuS.py:258-274)"""
        bound = bound.to(pts.device)
        mask_x = (pts[:, 0] < bound[0, 1]) & (pts[:, 0] > bound[0, 0])
        mask_y = (pts[:, 1] < bound[1, 1]) & (pts[:, 1] > bound[1, 0])
        mask_z = (pts[:, 2] < bound[2, 1]) & (pts[:, 2] > bound[2, 0])
        return (mask_x & mask_y & mask_z).bool()

    def _device(self):
        dev = self.bound.device
        if dev.type != 'cuda':
            raise RuntimeError("InstantNeuS mesh extraction: the network must be on a CUDA device (no CPU fallback)")
        return dev

    def _sdf_grid(self, bound_min, bound_max, resolution):
        """u [res]^3 f32 on the device for the lattice torch.linspace(bound_min[a], bound_max[a], res) (computed on the
        CPU, as the reference does), normalised by [bound_min, bound_max], masked by realtime_bound"""
        dev = self._device()
        res = int(resolution)
        if res < 1:
            raise ValueError("resolution must be positive")
        tabs = torch.cat([torch.linspace(float(bound_min[a]), float(bound_max[a]), res) for a in range(3)])
        tabs = tabs.pin_memory().to(dev, non_blocking=True)
        p, keep, _ = self._params_struct()
        for a in range(3):
            p.bound[2 * a], p.bound[2 * a + 1] = float(bound_min[a]), float(bound_max[a])
        u = torch.empty((res, res, res), dtype=torch.float32, device=dev)
        _lib.call("neus_sdf_grid", ctypes.byref(p), tabs[:res], tabs[res:2 * res], tabs[2 * res:], res, res, res, u)
        return u

    @torch.no_grad()
    def extract_fields(self, bound_min, bound_max, resolution: int):
        """numpy f32 [res]^3: -sdf on the lattice, -100 outside realtime_bound (src/InstantNeuS.py:423-455); one launch and
        one device-to-host copy"""
        bmin = torch.as_tensor(bound_min).detach().float().cpu().tolist()
        bmax = torch.as_tensor(bound_max).detach().float().cpu().tolist()
        return self._sdf_grid(bmin, bmax, resolution).cpu().numpy()

    def _vertex_colors(self, verts, bound):
        """uint8 [V,3] colours of f64 device vertices, the network normalised by `bound` (6 floats, x-major)"""
        dev = verts.device
        p, keep, _ = self._params_struct()
        for i in range(6):
            p.bound[i] = bound[i]
        rgb = torch.empty((verts.shape[0], 3), dtype=torch.uint8, device=dev)
        _lib.call("neus_vertex_color", ctypes.byref(p), verts, verts.shape[0], rgb)
        return rgb

    @torch.no_grad()
    def extract_color(self, bound, vertices):
        """numpy uint8 [V,3] vertex colours of numpy vertices (src/InstantNeuS.py:402-420)"""
        dev = self._device()
        b = torch.as_tensor(bound).detach().float().cpu().reshape(-1).tolist()
        verts = torch.as_tensor(vertices, dtype=torch.float64).reshape(-1, 3).to(dev).contiguous()
        return self._vertex_colors(verts, b).cpu().numpy()

    @torch.no_grad()
    def extract_mesh(self, resolution, threshold, c2w_ref=None, color=True):
        """extract_geometry on the device: (vertices [V,3] f64, faces [F,3] i64, colours [V,3] u8 or None), CUDA tensors.
        Field -> marching cubes -> world scaling -> c2w_ref -> bound cull -> colours of the kept vertices.  Two host
        synchronisations: the two count reads (and one on the first call after the bounds change)."""
        import numpy as np
        dev = self._device()
        res = int(resolution)
        self._params_struct()                                # refreshes the host copies of the bounds
        b, rb = self._host_cache[1], self._host_cache[2]
        bmin, bmax = [b[0], b[2], b[4]], [b[1], b[3], b[5]]
        u = self._sdf_grid(bmin, bmax, res)
        verts, faces = marching_cubes(u, threshold, bmin, bmax)
        del u
        if c2w_ref is not None:
            # np.matmul(c2w_ref[None], [v, 1][:, :, None])[:, :3, 0] in float64
            c = torch.as_tensor(c2w_ref).detach().to(dev, torch.float64)
            verts = ((verts[:, 0:1] * c[:3, 0] + verts[:, 1:2] * c[:3, 1]) + verts[:, 2:3] * c[:3, 2]) + c[:3, 3]
        # bound cull: thresholds in float32, as numpy computes `bound[:, 0] - eps` on the float32 array
        rt = np.array(rb, np.float32).reshape(3, 2)
        eps = 0.01
        out_v, out_f = cull_mesh(verts, faces, (rt[:, 0] - eps).tolist(), (rt[:, 1] + eps).tolist())
        del verts, faces
        rgb = self._vertex_colors(out_v, b) if color else None
        return out_v, out_f, rgb

    @torch.no_grad()
    def extract_geometry(self, resolution: int, threshold: float, c2w_ref=None, save_path='./mesh.ply', color=False):
        """the reference's extract_geometry (src/InstantNeuS.py:458-497): a trimesh.Trimesh of the culled mesh, exported to
        save_path unless it is None.  Runs extract_mesh; the arrays come back in one device-to-host copy."""
        import trimesh          # the reference imports it at module level
        verts, faces, rgb = self.extract_mesh(resolution, threshold, c2w_ref=c2w_ref, color=color)
        host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in (verts, faces, rgb) if t is not None]
        for h, t in zip(host, (verts, faces, rgb)):
            h.copy_(t, non_blocking=True)
        torch.cuda.current_stream(verts.device).synchronize()
        vertex_colors = host[2].numpy() if color else None
        mesh = trimesh.Trimesh(host[0].numpy(), host[1].numpy(), vertex_colors=vertex_colors)
        if save_path is not None:
            mesh.export(save_path)
        return mesh


def marching_cubes(u, iso, bound_min, bound_max):
    """marching cubes of the f32 CUDA field u [nx,ny,nz] at level iso (inside iff u > iso), on the generated tables of
    csrc/mc_tables.cuh: (vertices [V,3] f64 in world coordinates v / (n - 1.0) * (float32)(bound_max - bound_min) +
    bound_min, faces [F,3] i64), CUDA tensors.  Reads the two counts back (one host synchronisation)."""
    u = u.detach().float().contiguous()
    nx, ny, nz = u.shape
    dev = u.device
    i64 = dict(dtype=torch.int64, device=dev)
    ws = torch.empty(_lib.load().goslam_mc_workspace_bytes(nx, ny, nz), dtype=torch.uint8, device=dev)
    counts = torch.empty(2, **i64)
    _lib.call("mc_count", u, nx, ny, nz, float(iso), ws, ws.numel(), counts)
    nv, nf = counts.tolist()
    verts = torch.empty((nv, 3), dtype=torch.float64, device=dev)
    faces = torch.empty((nf, 3), **i64)
    lo = (ctypes.c_float * 3)(*[float(v) for v in bound_min])
    hi = (ctypes.c_float * 3)(*[float(v) for v in bound_max])
    _lib.call("mc_emit", u, nx, ny, nz, float(iso), lo, hi, ws, ws.numel(), verts, nv, faces, nf)
    return verts, faces


def cull_mesh(verts, faces, lo, hi):
    """keep the vertices with lo <= v <= hi (lo, hi: 3 float32 values each), the faces whose three vertices are kept,
    then drop unreferenced vertices; stable orders, faces re-indexed (update_faces + remove_unreferenced_vertices).
    CUDA tensors in and out; reads the two counts back (one host synchronisation)."""
    out_v, out_f, _ = keep_box(verts, faces, lo, hi)
    return out_v, out_f


class _NeusFunction(torch.autograd.Function):
    """InstantNeuS.forward as one autograd node (what autograd + tiny-cuda-nn do for the reference,
    src/InstantNeuS.py:295-370 under torch.enable_grad() in src/mapping.py:89-91).
    forward : the fused marcher with its per-sample intermediates kept.
    backward: goslam_neus_composite_backward -> goslam_neus_mlp_backward (row-wise colour-network backward on mma.sync)
              -> weight-gradient GEMMs over the sample dimension (cuBLAS, fp16 in / fp32 out, loss scale)
              -> goslam_neus_grid_backward (hash-grid scatter + the second-order path through the analytic normal)
              -> goslam_neus_ray_backward when rays_o or rays_d needs a gradient (composite_backward_ex then also keeps
              dL/d true_cos).  Chunked over rays to bound the activations."""
    CHUNK_RAYS = 1 << 16
    MAX_SAMPLES = 128            # goslam_neus_composite_backward keeps up to 4 chunks of 32 samples of a ray in registers
    KEYS = ('color', 'depth', 'sdf', 'gradient_error', 'depth_variance', 'normal', 'weight_sum', 'z_vals', 'sdf_variance')

    @staticmethod
    def forward(ctx, net, rays_o, rays_d, z_vals, dists, grid, mlp, sdf_w, sdf_b, color_B, variance):
        if z_vals.shape[1] > _NeusFunction.MAX_SAMPLES:
            raise RuntimeError("InstantNeuS.forward under grad: the renderer backward supports at most %d samples per ray, "
                               "got %d (the forward alone, under torch.no_grad(), takes up to 288)"
                               % (_NeusFunction.MAX_SAMPLES, z_vals.shape[1]))
        ctx.set_materialize_grads(False)
        ctx.ray_dtypes = (rays_o.dtype, rays_d.dtype)
        rays_o, rays_d = rays_o.detach().float().contiguous(), rays_d.detach().float().contiguous()
        z_vals, dists = z_vals.detach().float().contiguous(), dists.detach().float().contiguous()
        out = net._forward_impl(rays_o, rays_d, z_vals, dists, train=True)
        saved = net.last_debug
        net.last_debug = None
        ctx.net = net
        ctx.pstruct = net._params_struct()          # (struct, tensors it points to, inv_s) at forward time
        ctx.save_for_backward(rays_o, rays_d, z_vals, dists, saved['alpha'], saved['grad'], saved['rgb'], saved['mlp_in'],
                              saved['enc'], saved['pos'], out['sdf'], out['z_vals'], sdf_w.detach(), color_B.detach(),
                              mlp.detach(), saved['fallback'])
        vals = tuple(out[k] for k in _NeusFunction.KEYS)
        ctx.mark_non_differentiable(*vals[4:])
        return vals

    @staticmethod
    def backward(ctx, d_color, d_depth, d_sdf, d_gerr, *_non_differentiable):
        (rays_o, rays_d, z_vals, dists, alpha, grad, rgb, mlp_in, enc, pos, sdf, z_mid, sdf_w, color_B, mlp,
         fallback) = ctx.saved_tensors
        net = ctx.net
        p, keep, inv_s = ctx.pstruct
        dev = z_vals.device
        R, S = z_vals.shape
        f32 = dict(dtype=torch.float32, device=dev)
        c = lambda t: None if t is None else t.detach().float().contiguous()
        d_color, d_depth, d_sdf = c(d_color), c(d_depth), c(d_sdf)
        d_gerr = c(d_gerr)
        # The colour network backward is plain GEMMs (cuBLAS).  Like tcnn it runs in fp16 on the tensor cores with a loss
        # scale: the upstream gradients are multiplied by a power of two that brings their largest entry to ~1024 before
        # the cast to half (mean-reduced losses give ~1e-6 entries, fp16's smallest normal is 6e-5), weight gradients
        # accumulate in fp32 (mm out_dtype) and are divided by the scale at the end.  No host synchronisation.
        f16 = dict(dtype=torch.float16, device=dev)
        Wsdf_enc = sdf_w.float()[:, 3:].half().contiguous()                      # [32, 32]
        g_grid = torch.zeros(net.sdf_network.encoding.encoding.params.numel(), **f32)
        g_W1 = torch.zeros(MLP_HID, MLP_IN_PAD, **f32)
        g_W2 = torch.zeros(MLP_HID, MLP_HID, **f32)
        g_W3 = torch.zeros(MLP_OUT_PAD, MLP_HID, **f32)
        g_sdf_w, g_sdf_b = torch.zeros(32, 35, **f32), torch.zeros(32, **f32)
        g_B = torch.zeros(3, 33, **f32)
        g_w0 = torch.zeros(35, **f32)
        g_inv_s = torch.zeros(1, **f32)
        ray_grad = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        if ray_grad:
            g_ro, g_rd = torch.empty(R, 3, **f32), torch.empty(R, 3, **f32)
            Wsdf_xyz = sdf_w.float()[:, :3].contiguous()                         # [32, 3]
        for r0 in range(0, R, _NeusFunction.CHUNK_RAYS):
            r1 = min(R, r0 + _NeusFunction.CHUNK_RAYS)
            n = (r1 - r0) * S
            sl = slice(r0, r1)
            ro, rd, zv, ds = rays_o[sl], rays_d[sl], z_vals[sl], dists[sl]
            d_y = torch.empty(n, 3, **f32); d_s = torch.empty(n, **f32); d_g = torch.empty(n, 3, **f32)
            dc = None if d_color is None else d_color[sl].contiguous()
            dd = None if d_depth is None else d_depth[sl].contiguous()
            dsu = None if d_sdf is None else d_sdf[sl].contiguous()
            if ray_grad:
                d_tc = torch.empty(n, **f32)
                _lib.call("neus_composite_backward_ex", ctypes.byref(p), ro, rd, ds, alpha[sl], rgb[sl], sdf[sl], grad[sl],
                          z_mid[sl], dc, dd, dsu, d_gerr, fallback, R * S, r0 * S, r1 - r0, S, d_y, d_s, d_g, g_inv_s, d_tc)
            else:
                _lib.call("neus_composite_backward", ctypes.byref(p), ro, rd, ds, alpha[sl], rgb[sl], sdf[sl], grad[sl],
                          z_mid[sl], dc, dd, dsu, d_gerr, fallback, R * S, r0 * S, r1 - r0, S, d_y, d_s, d_g, g_inv_s)
            amax = torch.maximum(d_y.abs().max(), d_s.abs().max()).clamp_min(1e-30)
            sc = torch.exp2(torch.floor(torch.log2(1024.0 / amax))).clamp(max=2.0 ** 40).reshape(1).contiguous()   # device scalar
            # ---- colour network, row-wise half (one kernel): H1, H2, dH2, dH1, dX and what hangs off dX per sample ----
            X = mlp_in[sl].reshape(n, MLP_IN_PAD)                                 # half, as the forward built it
            H1, H2, dH1, dH2 = (torch.empty(n, MLP_HID, **f16) for _ in range(4))
            dY8, pts_hl = torch.empty(n, 8, **f16), torch.empty(n, 8, **f16)
            dE, h = torch.empty(n, 40, **f16), torch.empty(n, 40, **f16)
            d_out = torch.empty(n, 32, **f16)
            d_gt = torch.empty(n, 3, **f32)
            mo = _lib.NeusMlpBwdOut()
            mo.H1, mo.H2, mo.dH1, mo.dH2 = H1.data_ptr(), H2.data_ptr(), dH1.data_ptr(), dH2.data_ptr()
            mo.dY8, mo.dE, mo.d_out, mo.h = dY8.data_ptr(), dE.data_ptr(), d_out.data_ptr(), h.data_ptr()
            mo.pts_hl, mo.d_grad_total = pts_hl.data_ptr(), d_gt.data_ptr()
            _lib.call("neus_mlp_backward", ctypes.byref(p), X, enc[sl], pos[sl], d_y, d_s, d_g, ro, rd, z_mid[sl], sc,
                      r1 - r0, S, ctypes.byref(mo))
            # ---- weight gradients: GEMMs over the sample dimension (cuBLAS, fp16 in, fp32 out) ----
            g_W3[:8] += torch.mm(dY8.t(), H2, out_dtype=torch.float32) / sc
            g_W2 += torch.mm(dH2.t(), H1, out_dtype=torch.float32) / sc
            g_W1 += torch.mm(dH1.t(), X, out_dtype=torch.float32) / sc
            gb = torch.mm(pts_hl.t(), dE, out_dtype=torch.float32)                 # colour embedding sin(pts @ B)
            g_B += (gb[:3, :33] + gb[3:6, :33]) / sc
            gs = torch.mm(d_out.t(), h, out_dtype=torch.float32) / sc               # sdf_layer: out = W h + b
            g_sdf_w += gs[:, :35]
            g_sdf_b += gs[:, 35]
            d_enc = torch.mm(d_out, Wsdf_enc, out_dtype=torch.float32)             # [n, 32] f32, still scaled
            _lib.call("neus_grid_backward", ctypes.byref(p), ro, rd, zv, ds, fallback, r0 * S, r1 - r0, S, d_enc, sc,
                      d_gt, g_grid, g_w0)
            if ray_grad:
                d_xyz = torch.mm(d_out.float(), Wsdf_xyz)                         # [n, 3] f32, still scaled
                _lib.call("neus_ray_backward", ctypes.byref(p), ro, rd, zv, ds, fallback, r0 * S, r1 - r0, S, d_enc, d_xyz,
                          dE, sc, d_gt, d_tc, g_ro[sl], g_rd[sl])
        g_sdf_w[0] += g_w0
        # samples the forward kept out of the network (outside the real-time bound and not among the first 100 of a
        # nothing-in-bound call): rgb = 0, alpha = 0, the kernels return zeros for them, so the GEMMs above see zero rows.
        sf = net.variance_network.scale_factor
        raw = float(torch.exp(net.variance_network.variance.detach().float() * sf))
        g_var = (g_inv_s[0] * inv_s * sf) if 1e-6 <= raw <= 1e6 else torch.zeros((), **f32)
        g_mlp = torch.cat([g_W1.reshape(-1), g_W2.reshape(-1), g_W3.reshape(-1)])
        g_ro = g_ro.to(ctx.ray_dtypes[0]) if ctx.needs_input_grad[1] else None
        g_rd = g_rd.to(ctx.ray_dtypes[1]) if ctx.needs_input_grad[2] else None
        return (None, g_ro, g_rd, None, None, g_grid, g_mlp, g_sdf_w, g_sdf_b, g_B, g_var.reshape(()))
