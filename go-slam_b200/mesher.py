"""Mesher.cull_mesh (src/mesher.py:156-240) on the device: the depth maps of extract_depth_from_mesh (pyrender / OpenGL in the
reference), the seen / forecast vertex masks of point_masks, the connected-component filter of get_connected_mesh (trimesh)
and the face-mask culls between them, in csrc/mesh_view.cu and csrc/mesh.cu.

    Mesher.cull_mesh = goslam_b200.mesher.cull_mesh      # drop-in method; `import pyrender` can go

Tensor-level functions take CUDA tensors: vertices [V,3] f64, faces [F,3] i64, colours [V,C] (any dtype) or None.  Every
cull keeps faces and vertices in their input order (update_faces + remove_unreferenced_vertices) and carries the colours
of the kept vertices along.
"""
import ctypes

import torch

from . import _lib
from .droid_backends import _workspace

DEPTH_CHUNK_BYTES = 256 << 20          # default bound of the depth scratch of view_masks


def _mesh_args(verts, faces):
    if not verts.is_cuda:
        raise RuntimeError("mesher: CUDA tensors required (no CPU fallback)")
    verts = verts.detach().to(torch.float64).reshape(-1, 3).contiguous()
    faces = faces.detach().to(device=verts.device, dtype=torch.int64).reshape(-1, 3).contiguous()
    return verts, faces


def _poses(c2w, dev):
    if isinstance(c2w, (list, tuple)):
        c2w = torch.stack([torch.as_tensor(m) for m in c2w]) if len(c2w) else torch.zeros(0, 4, 4)
    return torch.as_tensor(c2w).detach().to(dev, torch.float32).reshape(-1, 4, 4).contiguous()


def render_depth(verts, faces, c2w, H, W, fx, fy, cx, cy, near=0.001, far=20.0):
    """depth [K,H,W] f32 of the mesh seen from c2w [K,4,4] (OpenCV camera-to-world), 0 where nothing is seen"""
    verts, faces = _mesh_args(verts, faces)
    dev = verts.device
    c2w = _poses(c2w, dev)
    K = c2w.shape[0]
    depth = torch.empty((K, int(H), int(W)), dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        for k0 in range(0, K, 65535):
            k1 = min(K, k0 + 65535)
            rc = lib.goslam_mesh_depth_render(_lib.ptr(verts), verts.shape[0], _lib.ptr(faces), faces.shape[0],
                                              _lib.ptr(c2w[k0:k1]), k1 - k0, int(H), int(W), float(fx), float(fy),
                                              float(cx), float(cy), float(near), float(far), _lib.ptr(depth[k0:k1]),
                                              _lib.stream_ptr())
            _lib.check(rc, "mesh_depth_render")
    return depth


def view_masks(verts, faces, c2w, H, W, fx, fy, cx, cy, radius, eps=0.05, chunk=None):
    """(seen, forecast) bool [V]: point_masks against the mesh's own depth maps.  Views go in chunks of `chunk` (default:
    as many as fit DEPTH_CHUNK_BYTES of depth): rasterize the chunk into scratch, then OR its masks in."""
    verts, faces = _mesh_args(verts, faces)
    dev = verts.device
    c2w = _poses(c2w, dev)
    K, V = c2w.shape[0], verts.shape[0]
    H, W = int(H), int(W)
    if chunk is None:
        chunk = max(1, DEPTH_CHUNK_BYTES // (4 * H * W))
    chunk = max(1, min(int(chunk), 65535))
    seen = torch.zeros(V, dtype=torch.uint8, device=dev)
    fore = torch.zeros(V, dtype=torch.uint8, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        for k0 in range(0, K, chunk):
            k1 = min(K, k0 + chunk)
            depth = render_depth(verts, faces, c2w[k0:k1], H, W, fx, fy, cx, cy, far=20.0)
            w2c = torch.inverse(c2w[k0:k1]).float().contiguous()      # the reference's call, on the device
            rc = lib.goslam_mesh_view_masks(_lib.ptr(verts), V, _lib.ptr(w2c), _lib.ptr(depth), k1 - k0, H, W,
                                            float(fx), float(fy), float(cx), float(cy), float(radius), float(eps),
                                            _lib.ptr(seen), _lib.ptr(fore), _lib.stream_ptr())
            _lib.check(rc, "mesh_view_masks")
            del depth
    return seen.bool(), fore.bool()


def _compact(verts, faces, colors, count):
    """run `count(lib, workspace, counts, stream)` (a cull count entry), then the emit, the kept vertices' ids and the
    colour gather.  One host synchronisation (the two counts)."""
    lib = _lib.load()
    nv, nf = verts.shape[0], faces.shape[0]
    dev = verts.device
    with torch.cuda.device(dev):
        st = _lib.stream_ptr()
        ws = torch.empty(lib.goslam_mesh_cull_workspace_bytes(nv, nf), dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        _lib.check(count(lib, ws, counts, st), "mesh cull count")
        kv, kf = counts.tolist()
        out_v = torch.empty((kv, 3), dtype=torch.float64, device=dev)
        out_f = torch.empty((kf, 3), dtype=torch.int64, device=dev)
        _lib.check(lib.goslam_mesh_cull_emit(_lib.ptr(verts), nv, _lib.ptr(faces), nf, _lib.ptr(ws), ws.numel(),
                                             _lib.ptr(out_v), kv, _lib.ptr(out_f), kf, st), "mesh_cull_emit")
        out_c = None
        if colors is not None:
            ids = torch.empty(kv, dtype=torch.int64, device=dev)
            _lib.check(lib.goslam_mesh_cull_vertex_ids(nv, nf, _lib.ptr(ws), ws.numel(), _lib.ptr(ids), kv, st),
                       "mesh_cull_vertex_ids")
            out_c = colors.index_select(0, ids)
    return out_v, out_f, out_c


def _mask_arg(m, n, dev):
    if m is None:
        return None
    m = torch.as_tensor(m).to(dev).reshape(-1)
    if m.numel() != n:
        raise ValueError("mask has %d entries, expected %d" % (m.numel(), n))
    return (m != 0).to(torch.uint8).contiguous()


def _colors_arg(colors, nv, dev):
    if colors is None:
        return None
    colors = torch.as_tensor(colors).to(dev)
    if colors.shape[0] != nv:
        raise ValueError("colours have %d rows, expected %d" % (colors.shape[0], nv))
    return colors


def keep_faces(verts, faces, face_mask=None, colors=None, vert_mask=None):
    """update_faces(face_mask & vert_mask[faces].all(1)) + remove_unreferenced_vertices: (vertices, faces, colours or
    None), stable orders.  face_mask [F] / vert_mask [V] are boolean (None keeps all)."""
    verts, faces = _mesh_args(verts, faces)
    dev = verts.device
    fm, vm = _mask_arg(face_mask, faces.shape[0], dev), _mask_arg(vert_mask, verts.shape[0], dev)
    colors = _colors_arg(colors, verts.shape[0], dev)
    return _compact(verts, faces, colors, lambda lib, ws, counts, st: lib.goslam_mesh_cull_mask_count(
        verts.shape[0], _lib.ptr(faces), faces.shape[0], _lib.ptr(fm), _lib.ptr(vm), _lib.ptr(ws), ws.numel(),
        _lib.ptr(counts), st))


def _keep_box(verts, faces, lo, hi, colors=None):
    """the bound cull of neus.cull_mesh (lo <= v <= hi, host float32 thresholds), colours carried along"""
    lo = (ctypes.c_float * 3)(*[float(v) for v in lo])
    hi = (ctypes.c_float * 3)(*[float(v) for v in hi])
    return _compact(verts, faces, colors, lambda lib, ws, counts, st: lib.goslam_mesh_cull_count(
        _lib.ptr(verts), verts.shape[0], _lib.ptr(faces), faces.shape[0], lo, hi, _lib.ptr(ws), ws.numel(),
        _lib.ptr(counts), st))


def component_mask(verts, faces, threshold, largest=False):
    """u8 [F]: 1 on the faces of the kept components (get_connected_mesh's rule).  One host synchronisation."""
    verts, faces = _mesh_args(verts, faces)
    nv, nf = verts.shape[0], faces.shape[0]
    dev = verts.device
    keep = torch.zeros(nf, dtype=torch.uint8, device=dev)
    if nf == 0:
        return keep
    lib = _lib.load()
    with torch.cuda.device(dev):
        st = _lib.stream_ptr()
        nbytes = lib.goslam_mesh_components_workspace_bytes(nv, nf)
        if nbytes == 0:
            raise RuntimeError("mesh components: cannot size the workspace for %d faces" % nf)
        ws = _workspace(nbytes, dev)
        counts = torch.empty(1, dtype=torch.int64, device=dev)
        _lib.check(lib.goslam_mesh_components_count(_lib.ptr(verts), nv, _lib.ptr(faces), nf, _lib.ptr(ws), ws.numel(),
                                                    _lib.ptr(counts), st), "mesh_components_count")
        n_comp = int(counts.item())
        _lib.check(lib.goslam_mesh_components_keep(nf, n_comp, float(threshold), int(bool(largest)), _lib.ptr(ws),
                                                   ws.numel(), _lib.ptr(keep), st), "mesh_components_keep")
    return keep


def filter_components(verts, faces, threshold, largest=False, colors=None):
    """get_connected_mesh: the components whose area is > threshold * the mesh's area (largest: only the largest one,
    ties to the smallest face id), as (vertices, faces, colours or None) in input order; empty if none passes"""
    verts, faces = _mesh_args(verts, faces)
    return keep_faces(verts, faces, component_mask(verts, faces, threshold, largest), colors)


# ---- the drop-in method -------------------------------------------------------------------------------------------
def _host(*ts):
    out = [None if t is None else torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in ts]
    for h, t in zip(out, ts):
        if t is not None:
            h.copy_(t, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    return [None if h is None else h.numpy() for h in out]


def _trimesh(v, f, c):
    import trimesh
    hv, hf, hc = _host(v, f, c)
    return trimesh.Trimesh(vertices=hv, faces=hf, vertex_colors=hc, process=False)


def _device_of(mesher):
    dev = torch.device(getattr(mesher, "device", "cuda"))
    if dev.type != "cuda":
        raise RuntimeError("Mesher.cull_mesh on the device needs a CUDA device (no CPU fallback)")
    return dev


@torch.no_grad()
def cull_mesh(self, mesh, estimate_c2w_list, bound, mesh_out_file):
    """Mesher.cull_mesh (src/mesher.py:156-240) with the projection, hole, component and forecast culls on the device;
    exports bound_mesh.ply (when bound is given), mesh_with_hole.ply, mesh_out_file and its _forecast.ply twin and returns
    (cull_mesh, forecast_mesh) as trimesh.Trimesh.  The forecast step's oriented box comes from the caller's Open3D."""
    import numpy as np
    import trimesh  # noqa: F401  (the reference imports it at module level)
    dev = _device_of(self)
    with torch.cuda.device(dev):
        verts = torch.as_tensor(np.asarray(mesh.vertices)[:, :3], dtype=torch.float64).to(dev)
        faces = torch.as_tensor(np.asarray(mesh.faces), dtype=torch.int64).to(dev)
        vc = getattr(getattr(mesh, "visual", None), "vertex_colors", None)
        colors = None if vc is None or len(vc) != len(verts) else torch.as_tensor(np.asarray(vc)).to(dev)
        out_dir = "%s/mesh" % self.output
        if bound is not None:
            if isinstance(bound, np.ndarray):
                eps = 0.001
                verts, faces, colors = _keep_box(verts, faces, bound[:, 0] - eps, bound[:, 1] + eps, colors)
            else:
                inb = bound.in_bound(_host(verts)[0])
                verts, faces, colors = keep_faces(verts, faces, colors=colors, vert_mask=torch.as_tensor(np.asarray(inb)))
            _trimesh(verts, faces, colors).export("%s/bound_mesh.ply" % out_dir)
        seen, fore = view_masks(verts, faces, estimate_c2w_list, self.H, self.W, self.fx, self.fy, self.cx, self.cy,
                                self.forecast_radius)
        hv, hf, hc = keep_faces(verts, faces, colors=colors, vert_mask=seen)
        _trimesh(hv, hf, hc).export("%s/mesh_with_hole.ply" % out_dir)
        thr, largest = self.remove_small_geometry_threshold, self.get_largest_components
        cv, cf, cc = filter_components(hv, hf, thr, largest, hc)
        cull = _trimesh(cv, cf, cc)
        if abs(self.forecast_radius) > 0:
            import open3d as o3d
            fv, ff, fc = keep_faces(verts, faces, colors=colors, vert_mask=fore)
            pc = o3d.geometry.PointCloud(o3d.utility.Vector3dVector(np.array(cull.vertices)))
            box = pc.get_oriented_bounding_box()
            idx = box.get_point_indices_within_bounding_box(o3d.utility.Vector3dVector(_host(fv)[0]))
            inb = np.zeros(fv.shape[0], bool)
            inb[np.asarray(idx, np.int64)] = True
            fv, ff, fc = keep_faces(fv, ff, colors=fc, vert_mask=torch.from_numpy(inb))
            forecast = _trimesh(*filter_components(fv, ff, thr, largest, fc))
        else:
            forecast = _trimesh(cv, cf, cc)
    cull.export(mesh_out_file)
    forecast.export(mesh_out_file.replace(".ply", "_forecast.ply"))
    return cull, forecast
