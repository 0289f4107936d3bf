"""Mesher.cull_mesh (src/mesher.py:156-240) on the device: the depth maps of extract_depth_from_mesh (pyrender / OpenGL in the
reference), the seen / forecast vertex masks of point_masks, the connected-component filter of get_connected_mesh (trimesh)
and the face-mask culls between them, in csrc/mesh_view.cu and csrc/mesh.cu.

    Mesher.cull_mesh = goslam_b200.mesher.cull_mesh      # drop-in method; `import pyrender` can go

The evaluation step of Mesher.__call__(the_end=True) (align_mesh, eval_mesh, src/mesher.py:339-421) runs on the device
too, in csrc/mesh_eval.cu: surface sampling, exact nearest-neighbour search on a uniform grid and point-to-point ICP.

    import src.mesher as m, goslam_b200.mesher as gm
    m.align_mesh, m.eval_mesh = gm.align_mesh, gm.eval_mesh

Tensor-level functions take CUDA tensors: vertices [V,3] f64, faces [F,3] i64, colours [V,C] (any dtype) or None.  Every
cull keeps faces and vertices in their input order (update_faces + remove_unreferenced_vertices) and carries the colours
of the kept vertices along.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib

DEPTH_CHUNK_BYTES = 256 << 20          # default bound of the depth scratch of view_masks


def _mesh_args(verts, faces):
    _lib.need_cuda("mesher", verts)
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
    for k0 in range(0, K, 65535):
        k1 = min(K, k0 + 65535)
        _lib.call("mesh_depth_render", verts, verts.shape[0], faces, faces.shape[0], c2w[k0:k1], k1 - k0, int(H), int(W),
                  float(fx), float(fy), float(cx), float(cy), float(near), float(far), depth[k0:k1])
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
    for k0 in range(0, K, chunk):
        k1 = min(K, k0 + chunk)
        depth = render_depth(verts, faces, c2w[k0:k1], H, W, fx, fy, cx, cy, far=20.0)
        w2c = torch.inverse(c2w[k0:k1]).float().contiguous()      # the reference's call, on the device
        _lib.call("mesh_view_masks", verts, V, w2c, depth, k1 - k0, H, W, float(fx), float(fy), float(cx), float(cy),
                  float(radius), float(eps), seen, fore)
        del depth
    return seen.bool(), fore.bool()


def _compact(verts, faces, colors, count):
    """run `count(workspace, counts)` (a cull count entry), then the emit, the kept vertices' ids and the colour gather.
    One host synchronisation (the two counts)."""
    nv, nf = verts.shape[0], faces.shape[0]
    dev = verts.device
    ws = torch.empty(_lib.load().goslam_mesh_cull_workspace_bytes(nv, nf), dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    count(ws, counts)
    kv, kf = counts.tolist()
    out_v = torch.empty((kv, 3), dtype=torch.float64, device=dev)
    out_f = torch.empty((kf, 3), dtype=torch.int64, device=dev)
    _lib.call("mesh_cull_emit", verts, nv, faces, nf, ws, ws.numel(), out_v, kv, out_f, kf)
    out_c = None
    if colors is not None:
        ids = torch.empty(kv, dtype=torch.int64, device=dev)
        _lib.call("mesh_cull_vertex_ids", nv, nf, ws, ws.numel(), ids, kv)
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
    return _compact(verts, faces, colors, lambda ws, counts: _lib.call(
        "mesh_cull_mask_count", verts.shape[0], faces, faces.shape[0], fm, vm, ws, ws.numel(), counts))


def keep_box(verts, faces, lo, hi, colors=None):
    """the bound cull (lo <= v <= hi, host float32 thresholds) as (vertices, faces, colours or None), stable orders"""
    verts, faces = _mesh_args(verts, faces)
    lo = (ctypes.c_float * 3)(*[float(v) for v in lo])
    hi = (ctypes.c_float * 3)(*[float(v) for v in hi])
    return _compact(verts, faces, colors, lambda ws, counts: _lib.call(
        "mesh_cull_count", verts, verts.shape[0], faces, faces.shape[0], lo, hi, ws, ws.numel(), counts))


def component_mask(verts, faces, threshold, largest=False):
    """u8 [F]: 1 on the faces of the kept components (get_connected_mesh's rule).  One host synchronisation."""
    verts, faces = _mesh_args(verts, faces)
    nv, nf = verts.shape[0], faces.shape[0]
    dev = verts.device
    keep = torch.zeros(nf, dtype=torch.uint8, device=dev)
    if nf == 0:
        return keep
    with torch.cuda.device(dev):
        # CUB sizes its scratch for the current device
        nbytes = _lib.load().goslam_mesh_components_workspace_bytes(nv, nf)
    if nbytes == 0:
        raise RuntimeError("mesh components: cannot size the workspace for %d faces" % nf)
    ws = _lib.workspace(nbytes, dev)
    counts = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.call("mesh_components_count", verts, nv, faces, nf, ws, ws.numel(), counts)
    n_comp = int(counts.item())
    _lib.call("mesh_components_keep", nf, n_comp, float(threshold), int(bool(largest)), ws, ws.numel(), keep)
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
                verts, faces, colors = keep_box(verts, faces, bound[:, 0] - eps, bound[:, 1] + eps, colors)
            elif isinstance(bound, OrientedBoundingBox):
                verts, faces, colors = keep_faces(verts, faces, colors=colors, vert_mask=bound.in_bound(verts))
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


# ---- reconstruction evaluation (align_mesh / eval_mesh) -----------------------------------------------------------
def _points(x, what):
    x = torch.as_tensor(x)
    _lib.need_cuda(what, x)
    x = x.detach().to(torch.float64).reshape(-1, 3).contiguous()
    if x.shape[0] == 0:
        raise ValueError("%s: no points" % what)
    return x


class NNIndex:
    """A uniform-grid index over points [n,3] (CUDA, f64), built once and queried any number of times.  Cells are at
    least `min_cell` wide (pass the radius of radius queries); results do not depend on it."""

    def __init__(self, points, min_cell=0.0):
        self.points = _points(points, "NNIndex")
        n = self.points.shape[0]
        with torch.cuda.device(self.points.device):
            # CUB sizes its scratch for the current device
            nbytes = _lib.load().goslam_nn_index_workspace_bytes(n)
        if nbytes == 0:
            raise RuntimeError("NNIndex: cannot index %d points" % n)
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=self.points.device)
        _lib.call("nn_index_build", self.points, n, float(min_cell), self.buf, nbytes)

    def __len__(self):
        return self.points.shape[0]

    def query(self, query, max_dist=math.inf):
        """(dist f64, idx i64) of the nearest indexed point to each query with distance < max_dist (inf / -1 where
        there is none); the smallest index among equal distances"""
        q = _points(query, "NNIndex.query") if torch.as_tensor(query).numel() else \
            torch.empty((0, 3), dtype=torch.float64, device=self.points.device)
        dist = torch.empty(q.shape[0], dtype=torch.float64, device=q.device)
        idx = torch.empty(q.shape[0], dtype=torch.int64, device=q.device)
        _lib.call("nn_query", self.buf, self.buf.numel(), len(self), q, q.shape[0], float(max_dist), dist, idx)
        return dist, idx


def nearest(query, points, max_dist=math.inf):
    """(dist f64, idx i64): the nearest of points [M,3] to each of query [N,3] (cKDTree.query; with a finite max_dist
    only distances < max_dist count, idx -1 where none does).  Exact."""
    return NNIndex(points, 0.0 if math.isinf(max_dist) else max_dist).query(query, max_dist)


def _uniforms(count, generator, dev):
    """the draws of sample_surface: [count, 3] f64 (face pick, two lengths) from torch's CUDA generator"""
    return torch.rand((count, 3), dtype=torch.float64, device=dev, generator=generator)


def sample_surface_from(verts, faces, uniforms):
    """trimesh.sample.sample_surface for given uniforms [count, 3] (u, l0, l1): area-weighted face choice
    (searchsorted side='left' on the fp64 cumulative areas) and trimesh's point rule.  [count, 3] f64."""
    verts, faces = _mesh_args(verts, faces)
    if faces.shape[0] == 0 or verts.shape[0] == 0:
        raise ValueError("sample_surface: the mesh has no faces")
    u = torch.as_tensor(uniforms).to(verts.device, torch.float64).reshape(-1, 3).contiguous()
    out = torch.empty((u.shape[0], 3), dtype=torch.float64, device=verts.device)
    with torch.cuda.device(verts.device):
        # CUB sizes its scratch for the current device
        nbytes = _lib.load().goslam_mesh_sample_workspace_bytes(faces.shape[0])
    if nbytes == 0:
        raise RuntimeError("sample_surface: cannot size the workspace for %d faces" % faces.shape[0])
    ws = _lib.workspace(nbytes, verts.device)
    _lib.call("mesh_sample_surface", verts, verts.shape[0], faces, faces.shape[0], u, u.shape[0], out, None, ws, nbytes)
    return out


def sample_surface(verts, faces, count, generator=None):
    """[count, 3] f64 area-weighted samples of the mesh's surface, uniforms from torch.rand on the mesh's device"""
    verts = torch.as_tensor(verts)
    _lib.need_cuda("sample_surface", verts)
    return sample_surface_from(verts, faces, _uniforms(int(count), generator, verts.device))


def icp_point_to_point(src, dst, threshold, init=None, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6):
    """Open3D's registration_icp(src, dst, threshold, init, TransformationEstimationPointToPoint()) with its default
    criteria: (T [4,4] f64 on the host, fitness, inlier_rmse, iterations).  dst is a point tensor or an NNIndex built
    with min_cell = threshold.  One host synchronisation."""
    src = _points(src, "icp_point_to_point")
    index = dst if isinstance(dst, NNIndex) else NNIndex(dst, float(threshold))
    dev = src.device
    if index.points.device != dev:
        raise ValueError("icp_point_to_point: source and target on different devices")
    T0 = torch.eye(4, dtype=torch.float64) if init is None else torch.as_tensor(np.asarray(init, np.float64))
    T0 = T0.to(dev, torch.float64).reshape(4, 4).contiguous()
    out = torch.empty(19, dtype=torch.float64, device=dev)
    nbytes = _lib.load().goslam_icp_workspace_bytes(src.shape[0])
    if nbytes == 0:
        raise RuntimeError("icp_point_to_point: cannot size the workspace for %d points" % src.shape[0])
    ws = _lib.workspace(nbytes, dev)
    _lib.call("icp_point_to_point", src, src.shape[0], index.buf, index.buf.numel(), len(index), float(threshold), T0,
              int(max_iteration), float(relative_fitness), float(relative_rmse), out, ws, nbytes)
    host = out.cpu()
    return host[:16].reshape(4, 4).clone(), float(host[16]), float(host[17]), int(host[18])


def _ratio(count, n):
    """np.mean((dist < th).astype(np.float32)) * 100: a float32 mean of exact 0/1 values"""
    return np.float32(np.float32(count) / np.float32(n)) * np.float32(100)


def mesh_metrics(est_pts, gt_pts, dist_th):
    """eval_mesh's five numbers for two point sets: accuracy / completion (mean nearest distance, cm), their ratios
    under dist_th (%) and the F-score, with the reference's dtypes (float64 means, float32 ratios).  One host read."""
    est, gt = _points(est_pts, "mesh_metrics"), _points(gt_pts, "mesh_metrics")
    stats = torch.empty(4, dtype=torch.float64, device=est.device)
    comp, _ = NNIndex(est).query(gt)
    _lib.call("nn_distance_stats", comp, comp.numel(), float(dist_th), stats[0:2])
    acc, _ = NNIndex(gt).query(est)
    _lib.call("nn_distance_stats", acc, acc.numel(), float(dist_th), stats[2:4])
    s = stats.tolist()
    completion = np.float64(s[0]) / gt.shape[0] * 100
    accuracy = np.float64(s[2]) / est.shape[0] * 100
    completion_ratio, accuracy_ratio = _ratio(int(s[1]), gt.shape[0]), _ratio(int(s[3]), est.shape[0])
    with np.errstate(invalid="ignore", divide="ignore"):
        f_score = (2.0 * accuracy_ratio * completion_ratio) / (accuracy_ratio + completion_ratio)
    return dict(accuracy=accuracy, completion=completion, accuracy_ratio=accuracy_ratio,
                completion_ratio=completion_ratio, f_score=f_score)


def metrics_message(m):
    return (f'\n\nMetrics of reconstructed mesh are:\n'
            f'\tAccuracy: {m["accuracy"]:.2f}cm\n'
            f'\tCompletion: {m["completion"]:.2f}cm\n'
            f'\tAccuracy Ratio: {m["accuracy_ratio"]:.2f}%\n'
            f'\tCompletion Ratio: {m["completion_ratio"]:.2f}%\n'
            f'\tF-score: {m["f_score"]:.2f}%\n\n')


def _mesh_tensors(mesh, dev, what):
    verts = torch.as_tensor(np.ascontiguousarray(np.asarray(mesh.vertices, np.float64)[:, :3])).to(dev)
    faces = torch.as_tensor(np.ascontiguousarray(np.asarray(mesh.faces, np.int64).reshape(-1, 3))).to(dev)
    if verts.shape[0] == 0:
        raise ValueError("%s: the mesh is empty" % what)
    return verts, faces


@torch.no_grad()
def align_mesh(est_mesh, gt_mesh, threshold=0.1, trans_init=None, return_transformation=False):
    """align_mesh (src/mesher.py:339-357): point-to-point ICP of est_mesh's vertices onto gt_mesh's, from trans_init
    (identity if None), then est_mesh.apply_transform(T).  Returns the aligned mesh (and T, numpy [4,4] f64)."""
    dev = torch.device("cuda", torch.cuda.current_device())
    src, _ = _mesh_tensors(est_mesh, dev, "align_mesh")
    dst, _ = _mesh_tensors(gt_mesh, dev, "align_mesh")
    T, _, _, _ = icp_point_to_point(src, dst, threshold, np.eye(4) if trans_init is None else trans_init)
    transformation = T.numpy()
    aligned_mesh = est_mesh.apply_transform(transformation)
    if return_transformation:
        return aligned_mesh, transformation
    return aligned_mesh


@torch.no_grad()
def eval_mesh(est_mesh, gt_mesh, N3d=2e5, dist_th=0.05, out_path=None, metric_2d=False, generator=None):
    """eval_mesh (src/mesher.py:390-421): N3d area-weighted samples of each mesh (est first, from torch's CUDA
    generator), nearest distances both ways, the reference's message written to out_path and printed.  Returns the
    metrics as a dict (the reference returns None).  metric_2d is accepted and ignored, as in the reference."""
    N3d = int(N3d)
    dev = torch.device("cuda", torch.cuda.current_device())
    ev, ef = _mesh_tensors(est_mesh, dev, "eval_mesh")
    gv, gf = _mesh_tensors(gt_mesh, dev, "eval_mesh")
    if ef.shape[0] == 0 or gf.shape[0] == 0:
        raise ValueError("eval_mesh: the mesh has no faces")
    est_pc = sample_surface_from(ev, ef, _uniforms(N3d, generator, dev))
    gt_pc = sample_surface_from(gv, gf, _uniforms(N3d, generator, dev))
    m = mesh_metrics(est_pc, gt_pc, dist_th)
    msg = metrics_message(m)
    if out_path is not None:
        with open(out_path, 'w') as fp:
            fp.write(msg)
    print(msg)
    return {k: float(v) for k, v in m.items()}


# ---- the scene bound (update_param_from_mapping, OrientedBoundingBox) ---------------------------------------------
_HULL_STATUS = {1: "fewer than four affinely independent points", 2: "the hull has too many facets",
                3: "a coordinate is not finite", 4: "inconsistent facet graph"}
MAPPING_EXTEND = 0.1            # src/mesher.py:279


def _hull_run(points, what):
    """goslam_hull_vertices on points (CUDA, any float dtype, [n,3]): (points f64, workspace, info [4] on the device)"""
    pts = _points(points, what)
    n = pts.shape[0]
    with torch.cuda.device(pts.device):
        # CUB sizes its scratch for the current device
        nbytes = _lib.load().goslam_hull_workspace_bytes(n)
    if nbytes == 0:
        raise ValueError("%s: %d points (at most 2^28)" % (what, n))
    ws = _lib.workspace(nbytes, pts.device)
    info = torch.empty(4, dtype=torch.int64, device=pts.device)
    _lib.call("hull_vertices", pts, n, ws, nbytes, info)
    return pts, ws, nbytes, info


def _hull_info(info, what):
    status, count, survivors, winners = info.tolist()
    if status:
        err = ValueError if status in (1, 3) else RuntimeError
        raise err("%s: %s" % (what, _HULL_STATUS.get(status, "status %d" % status)))
    return count


def hull_vertices(points):
    """sorted int64 ids of the convex-hull vertices of points [n,3] (CUDA): the exact extreme points, so a point on a
    hull face or edge is not one and of equal points only the lowest index can be.  ValueError when the points span
    less than three dimensions.  One host read."""
    pts, ws, nbytes, info = _hull_run(points, "hull_vertices")
    count = _hull_info(info, "hull_vertices")
    out = torch.empty(count, dtype=torch.int64, device=pts.device)
    _lib.call("hull_vertices_emit", ws, nbytes, pts.shape[0], out, count)
    return out


def _oriented_box(points, extend):
    """box [15] f64 on the device (center, R row-major, extent + extend).  One host read (the hull's status)."""
    pts, ws, nbytes, info = _hull_run(points, "oriented_box")
    box = torch.empty(15, dtype=torch.float64, device=pts.device)
    _lib.call("obb_from_hull", pts, pts.shape[0], ws, nbytes, float(extend), box)
    _hull_info(info, "oriented_box")
    return box


def oriented_box(points, extend=0.0):
    """Open3D 0.13's OrientedBoundingBox.create_from_points(points) as (center [3], R [3,3], extent [3]) f64 on the
    device, extent + extend as in compute_from_pointcloud.  R's columns are the hull vertices' principal axes by
    descending variance; columns 0 and 1 have their largest-magnitude component positive, column 2 = column 0 x 1."""
    box = _oriented_box(points, extend)
    return box[0:3], box[3:12].view(3, 3), box[12:15]


def in_oriented_box(points, center, R, extent):
    """bool [n]: Open3D's get_point_indices_within_bounding_box rule (six plane tests on the box corners) for points
    [n,3] (CUDA).  The box is read on the device."""
    pts = torch.as_tensor(points)
    _lib.need_cuda("in_oriented_box", pts)
    pts = pts.detach().to(torch.float64).reshape(-1, 3).contiguous()
    dev = pts.device
    box = torch.cat([torch.as_tensor(t).to(dev, torch.float64).reshape(-1) for t in (center, R, extent)])
    if box.numel() != 15:
        raise ValueError("in_oriented_box: center [3], R [3,3] and extent [3] expected")
    mask = torch.empty(pts.shape[0], dtype=torch.uint8, device=dev)
    _lib.call("obb_in_bound", box, pts, pts.shape[0], mask)
    return mask.bool()


class OrientedBoundingBox(torch.nn.Module):
    """src/oriented_bounding_box.py with the hull, the box and the in-bound test on the device.  Buffers center [3],
    R [3,3] and extent [3] are float64, as in the reference."""

    def __init__(self):
        super().__init__()
        self.register_buffer('center', torch.zeros(3,).double())
        self.register_buffer('R', torch.zeros(3, 3).double())
        self.register_buffer('extent', torch.zeros(3,).double())

    def _init(self, center, R, extent):
        device = self.center.device
        self.center[:] = torch.as_tensor(center).to(device).double()
        self.R[:] = torch.as_tensor(R).to(device).double()
        self.extent[:] = torch.as_tensor(extent).to(device).double()

    def _clone(self, aabb):
        self._init(aabb.center, aabb.R, aabb.extent)

    def _device(self):
        dev = self.center.device
        return dev if dev.type == "cuda" else torch.device("cuda", torch.cuda.current_device())

    def compute_from_pointcloud(self, pointcloud, extend=0.0):
        """the oriented box of pointcloud (ndarray or CUDA tensor [n,3]), extent + extend"""
        pts = torch.as_tensor(np.asarray(pointcloud) if isinstance(pointcloud, np.ndarray) else pointcloud)
        if not pts.is_cuda:
            pts = pts.to(self._device())
        box = _oriented_box(pts, extend)
        dev = self.center.device
        self.center[:] = box[0:3].to(dev)
        self.R[:] = box[3:12].view(3, 3).to(dev)
        self.extent[:] = box[12:15].to(dev)

    def in_bound(self, pointcloud):
        """points inside the box: a numpy bool [n] for an ndarray, a CUDA bool [n] for a CUDA tensor"""
        if isinstance(pointcloud, torch.Tensor) and pointcloud.is_cuda:
            dev = pointcloud.device
            return in_oriented_box(pointcloud, self.center.to(dev), self.R.to(dev), self.extent.to(dev))
        dev = self._device()
        pts = torch.as_tensor(np.asarray(pointcloud, np.float64)).to(dev)
        mask = in_oriented_box(pts, self.center.to(dev), self.R.to(dev), self.extent.to(dev))
        return mask.cpu().numpy().astype(np.bool_)

    def get_aabb(self):
        import open3d as o3d
        center = self.center.detach().cpu().numpy().astype(np.float64)
        R = self.R.detach().cpu().numpy().astype(np.float64)
        extent = self.extent.detach().cpu().numpy().astype(np.float64)
        return o3d.geometry.OrientedBoundingBox(center=center, R=R, extent=extent)

    def box_points(self):
        """the 8 corners [8,3] f64 in Open3D's GetBoxPoints order"""
        c, R, e = (t.detach().cpu().double() for t in (self.center, self.R, self.extent))
        ax = [R[:, j] * (e[j] / 2) for j in range(3)]
        sg = [(-1, -1, -1), (1, -1, -1), (-1, 1, -1), (-1, -1, 1), (1, 1, 1), (-1, 1, 1), (1, -1, 1), (1, 1, -1)]
        return torch.stack([c + s[0] * ax[0] + s[1] * ax[1] + s[2] * ax[2] for s in sg])

    def get_axis_aligned_bounding_box(self):
        """[3,2] float32: min and max of the 8 corners"""
        pts = self.box_points().numpy()
        return np.concatenate([pts.min(0).astype(np.float32)[:, None], pts.max(0).astype(np.float32)[:, None]], axis=1)


def mapping_points(video, cur_idx):
    """the points update_param_from_mapping(the_end=True) bounds (src/mesher.py:256-276) as f64 [n,3] on the video's
    device: iproj of keyframes [0, cur_idx) at full resolution under w2w * SE3(poses).inv(), where depth_filter gives
    >= 3 votes (thresh 0.01) and disps_up > 0.01 * the frame's mean, in [b, h, w] order.  One host read (the count)."""
    from . import lietorch
    T = int(cur_idx)
    dev = video.poses.device
    if dev.type != "cuda":
        raise RuntimeError("mapping_points: a CUDA video is required (no CPU fallback)")
    _, ht, wd = video.disps_up.shape
    with torch.cuda.device(dev):
        # CUB sizes its scratch for the current device
        nbytes = _lib.load().goslam_mapping_points_workspace_bytes(T, ht, wd)
    if nbytes == 0:
        raise ValueError("mapping_points: invalid shape (%d, %d, %d)" % (T, ht, wd))
    poses = video.poses.detach()[:T].float().contiguous()
    disps = video.disps_up.detach()[:T].float().contiguous()
    intr = (video.intrinsics[0].detach() * video.scale_factor).float().contiguous()
    w2w = lietorch.SE3(video.pose_compensate[0].clone().unsqueeze(dim=0)).to(dev)
    poses_world = (w2w * lietorch.SE3(poses).inv()).data.float().contiguous()
    ws = _lib.workspace(nbytes, dev)
    count = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.call("mapping_points_count", poses, poses_world, disps, intr, T, ht, wd, ws, nbytes, count)
    n = int(count.item())
    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    _lib.call("mapping_points_emit", poses_world, disps, intr, T, ht, wd, ws, nbytes, out, n)
    return out


@torch.no_grad()
def update_param_from_mapping(self, the_end=False):
    """Mesher.update_param_from_mapping (src/mesher.py:242-281): (timestamp, cur_idx - 1, a device copy of the shared
    mapping net, the scene's OrientedBoundingBox with extend 0.1 when the_end else None, keyframe camera-to-world
    matrices on the CPU).  The point selection, hull and box stay on the device."""
    import copy
    from . import lietorch
    net = copy.deepcopy(self.shared_mapping_net).to(self.device)
    cur_idx = self.video.counter.value
    timestamp = self.video.timestamp[cur_idx - 1]
    aabb = None
    kf_c2w_list = lietorch.SE3(self.video.poses.detach()[:cur_idx]).inv().matrix().data.cpu()
    if the_end:
        sel_points = mapping_points(self.video, cur_idx)
        aabb = OrientedBoundingBox().to(self.device)
        aabb.compute_from_pointcloud(sel_points, extend=MAPPING_EXTEND)
    return timestamp, cur_idx - 1, net, aabb, kf_c2w_list
