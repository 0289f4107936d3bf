"""CPU oracle (TEST INFRASTRUCTURE -- never imported by the product path) for the projection and component culls of
Mesher.cull_mesh (src/mesher.py:56-240).

* render_depth(...)     extract_depth_from_mesh under the rules csrc/mesh_view.cu states, vectorised numpy fp64, operation
                        by operation as the device evaluates them (the device must match it bit for bit): camera
                        coordinates R^T (p - t), near clip into up to two pieces, pixel centres (c + 0.5, r + 0.5),
                        inclusive edge functions of either winding, 1/z interpolated in screen space, far discard,
                        nearest fragment, 0 where nothing lands.
* point_masks(...)      point_masks restated in torch f32 on the CPU with the reference's operations and shapes
                        (w2c @ [p, 1], K @ cam, grid_sample border / align_corners=True, the eps front test).
* keep_faces(...)       update_faces(face_mask) + remove_unreferenced_vertices, stable orders, colours gathered.
* components(...)       get_connected_mesh: face adjacency through edges shared by exactly two faces,
                        scipy.sparse.csgraph.connected_components, per-component fp64 areas, the threshold / largest rule.
"""
import numpy as np

F32 = np.float32


# ---- depth rasterizer ---------------------------------------------------------------------------------------------
def _clip_point(a, b, znear):
    t = (znear - a[:, 2]) / (b[:, 2] - a[:, 2])
    return np.stack([a[:, 0] + t * (b[:, 0] - a[:, 0]), a[:, 1] + t * (b[:, 1] - a[:, 1]), np.full(len(a), znear)], 1)


def _rotate(a, b, c, first_b, first_c):
    """per row: (a, b, c) rotated so that b (first_b) or c (first_c) comes first, winding kept"""
    sel = lambda m, x, y: np.where(m[:, None], x, y)
    i = sel(first_c, c, sel(first_b, b, a))
    j = sel(first_c, a, sel(first_b, c, b))
    k = sel(first_c, b, sel(first_b, a, c))
    return i, j, k


def _pieces(A, B, C, znear):
    """camera-space triangles [n,3] x 3 -> clipped pieces (q0, q1, q2) against z = znear"""
    ia, ib, ic = A[:, 2] >= znear, B[:, 2] >= znear, C[:, 2] >= znear
    nin = ia.astype(int) + ib + ic
    out = []
    m = nin == 3
    out.append((A[m], B[m], C[m]))
    m = nin == 1
    i, j, k = _rotate(A[m], B[m], C[m], ib[m], ic[m])
    out.append((i, _clip_point(i, j, znear), _clip_point(i, k, znear)))
    m = nin == 2
    o, i, j = _rotate(A[m], B[m], C[m], ~ib[m], ~ic[m])
    qj, qi = _clip_point(j, o, znear), _clip_point(i, o, znear)
    out.append((i, j, qj))
    out.append((i, qj, qi))
    return [np.concatenate([p[n] for p in out]) for n in range(3)]


def render_depth(verts, faces, c2w, H, W, fx, fy, cx, cy, near=0.001, far=20.0):
    """depth [K,H,W] float32"""
    verts = np.asarray(verts, np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    c2w = np.asarray(c2w, F32).reshape(-1, 4, 4)
    fx, fy, cx, cy, near, far = (float(v) for v in (fx, fy, cx, cy, near, far))
    out = np.zeros((len(c2w), H, W), F32)
    for k, M in enumerate(c2w):
        R, t = M[:3, :3].astype(np.float64), M[:3, 3].astype(np.float64)
        d = verts - t
        cam = np.stack([(R[0, c] * d[:, 0] + R[1, c] * d[:, 1]) + R[2, c] * d[:, 2] for c in range(3)], 1)
        q = _pieces(cam[faces[:, 0]], cam[faces[:, 1]], cam[faces[:, 2]], near)
        x = [fx * (p[:, 0] / p[:, 2]) + cx for p in q]
        y = [fy * (p[:, 1] / p[:, 2]) + cy for p in q]
        iz = [1.0 / p[:, 2] for p in q]
        area = (x[1] - x[0]) * (y[2] - y[0]) - (y[1] - y[0]) * (x[2] - x[0])
        c0 = np.maximum(0.0, np.ceil(np.minimum(np.minimum(x[0], x[1]), x[2]) - 0.5))
        c1 = np.minimum(W - 1.0, np.floor(np.maximum(np.maximum(x[0], x[1]), x[2]) - 0.5))
        r0 = np.maximum(0.0, np.ceil(np.minimum(np.minimum(y[0], y[1]), y[2]) - 0.5))
        r1 = np.minimum(H - 1.0, np.floor(np.maximum(np.maximum(y[0], y[1]), y[2]) - 0.5))
        ok = (area != 0) & np.isfinite(area) & (c0 <= c1) & (r0 <= r1)
        x, y, iz = [v[ok] for v in x], [v[ok] for v in y], [v[ok] for v in iz]
        area = area[ok]
        c0, r0 = c0[ok].astype(np.int64), r0[ok].astype(np.int64)
        bw, bh = c1[ok].astype(np.int64) - c0 + 1, r1[ok].astype(np.int64) - r0 + 1
        n = bw * bh
        img = np.full(H * W, np.inf, F32)
        if n.sum():
            pid = np.repeat(np.arange(len(n)), n)
            loc = np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)
            r = r0[pid] + loc // bw[pid]
            c = c0[pid] + loc % bw[pid]
            px, py = c + 0.5, r + 0.5
            X = [v[pid] for v in x]
            Y = [v[pid] for v in y]
            e0 = (X[2] - X[1]) * (py - Y[1]) - (Y[2] - Y[1]) * (px - X[1])
            e1 = (X[0] - X[2]) * (py - Y[2]) - (Y[0] - Y[2]) * (px - X[2])
            e2 = (X[1] - X[0]) * (py - Y[0]) - (Y[1] - Y[0]) * (px - X[0])
            inside = ((e0 >= 0) & (e1 >= 0) & (e2 >= 0)) | ((e0 <= 0) & (e1 <= 0) & (e2 <= 0))
            a = area[pid]
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = ((e0 / a) * iz[0][pid] + (e1 / a) * iz[1][pid]) + (e2 / a) * iz[2][pid]
                z = 1.0 / inv
            keep = inside & (z > 0) & (z <= far)
            np.minimum.at(img, r[keep] * W + c[keep], z[keep].astype(F32))
        img[np.isinf(img)] = 0
        out[k] = img.reshape(H, W)
    return out


# ---- view masks ---------------------------------------------------------------------------------------------------
def point_masks(verts, depth, c2w, H, W, fx, fy, cx, cy, radius, eps=0.05):
    """(seen, forecast) bool [V]: the reference's f32 arithmetic on the CPU, one batch of all vertices"""
    import torch
    import torch.nn.functional as F
    pts = torch.as_tensor(np.asarray(verts)).clone().float()
    ones = torch.ones_like(pts[:, 0]).reshape(-1, 1)
    homo = torch.cat([pts, ones], 1).reshape(-1, 4, 1)
    Kd = np.eye(3)
    Kd[0, 0], Kd[0, 2], Kd[1, 1], Kd[1, 2] = fx, cx, fy, cy
    Kf = torch.from_numpy(Kd).float()
    seen = torch.zeros(len(pts), dtype=torch.bool)
    fore = torch.zeros(len(pts), dtype=torch.bool)
    r = radius
    for c2w_k, d_k in zip(torch.as_tensor(np.asarray(c2w)).float(), torch.as_tensor(np.asarray(depth))):
        w2c = torch.inverse(c2w_k).float()
        uvz = Kf @ (w2c @ homo)[:, :3, :].float()
        z = uvz[:, -1:] + 1e-8
        uv = uvz[:, :2] / z
        u, v, z = uv[:, 0, 0], uv[:, 1, 0], z[:, 0, 0]
        in_f = (u >= 0) & (u <= W - 1) & (v >= 0) & (v <= H - 1) & (z > 0)
        fc_f = (u >= -r) & (u <= W - 1 + r) & (v >= -r) & (v <= H - 1 + r) & (z > 0)
        g = uv.reshape(1, 1, -1, 2).clone()
        g[..., 0] = g[..., 0] / (W - 1) * 2.0 - 1.0
        g[..., 1] = g[..., 1] / (H - 1) * 2.0 - 1.0
        ds = F.grid_sample(d_k.float().reshape(1, 1, H, W), g, padding_mode="border", align_corners=True).reshape(-1)
        front = torch.where(ds > 0.0, z < ds + eps, torch.ones_like(z).bool())
        seen |= in_f & front
        fore |= (fc_f & front) | (in_f & front)
    return seen.numpy(), fore.numpy()


def mask_margins(verts, depth, c2w, H, W, fx, fy, cx, cy, radius, eps=0.05):
    """per vertex, the smallest relative distance (f64) to a decision boundary over all views: z against d + eps (d from
    the f64 bilinear sample) and u, v against the frustum bounds, measured where the vertex is in front of the camera"""
    verts = np.asarray(verts, np.float64)
    best = np.full(len(verts), np.inf)
    for M, d in zip(np.asarray(c2w, np.float64), np.asarray(depth, np.float64)):
        w2c = np.linalg.inv(M)
        cam = verts @ w2c[:3, :3].T + w2c[:3, 3]
        z = cam[:, 2] + 1e-8
        with np.errstate(divide="ignore", invalid="ignore"):
            u = (fx * cam[:, 0] + cx * cam[:, 2]) / z
            v = (fy * cam[:, 1] + cy * cam[:, 2]) / z
        ok = z > 0
        rel = lambda a, b: np.abs(a - b) / np.maximum(np.maximum(np.abs(a), np.abs(b)), 1.0)
        m = np.full(len(verts), np.inf)
        for val, bounds in ((u, (0.0, W - 1.0, -radius, W - 1.0 + radius)), (v, (0.0, H - 1.0, -radius, H - 1.0 + radius))):
            for bnd in bounds:
                m = np.minimum(m, np.where(ok, rel(val, bnd), np.inf))
        ix = np.clip(np.nan_to_num(u, nan=0.0, posinf=W - 1, neginf=0), 0, W - 1)
        iy = np.clip(np.nan_to_num(v, nan=0.0, posinf=H - 1, neginf=0), 0, H - 1)
        x0, y0 = np.floor(ix).astype(int), np.floor(iy).astype(int)
        x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
        fx_, fy_ = ix - x0, iy - y0
        ds = ((d[y0, x0] * (1 - fx_) + d[y0, x1] * fx_) * (1 - fy_) + (d[y1, x0] * (1 - fx_) + d[y1, x1] * fx_) * fy_)
        m = np.minimum(m, np.where(ok & (ds > 0), rel(z, ds + eps), np.inf))
        m = np.minimum(m, np.where(ok, rel(ds, 0.0), np.inf))
        best = np.minimum(best, m)
    return best


# ---- face-mask cull and components --------------------------------------------------------------------------------
def keep_faces(verts, faces, face_mask, colors=None):
    """(vertices, faces, colours or None, kept old vertex ids)"""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    f = faces[np.asarray(face_mask, bool)]
    ref = np.zeros(len(verts), bool)
    ref[f.reshape(-1)] = True
    new = np.cumsum(ref) - 1
    ids = np.nonzero(ref)[0]
    return (np.asarray(verts)[ref], new[f].reshape(-1, 3).astype(np.int64),
            None if colors is None else np.asarray(colors)[ref], ids)


def face_areas(verts, faces):
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b = v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]
    c = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    return 0.5 * np.sqrt((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2])


def component_labels(faces):
    """label per face = the smallest face id of its component (adjacency: edges on exactly two faces)"""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    nf = len(f)
    if nf == 0:
        return np.zeros(0, np.int64)
    e = np.sort(np.stack([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], 1).reshape(-1, 2), axis=1)
    ef = np.repeat(np.arange(nf), 3)
    _, inv, cnt = np.unique(e, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    pair = cnt[inv] == 2
    order = np.argsort(inv[pair], kind="stable")
    fa = ef[pair][order].reshape(-1, 2)
    g = sp.coo_matrix((np.ones(len(fa)), (fa[:, 0], fa[:, 1])), shape=(nf, nf))
    _, lab = connected_components(g, directed=False)
    smallest = np.full(lab.max() + 1, nf)
    np.minimum.at(smallest, lab, np.arange(nf))
    return smallest[lab]


def component_face_mask(verts, faces, threshold, largest=False):
    lab = component_labels(faces)
    if len(lab) == 0:
        return np.zeros(0, bool)
    area = face_areas(verts, faces)
    ids, seg = np.unique(lab, return_inverse=True)
    comp = np.bincount(seg.reshape(-1), weights=area, minlength=len(ids))
    if largest:
        keep = np.arange(len(ids)) == int(np.argmax(comp))        # first maximum: the smallest face id
    else:
        keep = comp > threshold * area.sum()
    return keep[seg.reshape(-1)]


def components(verts, faces, threshold, largest=False, colors=None):
    """get_connected_mesh in stable input order: (vertices, faces, colours or None)"""
    v, f, c, _ = keep_faces(verts, faces, component_face_mask(verts, faces, threshold, largest), colors)
    return v, f, c
