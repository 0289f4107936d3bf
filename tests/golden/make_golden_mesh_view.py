"""Generate tests/golden/mesh_view.npz by running THE REFERENCE'S OWN Mesher.point_masks (src/mesher.py:56-136) on the CPU.

The method is called unbound on a namespace that carries what it reads (H, W, fx, fy, cx, cy, device='cpu',
points_batch_size, forecast_radius).  Inputs: the mesh oracle/mesh_oracle.py extracts from the mesh.npz scene at res 40
(vertices, faces, colours), 12 seeded poses around and inside the scene (some see nothing, some stand inside the surface's
hull or close to it, so parts of the mesh are behind the camera or behind other parts), 60x80 intrinsics, radius 25, and
the depth maps of oracle/mesh_view_oracle.py's rasterizer (stored: the device must reproduce them bit for bit).

Stand-ins (make_golden.install_stubs, plus empty open3d / pyrender / trimesh / matplotlib modules, which point_masks does
not use).

Run:  python tests/golden/make_golden_mesh_view.py      (needs the reference source tree, see make_golden.REF)
"""
import os
import sys
import types

import numpy as np
import torch

import make_golden as mg
from oracle import mesh_oracle, mesh_view_oracle, neus_oracle  # noqa: E402  (make_golden puts the repository on sys.path)

H, W, FX, FY, CX, CY = 60, 80, 50.0, 48.0, 39.5, 29.5
RADIUS, RES, SEED = 25, 40, 11


def look_at(pos, target, roll=0.0):
    """OpenCV camera-to-world: z forward, y down"""
    z = np.asarray(target, np.float64) - pos
    z /= np.linalg.norm(z)
    x = np.cross(z, [0.0, 0.0, 1.0])
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    c, s = np.cos(roll), np.sin(roll)
    x, y = c * x + s * y, -s * x + c * y
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = x, y, z, pos
    return m


def poses(verts, rng):
    centre = verts.mean(0)
    out = []
    for k in range(6):                                   # around the scene, looking at it
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        out.append(look_at(centre + 3.0 * d, centre + rng.normal(0, 0.2, 3), rng.uniform(-0.3, 0.3)))
    for k in range(3):                                   # inside the scene's box, random directions
        p = centre + rng.uniform(-0.5, 0.5, 3)
        out.append(look_at(p, p + rng.normal(size=3), rng.uniform(-3, 3)))
    v = verts[rng.integers(len(verts))]                  # a few centimetres from the surface, looking along it
    out.append(look_at(v + rng.normal(0, 0.03, 3), centre))
    for k in range(2):                                   # looking away from the scene: sees nothing
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        p = centre + 4.0 * d
        out.append(look_at(p, p + d))
    return np.stack(out).astype(np.float32)


def main():
    mg.install_stubs()
    for name in ("open3d", "pyrender", "trimesh", "matplotlib", "matplotlib.pyplot"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    mesher = mg.ref_import("src.mesher")
    from goslam_b200 import synthetic
    g = np.load(os.path.join(mg.HERE, "mesh.npz"))
    metas, tot = neus_oracle.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [tot * 2]
    w = synthetic.make_neus_weights(seed=int(g["weights_seed"]), total_grid_params=tot * 2,
                                    layout=(offs, [m["res"] for m in metas]))
    _, verts, faces, colors = mesh_oracle.extract_mesh(w, g["bound"], g["rt_bound"], RES, 0.0, color=True)
    c2w = poses(verts, np.random.default_rng(SEED))
    depth = mesh_view_oracle.render_depth(verts, faces, c2w, H, W, FX, FY, CX, CY)
    ns = types.SimpleNamespace(H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY, device="cpu", points_batch_size=len(verts),
                               forecast_radius=RADIUS)
    seen, fore = mesher.Mesher.point_masks(ns, verts, [torch.from_numpy(d) for d in depth],
                                           [torch.from_numpy(m) for m in c2w])
    np.savez_compressed(os.path.join(mg.HERE, "mesh_view.npz"), verts=verts, faces=faces, colors=colors, c2w=c2w,
                        depth=depth, intrinsics=np.array([H, W, FX, FY, CX, CY], np.float64), radius=RADIUS,
                        seen=seen, forecast=fore)
    print("V %d F %d, seen %d forecast %d, views with depth %d of %d"
          % (len(verts), len(faces), seen.sum(), fore.sum(), int((depth > 0).any((1, 2)).sum()), len(c2w)))


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        raise SystemExit("needs the reference source tree (%s)" % mg.REF)
    main()
    print("wrote mesh_view")
