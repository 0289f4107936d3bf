"""Generate the marching-cubes case tables (go-slam_b200/csrc/mc_tables.cuh).

    python tools/gen_mc_tables.py            # rewrites the header next to the CUDA sources

No table is copied from anywhere: every one of the 256 cases is built here from the cube's faces.
The reference meshes with PyMCubes (`mcubes.marching_cubes`), whose table, triangle orientation and
vertex order are not pinned by the reference (it is an unpinned pip dependency, absent like
tiny-cuda-nn), so these tables define this project's marching cubes; the rules are:

* Corner c of a cell sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1).  A corner is inside iff
  u > iso (the mesher's u is -sdf, so inside means sdf < -iso).
* Edge e joins two corners that differ along axis a = e // 4; its start corner has 0 along a and
  bits (e & 1, (e >> 1) & 1) along the other two axes in increasing order.  The edge carries a
  vertex iff its two corners are classified differently.
* On each face the crossing edges are joined by segments that separate the inside corners from the
  outside ones.  On an ambiguous face (two diagonal corners inside) each inside corner is cut off
  on its own, so the inside corners are kept apart.  Both cells that share a face make the same
  choice, which keeps the surface closed across cells.
* Each segment is directed so that, seen from outside the cube through that face, the inside
  corners lie on its right; the segments then chain into closed loops, each crossing edge being the
  end of one segment and the start of the next.  Loops that come out separate stay separate.
* Each loop is fan-triangulated from its first vertex.  A loop starts at its lowest edge, or, where
  a fan from there would draw a diagonal between two edges of the same cube face (possible on an
  ambiguous face that the loop crosses twice), at the next vertex along the loop that draws none:
  a diagonal in a face could coincide with one from the neighbouring cell, and every mesh edge
  must stay shared by exactly two triangles.  With the segment direction above the normal
  (v1 - v0) x (v2 - v0) of each loop points from u > iso towards u < iso, i.e. outward for an SDF
  scene.
"""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "go-slam_b200", "csrc", "mc_tables.cuh")


def corner_pos(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.float64)


def edge_corners(e):
    """(start corner, end corner) of cell edge e."""
    a = e // 4
    o1, o2 = [d for d in range(3) if d != a]
    s = ((e & 1) << o1) | (((e >> 1) & 1) << o2)
    return s, s | (1 << a)


def edge_between(c0, c1):
    d = c0 ^ c1
    a = d.bit_length() - 1
    lo = min(c0, c1)
    o1, o2 = [x for x in range(3) if x != a]
    return 4 * a + ((lo >> o1) & 1) + 2 * ((lo >> o2) & 1)


def edge_mid(e):
    s, t = edge_corners(e)
    return 0.5 * (corner_pos(s) + corner_pos(t))


def faces():
    """the 6 cube faces: (outward normal, 4 corners in cyclic order)"""
    out = []
    for a in range(3):
        o1, o2 = [d for d in range(3) if d != a]
        for side in (0, 1):
            base = side << a
            ring = [base, base | (1 << o1), base | (1 << o1) | (1 << o2), base | (1 << o2)]
            n = np.zeros(3)
            n[a] = 1.0 if side else -1.0
            out.append((n, ring))
    return out


def face_segments(case, normal, ring):
    """directed segments (start edge, end edge) on one face"""
    inside = [bool((case >> c) & 1) for c in ring]
    segs = []
    if sum(inside) == 2 and inside[0] == inside[2]:
        # ambiguous face: cut off each inside corner separately
        groups = [[k] for k in range(4) if inside[k]]
    elif 0 < sum(inside) < 4:
        groups = [[k for k in range(4) if inside[k]]]
    else:
        return segs
    for g in groups:
        # the two crossing edges bounding this run of inside corners
        ends = []
        for k in g:
            for nb in ((k - 1) % 4, (k + 1) % 4):
                if not inside[nb]:
                    ends.append(edge_between(ring[k], ring[nb]))
        assert len(ends) == 2, (case, ring, g)
        e0, e1 = ends
        p0, p1 = edge_mid(e0), edge_mid(e1)
        cin = corner_pos(ring[g[0]])
        side = float(np.dot(normal, np.cross(p1 - p0, cin - p0)))
        assert side != 0.0
        segs.append((e0, e1) if side < 0 else (e1, e0))
    return segs


def case_loops(case):
    nxt = {}
    for n, ring in faces():
        for s, t in face_segments(case, n, ring):
            assert s not in nxt, (case, s)
            nxt[s] = t
    assert sorted(nxt) == sorted(nxt.values())
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start
        loops.append(loop)
    return loops


def edge_faces(e):
    """indices (into faces()) of the two cube faces that contain edge e"""
    s, t = edge_corners(e)
    return {i for i, (_, ring) in enumerate(faces()) if s in ring and t in ring}


def fan_start(loop):
    """the loop rotated to its first vertex whose fan diagonals leave the cube faces"""
    n = len(loop)
    for r in range(n):
        lp = loop[r:] + loop[:r]
        if all(not (edge_faces(lp[0]) & edge_faces(lp[k])) for k in range(2, n - 1)):
            return lp
    raise AssertionError("no fan start for loop %s" % (loop,))


def case_triangles(case):
    tris = []
    for loop in case_loops(case):
        loop = fan_start(loop)
        for k in range(1, len(loop) - 1):
            tris.append((loop[0], loop[k], loop[k + 1]))
    return tris


def build_tables():
    """(ntri [256] uint8, tris [256, 3 * max_tris] int8 padded with -1)"""
    all_tris = [case_triangles(c) for c in range(256)]
    mt = max(len(t) for t in all_tris)
    ntri = np.array([len(t) for t in all_tris], np.uint8)
    tab = np.full((256, 3 * mt), -1, np.int8)
    for c, tl in enumerate(all_tris):
        for k, t in enumerate(tl):
            tab[c, 3 * k:3 * k + 3] = t
    return ntri, tab


def render_header():
    ntri, tab = build_tables()
    mt = tab.shape[1] // 3
    lines = [
        "// Generated by tools/gen_mc_tables.py -- do not edit.  The rules that define the tables are in",
        "// that script's docstring: corner c at (c&1, c>>1&1, c>>2&1), inside iff u > iso, edge e along",
        "// axis e/4, ambiguous faces keep their inside corners apart, loops fan-triangulated, normals",
        "// pointing from u > iso towards u < iso.",
        "#pragma once",
        "",
        "#define GOSLAM_MC_MAX_TRIS %d" % mt,
        "",
        "__device__ const unsigned char c_mc_ntri[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("  " + ", ".join(str(int(v)) for v in ntri[r:r + 32]) + ",")
    lines.append("};")
    lines.append("")
    lines.append("__device__ const signed char c_mc_tris[256][%d] = {" % (3 * mt))
    for c in range(256):
        lines.append("  {" + ", ".join(str(int(v)) for v in tab[c]) + "},")
    lines.append("};")
    return "\n".join(lines) + "\n"


if __name__ == "__main__":
    with open(OUT, "w") as f:
        f.write(render_header())
    ntri, _ = build_tables()
    print("wrote %s: max %d triangles per case, %d triangles over all cases" % (OUT, ntri.max(), int(ntri.sum())))
