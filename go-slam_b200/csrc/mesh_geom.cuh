// mesh_geom.cuh — per-face geometry shared by the mesh kernels (component filter, surface sampling).
#pragma once
#include <cuda_runtime.h>

// 0.5 |(p1 - p0) x (p2 - p0)| in fp64, every operation rounded on its own (no FMA contraction), so that
// oracle/mesh_view_oracle.py:face_areas reproduces it bit for bit
__device__ __forceinline__ double gs_face_area(const double* p0, const double* p1, const double* p2) {
  const double ax = __dsub_rn(p1[0], p0[0]), ay = __dsub_rn(p1[1], p0[1]), az = __dsub_rn(p1[2], p0[2]);
  const double bx = __dsub_rn(p2[0], p0[0]), by = __dsub_rn(p2[1], p0[1]), bz = __dsub_rn(p2[2], p0[2]);
  const double cx = __dsub_rn(__dmul_rn(ay, bz), __dmul_rn(az, by));
  const double cy = __dsub_rn(__dmul_rn(az, bx), __dmul_rn(ax, bz));
  const double cz = __dsub_rn(__dmul_rn(ax, by), __dmul_rn(ay, bx));
  return __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz))));
}
