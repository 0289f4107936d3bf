// mesh_geom.cuh — geometry shared by the mesh kernels: per-face areas (component filter, surface sampling) and the
// one-thread 3x3 Jacobi SVD (ICP's Umeyama update, the trajectory's Sim(3) alignment, the oriented box's principal axes).
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

// One-sided Jacobi SVD of the 3x3 row-major A: B = A V with mutually orthogonal columns, V orthogonal (row-major).  The
// singular values are the column norms of B; for a symmetric positive semi-definite A they are its eigenvalues and the
// columns of V its eigenvectors.  One thread, at most 64 sweeps.
__device__ __forceinline__ void gs_jacobi3(const double A[9], double B[9], double V[9]) {
  for (int k = 0; k < 9; ++k) {
    B[k] = A[k];
    V[k] = (k % 4 == 0) ? 1.0 : 0.0;
  }
  for (int sweep = 0; sweep < 64; ++sweep) {
    bool rotated = false;
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      double al = 0.0, be = 0.0, ga = 0.0;
      for (int r = 0; r < 3; ++r) {
        al += B[3 * r + p] * B[3 * r + p];
        be += B[3 * r + q] * B[3 * r + q];
        ga += B[3 * r + p] * B[3 * r + q];
      }
      if (ga == 0.0 || fabs(ga) <= 1e-16 * sqrt(al * be)) continue;
      rotated = true;
      const double zeta = (be - al) / (2.0 * ga);
      const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
      for (int r = 0; r < 3; ++r) {
        const double bp = B[3 * r + p], bq = B[3 * r + q];
        B[3 * r + p] = c * bp - sn * bq;
        B[3 * r + q] = sn * bp + c * bq;
        const double vp = V[3 * r + p], vq = V[3 * r + q];
        V[3 * r + p] = c * vp - sn * vq;
        V[3 * r + q] = sn * vp + c * vq;
      }
    }
    if (!rotated) break;
  }
}

// The SVD part of Umeyama's method for the 3x3 cross-covariance A (the ICP's update, the trajectory's Sim(3)
// alignment): gs_jacobi3, then the singular values sv (the column norms of B) and the order ord that sorts them
// descending, sv[ord[0]] >= sv[ord[1]] >= sv[ord[2]].  Column ord[k] of B is sigma_k u_k, column ord[k] of V is v_k.
__device__ __forceinline__ void gs_umeyama_svd(const double A[9], double B[9], double V[9], double sv[3], int ord[3]) {
  gs_jacobi3(A, B, V);
  for (int j = 0; j < 3; ++j) {
    ord[j] = j;
    sv[j] = sqrt(B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j]);
  }
  for (int a = 0; a < 3; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (sv[ord[b]] > sv[ord[a]]) { const int t = ord[a]; ord[a] = ord[b]; ord[b] = t; }
}
