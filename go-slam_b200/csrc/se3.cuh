// se3.cuh — the SE3 subset of lietorch that GO-SLAM's hot path uses, as plain device
// functions.  lietorch's source is absent from the reference snapshot; the algebra is
// pinned by its in-repo CUDA twins (src/lib/droid_kernels.cu:58-175 act/adj/rel/exp,
// :877-895 retraction).  Pose storage: t = (tx,ty,tz), q = (qx,qy,qz,qw); tangent
// xi = (tau, phi); retraction is the LEFT one, T <- exp(xi) * T.
#pragma once
#include <cuda_runtime.h>

struct GsSE3 { float t[3]; float q[4]; };

// Y = R(q) X   (src/lib/droid_kernels.cu:58-68)
__device__ __forceinline__ void gs_rot(const float* q, const float* X, float* Y) {
  const float ux = 2.0f * (q[1] * X[2] - q[2] * X[1]);
  const float uy = 2.0f * (q[2] * X[0] - q[0] * X[2]);
  const float uz = 2.0f * (q[0] * X[1] - q[1] * X[0]);
  Y[0] = X[0] + q[3] * ux + (q[1] * uz - q[2] * uy);
  Y[1] = X[1] + q[3] * uy + (q[2] * ux - q[0] * uz);
  Y[2] = X[2] + q[3] * uz + (q[0] * uy - q[1] * ux);
}

// homogeneous action on (X,Y,Z,d): rotate the first three, add d * t, keep d
// (src/lib/droid_kernels.cu:70-77)
__device__ __forceinline__ void gs_act4(const GsSE3& G, const float* X, float* Y) {
  gs_rot(G.q, X, Y);
  Y[3] = X[3];
  Y[0] += X[3] * G.t[0];
  Y[1] += X[3] * G.t[1];
  Y[2] += X[3] * G.t[2];
}

// dual adjoint applied to a 6-covector (row of a Jacobian): Y = Ad(G)^T X
// (src/lib/droid_kernels.cu:79-94)
__device__ __forceinline__ void gs_adjT(const GsSE3& G, const float* X, float* Y) {
  const float qi[4] = {-G.q[0], -G.q[1], -G.q[2], G.q[3]};
  gs_rot(qi, X, Y);
  gs_rot(qi, X + 3, Y + 3);
  const float u[3] = {G.t[2] * X[1] - G.t[1] * X[2],
                      G.t[0] * X[2] - G.t[2] * X[0],
                      G.t[1] * X[0] - G.t[0] * X[1]};
  float v[3];
  gs_rot(qi, u, v);
  Y[3] += v[0]; Y[4] += v[1]; Y[5] += v[2];
}

// G_ij = G_j * G_i^{-1}   (src/lib/droid_kernels.cu:96-107)
__device__ __forceinline__ void gs_rel(const float* ti, const float* qi, const float* tj,
                                       const float* qj, GsSE3& G) {
  G.q[0] = -qj[3] * qi[0] + qj[0] * qi[3] - qj[1] * qi[2] + qj[2] * qi[1];
  G.q[1] = -qj[3] * qi[1] + qj[1] * qi[3] - qj[2] * qi[0] + qj[0] * qi[2];
  G.q[2] = -qj[3] * qi[2] + qj[2] * qi[3] - qj[0] * qi[1] + qj[1] * qi[0];
  G.q[3] =  qj[3] * qi[3] + qj[0] * qi[0] + qj[1] * qi[1] + qj[2] * qi[2];
  float r[3];
  gs_rot(G.q, ti, r);
  G.t[0] = tj[0] - r[0];
  G.t[1] = tj[1] - r[1];
  G.t[2] = tj[2] - r[2];
}

// relative pose of an edge; ii == jj is the fixed stereo baseline
// (src/lib/droid_kernels.cu:218-249, src/geom/projective_ops.py:124)
__device__ __forceinline__ void gs_edge_pose(const float* poses, int ix, int jx, GsSE3& G) {
  if (ix == jx) {
    G.t[0] = -0.1f; G.t[1] = 0.f; G.t[2] = 0.f;
    G.q[0] = 0.f; G.q[1] = 0.f; G.q[2] = 0.f; G.q[3] = 1.f;
  } else {
    const float* pi = poses + 7 * (size_t)ix;
    const float* pj = poses + 7 * (size_t)jx;
    gs_rel(pi, pi + 3, pj, pj + 3, G);
  }
}

__device__ __forceinline__ void gs_cross_inplace(const float* a, float* b) {
  const float x = a[1] * b[2] - a[2] * b[1];
  const float y = a[2] * b[0] - a[0] * b[2];
  const float z = a[0] * b[1] - a[1] * b[0];
  b[0] = x; b[1] = y; b[2] = z;
}

// exp: se3 -> SE3 (src/lib/droid_kernels.cu:110-175), same small-angle branches.
__device__ __forceinline__ void gs_exp(const float* xi, float* t, float* q) {
  const float* phi = xi + 3;
  const float th2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
  const float th4 = th2 * th2;
  const float th = sqrtf(th2);
  float imag, real;
  if (th2 < 1e-8f) {
    imag = 0.5f - (1.0f / 48.0f) * th2 + (1.0f / 3840.0f) * th4;
    real = 1.0f - (1.0f / 8.0f) * th2 + (1.0f / 384.0f) * th4;
  } else {
    imag = sinf(0.5f * th) / th;
    real = cosf(0.5f * th);
  }
  q[0] = imag * phi[0]; q[1] = imag * phi[1]; q[2] = imag * phi[2]; q[3] = real;

  float tau[3] = {xi[0], xi[1], xi[2]};
  t[0] = tau[0]; t[1] = tau[1]; t[2] = tau[2];
  if (th > 1e-4f) {
    const float a = (1.0f - cosf(th)) / th2;
    gs_cross_inplace(phi, tau);
    t[0] += a * tau[0]; t[1] += a * tau[1]; t[2] += a * tau[2];
    const float b = (th - sinf(th)) / (th * th2);
    gs_cross_inplace(phi, tau);
    t[0] += b * tau[0]; t[1] += b * tau[1]; t[2] += b * tau[2];
  }
}

// log: SE3 -> se3, the inverse of gs_exp with lietorch.SE3.log's closed form and switches (go-slam_b200/lietorch.py):
// the rotation vector from the quaternion in the atan2 form that stays continuous for qw < 0 (series below
// |qv|^2 = 1e-12), then tau = V(phi)^-1 t, left as t at or below theta = 1e-4 where gs_exp leaves t = tau.
__device__ __forceinline__ void gs_log(const float* t, const float* q, float* xi) {
  const float n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2];
  const float w = q[3];
  float two_atan;
  if (n2 < 1e-12f) {
    two_atan = 2.0f / w - (2.0f / 3.0f) * n2 / (w * w * w);
  } else {
    const float n = sqrtf(n2);
    const float sgn = w < 0.0f ? -1.0f : 1.0f;
    two_atan = 2.0f * sgn * atan2f(n, w * sgn) / n;
  }
  float* phi = xi + 3;
  phi[0] = two_atan * q[0]; phi[1] = two_atan * q[1]; phi[2] = two_atan * q[2];
  const float th = sqrtf(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]);
  xi[0] = t[0]; xi[1] = t[1]; xi[2] = t[2];
  if (th > 1e-4f) {
    const float half = 0.5f * th;
    const float coef = (1.0f - th * cosf(half) / (2.0f * sinf(half))) / (th * th);
    float c[3] = {t[0], t[1], t[2]};
    gs_cross_inplace(phi, c);                       // c1 = phi x t
    xi[0] -= 0.5f * c[0]; xi[1] -= 0.5f * c[1]; xi[2] -= 0.5f * c[2];
    gs_cross_inplace(phi, c);                       // c2 = phi x c1
    xi[0] += coef * c[0]; xi[1] += coef * c[1]; xi[2] += coef * c[2];
  }
}

// T1 = exp(xi) * T   (src/lib/droid_kernels.cu:877-895)
__device__ __forceinline__ void gs_retr(const float* xi, const float* t, const float* q,
                                        float* t1, float* q1) {
  float dt[3], dq[4];
  gs_exp(xi, dt, dq);
  q1[0] = dq[3] * q[0] + dq[0] * q[3] + dq[1] * q[2] - dq[2] * q[1];
  q1[1] = dq[3] * q[1] + dq[1] * q[3] + dq[2] * q[0] - dq[0] * q[2];
  q1[2] = dq[3] * q[2] + dq[2] * q[3] + dq[0] * q[1] - dq[1] * q[0];
  q1[3] = dq[3] * q[3] - dq[0] * q[0] - dq[1] * q[1] - dq[2] * q[2];
  gs_rot(dq, t, t1);
  t1[0] += dt[0]; t1[1] += dt[1]; t1[2] += dt[2];
}
