// fill.cu — PoseTrajectoryFiller.__fill's pose interpolation and video hand-over
// (src/trajectory_filler.py:38-63, src/depth_video.py:85-120) as one launch per chunk.
//
// One block per frame of the chunk.  The block counts the keyframe timestamps ts[0:N] that are <= t with
// __syncthreads_count (the reference's `ts[ts<=t].shape[0] - 1`, a count over every entry, not a search), thread 0
// interpolates the pose in the reference's operation order, and the block writes the frame's 1/8-resolution disps.
#include "common.cuh"
#include "se3.cuh"

namespace {

constexpr int kFillThreads = 256;

__global__ void __launch_bounds__(kFillThreads)
fill_interpolate_kernel(float* __restrict__ timestamp, float* __restrict__ poses, float* __restrict__ intrinsics,
                        float* __restrict__ disps, float* __restrict__ disps_sens, int N, const float* __restrict__ tt,
                        const float* __restrict__ intr_full, const float* __restrict__ depth, int H, int W,
                        int64_t* __restrict__ t0_out, int64_t* __restrict__ t1_out) {
  const int k = blockIdx.x;
  const int row = N + k;
  const float t = tt[k];
  int count = 0;
  for (int base = 0; base < N; base += kFillThreads) {
    const int i = base + threadIdx.x;
    count += __syncthreads_count(i < N && timestamp[i] <= t);
  }
  // a frame before the first keyframe (count 0) brackets as keyframe 0 here; the Python layer rejects it first
  const int t0 = count > 0 ? count - 1 : 0;
  const int t1 = t0 < N - 1 ? t0 + 1 : t0;

  if (threadIdx.x == 0) {
    const float ts0 = timestamp[t0];
    const float dt = timestamp[t1] - ts0 + 1e-3f;
    const float* P0 = poses + 7 * (size_t)t0;
    const float* P1 = poses + 7 * (size_t)t1;
    // P0^-1 = (-R(q0^*) t0, q0^*), then dP = P1 * P0^-1 (lietorch: Ps[t1] * Ps[t0].inv())
    const float qi[4] = {-P0[3], -P0[4], -P0[5], P0[6]};
    float ti[3];
    gs_rot(qi, P0, ti);
    ti[0] = -ti[0]; ti[1] = -ti[1]; ti[2] = -ti[2];
    const float* q1 = P1 + 3;
    float dq[4], dtr[3], r[3];
    dq[0] = q1[3] * qi[0] + q1[0] * qi[3] + q1[1] * qi[2] - q1[2] * qi[1];
    dq[1] = q1[3] * qi[1] + q1[1] * qi[3] + q1[2] * qi[0] - q1[0] * qi[2];
    dq[2] = q1[3] * qi[2] + q1[2] * qi[3] + q1[0] * qi[1] - q1[1] * qi[0];
    dq[3] = q1[3] * qi[3] - q1[0] * qi[0] - q1[1] * qi[1] - q1[2] * qi[2];
    gs_rot(q1, ti, r);
    dtr[0] = P1[0] + r[0]; dtr[1] = P1[1] + r[1]; dtr[2] = P1[2] + r[2];
    float xi[6];
    gs_log(dtr, dq, xi);
    const float s = t - ts0;
#pragma unroll
    for (int j = 0; j < 6; ++j) xi[j] = (xi[j] / dt) * s;     // v = log(dP) / dt, then w = v * (t - ts[t0])
    float* G = poses + 7 * (size_t)row;
    gs_retr(xi, P0, P0 + 3, G, G + 3);                         // G = exp(w) * P[t0]
    timestamp[row] = t;
#pragma unroll
    for (int j = 0; j < 4; ++j) intrinsics[4 * (size_t)row + j] = intr_full[4 * k + j] / 8.0f;
    t0_out[k] = t0;
    t1_out[k] = t1;
  }

  // disps = 1; with a depth map disps_sens = where(d > 0, 1 / d, d) at [3::8, 3::8] and disps = disps_sens
  const int h8 = H / 8, w8 = W / 8;
  float* drow = disps + (size_t)row * h8 * w8;
  float* srow = disps_sens + (size_t)row * h8 * w8;
  const float* dep = depth != nullptr ? depth + (size_t)k * H * W : nullptr;
  for (int p = threadIdx.x; p < h8 * w8; p += kFillThreads) {
    if (dep == nullptr) {
      drow[p] = 1.0f;
    } else {
      const int y = p / w8, x = p - y * w8;
      const float d = dep[(size_t)(3 + 8 * y) * W + 3 + 8 * x];
      const float v = d > 0.0f ? 1.0f / d : d;
      srow[p] = v;
      drow[p] = v;
    }
  }
}

}  // namespace

extern "C" {

int goslam_fill_interpolate(float* timestamp, float* poses, float* intrinsics, float* disps, float* disps_sens, int N,
                            int M, const float* tt, const float* intr_full, const float* depth, int H, int W,
                            int64_t* t0, int64_t* t1, void* stream) {
  if (N < 1 || M < 0 || M > 65535 || H <= 0 || W <= 0 || H % 8 || W % 8) return GOSLAM_EINVAL;
  if (M == 0) return GOSLAM_OK;
  fill_interpolate_kernel<<<M, kFillThreads, 0, (cudaStream_t)stream>>>(
      timestamp, poses, intrinsics, disps, disps_sens, N, tt, intr_full, depth, H, W, t0, t1);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
