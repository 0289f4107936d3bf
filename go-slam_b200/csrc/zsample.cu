// zsample.cu — per-ray depth sampling of the renderer in one launch.
//
// Replaces the z-sampling half of Renderer.render_batch_ray (src/render.py:99-171): ~25 eager
// [R,S] torch kernels + a torch.sort over [R,72] in the reference.  One warp per ray:
//   far  = min_axis max_side((bound - o) / d) + 0.01, clamped to [0, 1.2 * max(gt_depth)]   (:112-123)
//   near = 0.01 * gt_depth (or 0.01 without a depth prior)                                  (:99-105)
//   n_samples stratified samples in [near, far], jittered by ONE shared perturb_rand[i] per
//   sample index (:143-159); n_surface samples in +-10 % of the sensor depth, or spread over
//   [0.001, max depth] where the sensor has no reading (:125-141); the union sorted (:161-165);
//   dists = successive differences, last one = (far - near) / n_samples                      (:167-170)
// Every value is produced by the same sequence of individually rounded fp32 operations as the
// eager reference (no FMA contraction), so z_vals are bit-identical given the same three small
// tables (the two torch.linspace tables and perturb_rand come from torch so that the RNG stream
// and linspace's own rounding are the reference's).
#include "common.cuh"

namespace {

constexpr int kZWarps = 8;
constexpr int kZMaxS = 128;

__device__ __forceinline__ unsigned f2ord(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// max over gt_depth[R] -> scal[0] as an order-preserving unsigned key (scal zeroed beforehand)
__global__ void __launch_bounds__(256) zs_max_kernel(const float* __restrict__ x, int R, unsigned* scal) {
  float m = -INFINITY;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < R; i += gridDim.x * blockDim.x) m = fmaxf(m, x[i]);
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(scal, f2ord(m));
}

// torch.max / torch.min / torch.clamp propagate NaN
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a) ? a : ((b != b) ? b : fmaxf(a, b)); }
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a) ? a : ((b != b) ? b : fminf(a, b)); }

struct ZArgs {
  const float* rays_o; const float* rays_d; const float* bound; const float* gt_depth;
  const float* t_samples; const float* t_surface; const float* perturb_rand;
  int R, n_samples, n_surface, lindisp;
  float* z_vals; float* dists;
  const unsigned* scal;
};

__device__ __forceinline__ float z_linear(float near, float far, float t, int lindisp) {
  if (!lindisp) return __fadd_rn(near, __fmul_rn(__fsub_rn(far, near), t));
  const float inv_far = __fdiv_rn(1.0f, far), inv_near = __fdiv_rn(1.0f, near);
  return __fdiv_rn(1.0f, __fadd_rn(inv_far, __fmul_rn(__fsub_rn(inv_near, inv_far), t)));
}

__global__ void __launch_bounds__(kZWarps * 32) zs_sample_kernel(const ZArgs a) {
  __shared__ float vals[kZWarps][kZMaxS];
  __shared__ float sorted[kZWarps][kZMaxS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int S = a.n_samples + a.n_surface;
  const bool has_depth = a.gt_depth != nullptr;
  const float gtmax = has_depth ? ord2f(*a.scal) : 0.f;
  float b[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) b[i] = a.bound[i];
  float* v = vals[warp];
  float* s = sorted[warp];

  for (int r = blockIdx.x * kZWarps + warp; r < a.R; r += gridDim.x * kZWarps) {
    float far = INFINITY;
    {
      bool first = true;
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) {
        const float o = a.rays_o[3 * r + ax], d = a.rays_d[3 * r + ax];
        const float t0 = __fdiv_rn(__fsub_rn(b[2 * ax], o), d), t1 = __fdiv_rn(__fsub_rn(b[2 * ax + 1], o), d);
        const float m = nan_max(t0, t1);
        far = first ? m : nan_min(far, m);
        first = false;
      }
      far = __fadd_rn(far, 0.01f);
    }
    float near = 0.01f, gt = 0.f;
    if (has_depth) {
      gt = a.gt_depth[r];
      near = __fmul_rn(gt, 0.01f);
      far = nan_min(nan_max(far, 0.0f), __fmul_rn(gtmax, 1.2f));      // torch.clamp(far, 0, max)
    }
    // stratified samples
    for (int i = lane; i < a.n_samples; i += 32) {
      float z = z_linear(near, far, a.t_samples[i], a.lindisp);
      if (a.perturb_rand) {
        const float zl = i > 0 ? z_linear(near, far, a.t_samples[i - 1], a.lindisp) : z;
        const float zu = i + 1 < a.n_samples ? z_linear(near, far, a.t_samples[i + 1], a.lindisp) : z;
        const float lower = i > 0 ? __fmul_rn(0.5f, __fadd_rn(zl, z)) : z;
        const float upper = i + 1 < a.n_samples ? __fmul_rn(0.5f, __fadd_rn(z, zu)) : z;
        z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), a.perturb_rand[i]));
      }
      v[i] = z;
    }
    // surface-guided samples
    if (a.n_surface > 0) {
      const float valid = gt > 0.f ? 1.0f : 0.0f;
      const float vd = __fmul_rn(gt, valid);
      const float snr = __fmul_rn(0.9f, vd), sfar = __fmul_rn(1.1f, vd);
      const float span_inv = __fsub_rn(gtmax, 0.001f);
      for (int i = lane; i < a.n_surface; i += 32) {
        const float t = a.t_surface[i];
        const float zv = __fadd_rn(snr, __fmul_rn(__fsub_rn(sfar, snr), t));
        const float zi = __fadd_rn(0.001f, __fmul_rn(span_inv, t));
        v[a.n_samples + i] = __fadd_rn(__fmul_rn(zv, valid), __fmul_rn(zi, __fsub_rn(1.0f, valid)));
      }
      __syncwarp();
      // Both lists are normally ascending already (stratified bins; surface offsets grow with t):
      // then the sorted union is a two-way merge, each element's rank by binary search in the
      // other list (ties: the stratified sample first, as a stable sort of the concatenation).
      bool ok = true;
      for (int i = lane; i < S; i += 32) {
        const float x = v[i];
        ok = ok && (x == x);
        if (i + 1 < S && i + 1 != a.n_samples) ok = ok && (x <= v[i + 1]);
      }
      if (__all_sync(0xffffffffu, ok)) {
        const float* su = v + a.n_samples;
        for (int i = lane; i < S; i += 32) {
          const float x = v[i];
          int lo = 0, hi, rank;
          if (i < a.n_samples) {               // surface values strictly below x
            hi = a.n_surface;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (su[mid] < x) lo = mid + 1; else hi = mid; }
            rank = i + lo;
          } else {                             // stratified values <= x
            hi = a.n_samples;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (v[mid] <= x) lo = mid + 1; else hi = mid; }
            rank = (i - a.n_samples) + lo;
          }
          s[rank] = x;
        }
      } else
      // general case — rank sort (ascending, NaN last, ties by position): S <= 128 values, 32 lanes
      for (int i = lane; i < S; i += 32) {
        const float x = v[i];
        const bool xnan = x != x;
        int rank = 0;
        for (int j = 0; j < S; ++j) {
          const float y = v[j];
          const bool ynan = y != y;
          const bool less = xnan ? (!ynan || j < i) : (!ynan && (y < x || (y == x && j < i)));
          rank += less ? 1 : 0;
        }
        s[rank] = x;
      }
    } else {
      __syncwarp();
      for (int i = lane; i < S; i += 32) s[i] = v[i];
    }
    __syncwarp();
    // (far - near) / n_samples: the reference takes the mean of n_samples identical copies of it
    float last;
    if (!a.lindisp) last = __fdiv_rn(__fsub_rn(far, near), (float)a.n_samples);
    else last = __fdiv_rn(1.0f, __fdiv_rn(__fsub_rn(__fdiv_rn(1.0f, near), __fdiv_rn(1.0f, far)), (float)a.n_samples));
    float* zo = a.z_vals + (size_t)r * S;
    float* dd = a.dists + (size_t)r * S;
    for (int i = lane; i < S; i += 32) {
      const float z = s[i];
      zo[i] = z;
      dd[i] = (i + 1 < S) ? __fsub_rn(s[i + 1], z) : last;
    }
    __syncwarp();
  }
}

// one 256-byte block: the batch's largest sensor depth, as order-preserving bits
size_t zs_layout(void* base, unsigned** scal) {
  GsArena ar(base);
  *scal = ar.take<unsigned>(1);
  return ar.off;
}

}  // namespace

extern "C" {

int goslam_sample_z(const float* rays_o, const float* rays_d, const float* bound, const float* gt_depth,
                    const float* t_samples, const float* t_surface, const float* perturb_rand, int R,
                    int n_samples, int n_surface, int lindisp, float* z_vals, float* dists,
                    void* workspace, size_t workspace_bytes, void* stream) {
  if (R < 0 || n_samples < 1 || n_surface < 0 || n_samples + n_surface > kZMaxS) return GOSLAM_EINVAL;
  if (gt_depth == nullptr) n_surface = 0;                 // src/render.py:99-101
  if (n_surface > 0 && t_surface == nullptr) return GOSLAM_EINVAL;
  unsigned* scal;
  if (!workspace || workspace_bytes < zs_layout(workspace, &scal)) return GOSLAM_EWORKSPACE;
  if (R == 0) return GOSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (gt_depth) {
    GS_CUDA(cudaMemsetAsync(scal, 0, sizeof(unsigned), st));
    const int blocks = gs_cdiv(R, 256 * 8) < kNumSms ? gs_cdiv(R, 256 * 8) : kNumSms;
    zs_max_kernel<<<blocks, 256, 0, st>>>(gt_depth, R, scal);
    GS_CHECK_LAUNCH();
  }
  ZArgs a{rays_o, rays_d, bound, gt_depth, t_samples, t_surface, perturb_rand, R, n_samples, n_surface,
          lindisp, z_vals, dists, scal};
  const int want = gs_cdiv(R, kZWarps);
  const int grid = want < kNumSms * 8 ? want : kNumSms * 8;
  zs_sample_kernel<<<grid, kZWarps * 32, 0, st>>>(a);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
