// render_eval.cu — quality of rendered views against the keyframes they reproduce: PSNR, SSIM and depth L1 per frame.
// This is not a function of the reference; the definitions are stated in include/goslam_b200.h and restated in
// float64 in oracle/render_eval_oracle.py.
//
//  * one launch over (output tile, frame): a tile is kTH x kTW SSIM positions.  Per channel, the tile's inputs plus
//    the 10-pixel window extent are staged in shared memory, a horizontal then a vertical 11-tap Gaussian pass gives
//    the five moments (mu_x, mu_y, E[x^2], E[y^2], E[xy]) at every position, and the SSIM map is summed over the
//    tile's positions.  The same block sums the squared colour error and the depth terms over the pixels it owns
//    (its tile's rows and columns, extended to the image's last row / column for the last tile row / column), so every
//    pixel is counted once.  Four f64 partials per (frame, tile) go to the workspace.
//  * the moments are filtered in f64: SSIM divides sigma^2 = E[x^2] - mu^2 by sigma_x^2 + sigma_y^2 + C2 with C2 = 9e-4,
//    so in flat regions an f32 rounding of E[x^2] (~1e-7) would move a position's SSIM by ~1e-4.  x^2, y^2 and xy of f32
//    inputs are exact in f64; only the weighted sums round.
//  * a second kernel sums each frame's tile partials in tile order, one block per frame.
//  * every sum has a fixed order (per-thread loops, a shuffle butterfly, warps in order, no atomics): two calls give
//    the same bits, and a frame's results do not depend on the other frames of the call.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kTW = 32;                   // tile width in SSIM positions (one warp's columns)
constexpr int kTH = 16;                   // tile height
constexpr int kWin = 11;                  // Gaussian window
constexpr int kExt = kWin - 1;            // extra input rows / columns a tile reads
constexpr int kSW = kTW + kExt;           // staged columns
constexpr int kSH = kTH + kExt;           // staged rows
constexpr int kSP = kSW + 1;              // staged row pitch (floats); odd, so row-strided lanes hit distinct banks
constexpr int kHP = kTW + 1;              // horizontal-pass row pitch (doubles)
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kHCols = 4;                 // horizontal-pass positions per thread (kSH * kTW / kHCols <= kThreads)
constexpr int kVRows = kTH / kWarps;      // vertical-pass positions per thread: warp w owns rows [w*kVRows, +kVRows)
constexpr int kParts = 4;                 // SSIM sum, squared-error sum, depth |error| sum, depth count
constexpr int kReduceThreads = 128;
constexpr int kMaxFramesPerLaunch = 65535; // gridDim.y
constexpr double kC1 = 0.01 * 0.01;
constexpr double kC2 = 0.03 * 0.03;
static_assert(kSH * (kTW / kHCols) <= kThreads, "one horizontal work item per thread");
static_assert(kVRows * kWarps == kTH, "warps cover the tile's rows");

// exp(-(i-5)^2 / 4.5) normalised to sum 1, in float64 (numpy's values)
__constant__ double kGauss[kWin] = {0.00102838008447911, 0.007598758135239185, 0.03600077212843083,
                                    0.10936068950970002, 0.2130055377112537,   0.26601172486179436,
                                    0.2130055377112537,  0.10936068950970002, 0.03600077212843083,
                                    0.007598758135239185, 0.00102838008447911};

struct Shape {
  int tiles_x, tiles_y;
  int tiles() const { return tiles_x * tiles_y; }
};

Shape shape_of(int H, int W) { return {gs_cdiv(W - kExt, kTW), gs_cdiv(H - kExt, kTH)}; }

bool valid_shape(int K, int H, int W) {
  return K >= 0 && H >= kWin && W >= kWin && (long long)H * W <= 0x7fffffffll;
}

struct RenderMetricsWork {
  double* part;     // [K, tiles, kParts]
};

size_t render_metrics_layout(int K, int H, int W, void* base, RenderMetricsWork* w) {
  GsArena ar(base);
  w->part = ar.take<double>((size_t)std::max(K, 1) * shape_of(H, W).tiles() * kParts);
  return ar.off;
}

// SSIM of one position from its moments m = (mu_x, mu_y, E[x^2], E[y^2], E[xy]); every operation rounded on its own,
// so identical inputs (mu_x = mu_y, E[x^2] = E[y^2] = E[xy] bit for bit) give exactly 1
__device__ __forceinline__ double ssim_at(const double (&m)[5]) {
  const double mx2 = __dmul_rn(m[0], m[0]), my2 = __dmul_rn(m[1], m[1]), mxy = __dmul_rn(m[0], m[1]);
  const double sx = __dsub_rn(m[2], mx2), sy = __dsub_rn(m[3], my2), sxy = __dsub_rn(m[4], mxy);
  const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mxy), kC1), __dadd_rn(__dmul_rn(2.0, sxy), kC2));
  const double den = __dmul_rn(__dadd_rn(__dadd_rn(mx2, my2), kC1), __dadd_rn(__dadd_rn(sx, sy), kC2));
  return __ddiv_rn(num, den);
}

__global__ void __launch_bounds__(kThreads) render_metrics_tile_kernel(
    const float* __restrict__ color, const float* __restrict__ depth, const float* __restrict__ gt_color,
    const float* __restrict__ gt_depth, const uint8_t* __restrict__ mask, int H, int W, int tiles_x, int frame0,
    double* __restrict__ part) {
  __shared__ float xs[2][kSH][kSP];         // one channel of the rendered (0) and reference (1) image
  __shared__ double hb[5][kSH][kHP];        // horizontal pass: the five moments per staged row and position
  __shared__ double red[kWarps][kParts];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int k = frame0 + blockIdx.y;
  const int tiles_y = gridDim.x / tiles_x;
  const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
  const int r0 = ty * kTH, c0 = tx * kTW;
  const int own_r1 = ty == tiles_y - 1 ? H : r0 + kTH;     // the pixels this block owns: [r0, own_r1) x [c0, own_c1)
  const int own_c1 = tx == tiles_x - 1 ? W : c0 + kTW;
  const int Hv = H - kExt, Wv = W - kExt;
  const long long HW = (long long)H * W;
  const float* cr = color + (long long)k * HW * 3;
  const float* cg = gt_color + (long long)k * HW * 3;
  double v[kParts] = {0.0, 0.0, 0.0, 0.0};

  // depth: |d - d_gt| where d_gt is finite and > 0 and the mask, if any, is set
  for (int i = tid; i < kSH * kSW; i += kThreads) {
    const int r = r0 + i / kSW, c = c0 + i % kSW;
    if (r >= own_r1 || c >= own_c1) continue;
    const long long p = (long long)k * HW + (long long)r * W + c;
    const float g = gt_depth[p];
    if (isfinite(g) && g > 0.0f && (!mask || mask[p])) {
      v[2] = __dadd_rn(v[2], fabs(__dsub_rn((double)depth[p], (double)g)));
      v[3] = __dadd_rn(v[3], 1.0);
    }
  }

  for (int ch = 0; ch < 3; ++ch) {
    // stage the channel (zeros past the image: they reach only positions past the valid range); squared error of
    // the owned pixels
    for (int i = tid; i < kSH * kSW; i += kThreads) {
      const int rr = i / kSW, cc = i % kSW;
      const int r = r0 + rr, c = c0 + cc;
      float x = 0.0f, y = 0.0f;
      if (r < H && c < W) {
        const long long p = (long long)r * W + c;
        x = cr[3 * p + ch];
        y = cg[ch * HW + p];
        if (r < own_r1 && c < own_c1) {
          const double d = __dsub_rn((double)x, (double)y);
          v[1] = __dadd_rn(v[1], __dmul_rn(d, d));
        }
      }
      xs[0][rr][cc] = x;
      xs[1][rr][cc] = y;
    }
    __syncthreads();

    // horizontal pass: thread -> (staged row, kHCols consecutive positions)
    if (tid < kSH * (kTW / kHCols)) {
      const int rr = tid % kSH, cb = (tid / kSH) * kHCols;
      double acc[kHCols][5];
#pragma unroll
      for (int o = 0; o < kHCols; ++o)
#pragma unroll
        for (int m = 0; m < 5; ++m) acc[o][m] = 0.0;
#pragma unroll
      for (int j = 0; j < kHCols + kExt; ++j) {
        const double x = xs[0][rr][cb + j], y = xs[1][rr][cb + j];
        const double mo[5] = {x, y, x * x, y * y, x * y};      // products of f32 values: exact
#pragma unroll
        for (int o = 0; o < kHCols; ++o) {
          const int t = j - o;
          if (t >= 0 && t < kWin) {
#pragma unroll
            for (int m = 0; m < 5; ++m) acc[o][m] = __fma_rn(kGauss[t], mo[m], acc[o][m]);
          }
        }
      }
#pragma unroll
      for (int o = 0; o < kHCols; ++o)
#pragma unroll
        for (int m = 0; m < 5; ++m) hb[m][rr][cb + o] = acc[o][m];
    }
    __syncthreads();

    // vertical pass: lane -> column, warp -> kVRows consecutive rows; the SSIM of each valid position
    {
      double acc[kVRows][5];
#pragma unroll
      for (int o = 0; o < kVRows; ++o)
#pragma unroll
        for (int m = 0; m < 5; ++m) acc[o][m] = 0.0;
#pragma unroll
      for (int j = 0; j < kVRows + kExt; ++j) {
        double mo[5];
#pragma unroll
        for (int m = 0; m < 5; ++m) mo[m] = hb[m][warp * kVRows + j][lane];
#pragma unroll
        for (int o = 0; o < kVRows; ++o) {
          const int t = j - o;
          if (t >= 0 && t < kWin) {
#pragma unroll
            for (int m = 0; m < 5; ++m) acc[o][m] = __fma_rn(kGauss[t], mo[m], acc[o][m]);
          }
        }
      }
#pragma unroll
      for (int o = 0; o < kVRows; ++o) {
        if (r0 + warp * kVRows + o < Hv && c0 + lane < Wv) v[0] = __dadd_rn(v[0], ssim_at(acc[o]));
      }
    }
    __syncthreads();      // the next channel overwrites xs and hb
  }

  // block sums: a shuffle butterfly per warp, then the warps in order
#pragma unroll
  for (int m = 0; m < kParts; ++m) v[m] = gs_warp_sum(v[m]);
  if (lane == 0) {
#pragma unroll
    for (int m = 0; m < kParts; ++m) red[warp][m] = v[m];
  }
  __syncthreads();
  if (tid < kParts) {
    double s = red[0][tid];
    for (int w = 1; w < kWarps; ++w) s = __dadd_rn(s, red[w][tid]);
    part[((long long)k * gridDim.x + blockIdx.x) * kParts + tid] = s;
  }
}

// one block per frame: its tiles' partials in tile order, then the four results
__global__ void __launch_bounds__(kReduceThreads) render_metrics_reduce_kernel(
    const double* __restrict__ part, int tiles, int H, int W, double* __restrict__ psnr, double* __restrict__ ssim,
    double* __restrict__ depth_l1, int64_t* __restrict__ depth_count) {
  __shared__ double sh[kParts][kReduceThreads];
  const int k = blockIdx.x;
  const double* p = part + (long long)k * tiles * kParts;
  double v[kParts] = {0.0, 0.0, 0.0, 0.0};
  for (int t = threadIdx.x; t < tiles; t += kReduceThreads) {
#pragma unroll
    for (int m = 0; m < kParts; ++m) v[m] = __dadd_rn(v[m], p[(long long)t * kParts + m]);
  }
  gs_block_sum(v, sh);
  if (threadIdx.x != 0) return;
  const double mse = __ddiv_rn(v[1], 3.0 * (double)H * (double)W);
  psnr[k] = -10.0 * log10(mse);                                           // mse = 0: +inf
  ssim[k] = __ddiv_rn(v[0], 3.0 * (double)(H - kExt) * (double)(W - kExt));
  depth_l1[k] = v[3] > 0.0 ? __ddiv_rn(v[2], v[3]) : nan("");
  depth_count[k] = (int64_t)v[3];
}

}  // namespace

extern "C" {

size_t goslam_render_metrics_workspace_bytes(int K, int H, int W) {
  if (!valid_shape(K, H, W)) return 0;
  RenderMetricsWork w;
  return render_metrics_layout(K, H, W, nullptr, &w);
}

int goslam_render_metrics(const float* color, const float* depth, const float* gt_color, const float* gt_depth,
                          const uint8_t* mask, int K, int H, int W, void* workspace, size_t workspace_bytes,
                          double* psnr, double* ssim, double* depth_l1, int64_t* depth_count, void* stream) {
  if (!valid_shape(K, H, W)) return GOSLAM_EINVAL;
  if (K == 0) return GOSLAM_OK;
  if (!color || !depth || !gt_color || !gt_depth || !psnr || !ssim || !depth_l1 || !depth_count) return GOSLAM_EINVAL;
  RenderMetricsWork w;
  if (!workspace || workspace_bytes < render_metrics_layout(K, H, W, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const Shape s = shape_of(H, W);
  for (int f0 = 0; f0 < K; f0 += kMaxFramesPerLaunch) {
    const dim3 grid((unsigned)s.tiles(), (unsigned)std::min(K - f0, kMaxFramesPerLaunch));
    render_metrics_tile_kernel<<<grid, kThreads, 0, st>>>(color, depth, gt_color, gt_depth, mask, H, W, s.tiles_x, f0,
                                                          w.part);
    GS_CHECK_LAUNCH();
  }
  render_metrics_reduce_kernel<<<(unsigned)K, kReduceThreads, 0, st>>>(w.part, s.tiles(), H, W, psnr, ssim, depth_l1,
                                                                       depth_count);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
