// mapping.cu — the mapping process's frame hand-over and ray sampling (src/mapping.py:151-300,
// src/depth_video.py:153-173, src/nerf_func.py:115-221) for sm_90a.
//
// snapshot (once per Mapper.__call__, under the video's mapping lock):
//   count   one block per (1024-pixel tile, frame): the tile's number of masked pixels
//   scan    one block per frame: exclusive tile prefixes, N_f, and the update_priority decay
//   emit    one block per (tile, frame): the tile's masked pixels as compact records in raster order
// rays (once per training iteration): one launch for the whole concatenated batch.
// all rays (render_img): every pixel of one image in raster order, the same per-pixel arithmetic.
// camera refinement (mapping.BA, src/mapping.py:173-194, src/nerf_func.py:44-112):
//   c2w_to_quadt  one thread per matrix: Rt_to_quaternion's (w, x, y, z, t) by Shepperd's method in f64, w >= 0
//   pose rays     the ray batch with each entry's [R | t] taken from its quaternion-translation leaf (quad2rotation)
//   pose backward one block per entry: G = sum_r g_d[r] dirs[r]^T and sum_r g_o[r] in f64 with a fixed reduction
//                 order, then the chain rule through quad2rotation; no atomics, independent of the launch chunking
#include <cub/cub.cuh>

#include "common.cuh"

namespace {

constexpr int kTile = 1024;                 // pixels per snapshot tile
constexpr int kSnapThreads = 256;           // 4 consecutive pixels per thread
constexpr int kPixPerThread = kTile / kSnapThreads;
constexpr int kMaxEntries = 64;             // frame-list entries per ray launch (longer lists launch in chunks)
constexpr int kRayThreads = 256;
constexpr long long kMaxPixels = 1 << 26;   // per frame; pixel ids and per-frame offsets stay in int32

struct SnapWork {
  int* tile_count;   // [F, T]
  int* tile_off;     // [F, T]
  int* pix;          // [F, H*W]  pixel id y*W + x, frame f's records at [f*H*W, f*H*W + N_f)
  float4* rec;       // [F, H*W]  (r, g, b, depth)
};

int num_tiles(long long hw) { return (int)((hw + kTile - 1) / kTile); }

size_t snap_layout(int F, long long hw, const void* base, SnapWork* w) {
  const size_t ft = (size_t)F * num_tiles(hw), fp = (size_t)F * hw;
  GsArena ar(base);
  w->tile_count = ar.take<int>(ft);
  w->tile_off = ar.take<int>(ft);
  w->pix = ar.take<int>(fp);
  w->rec = ar.take<float4>(fp);
  return ar.off;
}

bool snap_shape_ok(int F, int H, int W) {
  return F >= 0 && F <= 65535 && H > 0 && W > 0 && (long long)H * W <= kMaxPixels;
}

// the reference's `mask.reshape(-1).bool()`: every non-zero value (NaN included) selects the pixel
__device__ __forceinline__ bool selected(float m) { return m != 0.0f; }

__global__ void __launch_bounds__(kSnapThreads) snapshot_count_kernel(const float* __restrict__ mask, const int* __restrict__ frames,
                                                                       int buffer, int hw, int T, int* __restrict__ tile_count) {
  const int t = blockIdx.x, f = blockIdx.y;
  const int frame = frames[f];
  int n = 0;
  if (frame >= 0 && frame < buffer) {
    const float* m = mask + (size_t)frame * hw;
    const int p0 = t * kTile + threadIdx.x * kPixPerThread;
#pragma unroll
    for (int j = 0; j < kPixPerThread; ++j)
      if (p0 + j < hw && selected(__ldg(m + p0 + j))) ++n;
  }
  typedef cub::BlockReduce<int, kSnapThreads> Reduce;
  __shared__ typename Reduce::TempStorage tmp;
  n = Reduce(tmp).Sum(n);
  if (threadIdx.x == 0) tile_count[(size_t)f * T + t] = n;
}

// one block per frame: tile prefixes and N_f; thread 0 multiplies the frame's priority by decay once per occurrence,
// one rounded multiply at a time, as the reference's `update_priority[index] *= decay` per get_mapping_item call
__global__ void __launch_bounds__(kSnapThreads) snapshot_scan_kernel(const int* __restrict__ tile_count, int T,
                                                                      const int* __restrict__ frames,
                                                                      const int* __restrict__ occurrences, int buffer,
                                                                      float decay, float* __restrict__ update_priority,
                                                                      int* __restrict__ tile_off, int* __restrict__ counts) {
  const int f = blockIdx.x;
  typedef cub::BlockScan<int, kSnapThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  int carry = 0;
  for (int base = 0; base < T; base += kSnapThreads) {
    const int t = base + threadIdx.x;
    const int c = t < T ? tile_count[(size_t)f * T + t] : 0;
    int pre, total;
    Scan(tmp).ExclusiveSum(c, pre, total);
    if (t < T) tile_off[(size_t)f * T + t] = carry + pre;
    carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    counts[f] = carry;
    const int frame = frames[f];
    if (frame >= 0 && frame < buffer) {
      float p = update_priority[frame];
      for (int k = 0; k < occurrences[f]; ++k) p = __fmul_rn(p, decay);
      update_priority[frame] = p;
    }
  }
}

__global__ void __launch_bounds__(kSnapThreads) snapshot_emit_kernel(const float* __restrict__ images, const float* __restrict__ mask,
                                                                      const float* __restrict__ disps, const int* __restrict__ frames,
                                                                      int buffer, int hw, int T, const int* __restrict__ tile_off,
                                                                      int* __restrict__ pix, float4* __restrict__ rec) {
  const int t = blockIdx.x, f = blockIdx.y;
  const int frame = frames[f];
  const bool live = frame >= 0 && frame < buffer;
  const int p0 = t * kTile + threadIdx.x * kPixPerThread;
  const float* m = mask + (size_t)(live ? frame : 0) * hw;
  bool sel[kPixPerThread];
  int n = 0;
#pragma unroll
  for (int j = 0; j < kPixPerThread; ++j) {
    sel[j] = live && p0 + j < hw && selected(__ldg(m + p0 + j));
    n += sel[j];
  }
  typedef cub::BlockScan<int, kSnapThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  int pre;
  Scan(tmp).ExclusiveSum(n, pre);
  if (!live) return;
  size_t o = (size_t)f * hw + tile_off[(size_t)f * T + t] + pre;
  const float* img = images + (size_t)frame * 3 * hw;
  const float* dsp = disps + (size_t)frame * hw;
#pragma unroll
  for (int j = 0; j < kPixPerThread; ++j) {
    if (!sel[j]) continue;
    const int p = p0 + j;
    // depth = 1.0 / (disp + 1e-7): torch adds the f32 scalar, then `1.0 / x` is reciprocal(x) * 1.0
    const float depth = __fdiv_rn(1.0f, __fadd_rn(__ldg(dsp + p), 1e-7f));
    pix[o] = p;
    rec[o] = make_float4(__ldg(img + p), __ldg(img + hw + p), __ldg(img + 2 * hw + p), depth);
    ++o;
  }
}

struct Intr { float cx, cy, rfx, rfy; };

// the ray of pixel (x, y) under the pose m = rows of [R | t] (row stride 4: a row-major 4x4 c2w, or a 3x4 in
// registers):
//   dirs = ((x - cx) * rfx, (y - cy) * rfy, 1) with cx = (float)cx and rfx = (float)(1.0 / fx) — torch's CUDA true
//   division by a Python scalar multiplies by the reciprocal, taken in double and rounded to f32 (measured on an H100
//   with torch 2.11: bit-identical, where 1.0f / (float)fx and a true f32 division both differ);
//   rays_d[r] = (dirs.x * R[r][0] + dirs.y * R[r][1]) + R[r][2], every product and sum rounded separately (no FMA),
//   the order documented in the header; rays_o = t(c2w).
__device__ __forceinline__ void pixel_dirs(float x, float y, const Intr& in, float* dx, float* dy) {
  *dx = __fmul_rn(__fsub_rn(x, in.cx), in.rfx);
  *dy = __fmul_rn(__fsub_rn(y, in.cy), in.rfy);
}

__device__ __forceinline__ void pixel_ray(float x, float y, const float* m, const Intr& in, float* __restrict__ o,
                                          float* __restrict__ d) {
  float dx, dy;
  pixel_dirs(x, y, in, &dx, &dy);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float* row = m + 4 * r;
    d[r] = __fadd_rn(__fadd_rn(__fmul_rn(dx, row[0]), __fmul_rn(dy, row[1])), row[2]);
    o[r] = row[3];
  }
}

// quad2rotation (src/nerf_func.py:44-66) with the reference's expressions, every f32 operation rounded on its own:
// two_s = 2 / (((r^2 + i^2) + j^2) + k^2), R00 = 1 - two_s (j^2 + k^2), R01 = two_s (i j - k r), ...; m = [R | t]
__device__ __forceinline__ void quadt_pose(const float* __restrict__ q, float* m) {
  const float r = __ldg(q), i = __ldg(q + 1), j = __ldg(q + 2), k = __ldg(q + 3);
  const float rr = __fmul_rn(r, r), ii = __fmul_rn(i, i), jj = __fmul_rn(j, j), kk = __fmul_rn(k, k);
  const float two_s = __fdiv_rn(2.0f, __fadd_rn(__fadd_rn(__fadd_rn(rr, ii), jj), kk));
  const float ij = __fmul_rn(i, j), ik = __fmul_rn(i, k), jk = __fmul_rn(j, k);
  const float kr = __fmul_rn(k, r), jr = __fmul_rn(j, r), ir = __fmul_rn(i, r);
  m[0] = __fsub_rn(1.0f, __fmul_rn(two_s, __fadd_rn(jj, kk)));
  m[1] = __fmul_rn(two_s, __fsub_rn(ij, kr));
  m[2] = __fmul_rn(two_s, __fadd_rn(ik, jr));
  m[4] = __fmul_rn(two_s, __fadd_rn(ij, kr));
  m[5] = __fsub_rn(1.0f, __fmul_rn(two_s, __fadd_rn(ii, kk)));
  m[6] = __fmul_rn(two_s, __fsub_rn(jk, ir));
  m[8] = __fmul_rn(two_s, __fsub_rn(ik, jr));
  m[9] = __fmul_rn(two_s, __fadd_rn(jk, ir));
  m[10] = __fsub_rn(1.0f, __fmul_rn(two_s, __fadd_rn(ii, jj)));
  m[3] = __ldg(q + 4);
  m[7] = __ldg(q + 5);
  m[11] = __ldg(q + 6);
}

struct RayEntries {
  int n;
  int slot[kMaxEntries];       // snapshot slot of the entry's frame
  int draw[kMaxEntries];       // > 0: that many random records (indices from `draws`); 0: all records in raster order
  int out_off[kMaxEntries];    // first output row, relative to the launch
  int rand_off[kMaxEntries];   // first index in `draws`
  int count[kMaxEntries];      // N_f of the slot
};

// the last entry starting at or before row i (empty entries share their successor's start)
__device__ __forceinline__ int entry_of(const RayEntries& e, int i) {
  int lo = 0, hi = e.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (e.out_off[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// the snapshot record (index into pix / rec) of row j of entry b
__device__ __forceinline__ size_t record_of(const RayEntries& e, int b, int j, int hw,
                                            const long long* __restrict__ draws) {
  long long k = j;
  if (e.draw[b] > 0) {
    k = __ldg(draws + e.rand_off[b] + j);              // torch.randint(N, (n_rays,)).clamp(0, N - 1)
    k = k < 0 ? 0 : (k > e.count[b] - 1 ? e.count[b] - 1 : k);
  }
  return (size_t)e.slot[b] * hw + k;
}

// kQuadt false: pose = c2w [F,4,4] indexed by the entry's slot; true: pose = quadt [n,7] indexed by the entry
template <bool kQuadt>
__global__ void __launch_bounds__(kRayThreads) ray_batch_kernel(const __grid_constant__ RayEntries e, int R, int hw, int W,
                                                                 const int* __restrict__ pix, const float4* __restrict__ rec,
                                                                 const float* __restrict__ pose, const long long* __restrict__ draws,
                                                                 Intr in, float* __restrict__ rays_o, float* __restrict__ rays_d,
                                                                 float* __restrict__ depth, float* __restrict__ color) {
  const int i = blockIdx.x * kRayThreads + threadIdx.x;
  if (i >= R) return;
  const int lo = entry_of(e, i);
  const size_t r = record_of(e, lo, i - e.out_off[lo], hw, draws);
  const int p = __ldg(pix + r);
  const float4 v = __ldg(rec + r);
  float o[3], d[3];
  if constexpr (kQuadt) {
    float m[12];
    quadt_pose(pose + 7 * lo, m);
    pixel_ray((float)(p % W), (float)(p / W), m, in, o, d);
  } else {
    const float* c = pose + 16 * e.slot[lo];
    float m[12];
#pragma unroll
    for (int t = 0; t < 12; ++t) m[t] = __ldg(c + t);
    pixel_ray((float)(p % W), (float)(p / W), m, in, o, d);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    rays_o[3 * (size_t)i + c] = o[c];
    rays_d[3 * (size_t)i + c] = d[c];
  }
  depth[i] = v.w;
  color[3 * (size_t)i + 0] = v.x;
  color[3 * (size_t)i + 1] = v.y;
  color[3 * (size_t)i + 2] = v.z;
}

constexpr int kPoseBwdThreads = 256;

// one block per entry b: acc = (G[3][3] row-major, g_t[3]) with G[a][c] = sum_r g_d[r][a] dirs[r][c], summed in f64,
// each thread over rows tid, tid + 256, ... in order, then a fixed butterfly per warp and warp 0 over the 8 warps in
// order.  Thread 0 takes the chain rule through quad2rotation in f64 and writes d_quadt[b] (zeros for an empty entry).
// R = I + s A(q) with s = 2 / |q|^2 (|q| need not be 1): dL/dq_m = -s^2 q_m <G, A> + s <G, dA/dq_m>.
__global__ void __launch_bounds__(kPoseBwdThreads) pose_rays_backward_kernel(
    const __grid_constant__ RayEntries e, int hw, int W, const int* __restrict__ pix, const float* __restrict__ quadt,
    const long long* __restrict__ draws, Intr in, const float* __restrict__ d_rays_o, const float* __restrict__ d_rays_d,
    float* __restrict__ d_quadt) {
  const int b = blockIdx.x;
  const int rows = e.draw[b] > 0 ? e.draw[b] : e.count[b];
  double acc[12];
#pragma unroll
  for (int t = 0; t < 12; ++t) acc[t] = 0.0;
  for (int j = threadIdx.x; j < rows; j += kPoseBwdThreads) {
    const int p = __ldg(pix + record_of(e, b, j, hw, draws));
    float dx, dy;
    pixel_dirs((float)(p % W), (float)(p / W), in, &dx, &dy);
    const size_t row = 3 * ((size_t)e.out_off[b] + j);
    const double dir[3] = {(double)dx, (double)dy, 1.0};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double gd = (double)__ldg(d_rays_d + row + a);
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[3 * a + c] += gd * dir[c];
      acc[9 + a] += (double)__ldg(d_rays_o + row + a);
    }
  }
#pragma unroll
  for (int t = 0; t < 12; ++t)
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc[t] += __shfl_xor_sync(0xffffffffu, acc[t], off);
  __shared__ double part[kPoseBwdThreads / 32][12];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
#pragma unroll
    for (int t = 0; t < 12; ++t) part[warp][t] = acc[t];
  __syncthreads();
  if (threadIdx.x != 0) return;
  double G[12];
#pragma unroll
  for (int t = 0; t < 12; ++t) {
    double v = part[0][t];
    for (int w = 1; w < kPoseBwdThreads / 32; ++w) v += part[w][t];
    G[t] = v;
  }
  const float* q = quadt + 7 * b;
  const double r = __ldg(q), i = __ldg(q + 1), j = __ldg(q + 2), k = __ldg(q + 3);
  const double s = 2.0 / (r * r + i * i + j * j + k * k);
  // A with R = I + s A, row-major
  const double A[9] = {-(j * j + k * k), i * j - k * r, i * k + j * r,
                       i * j + k * r, -(i * i + k * k), j * k - i * r,
                       i * k - j * r, j * k + i * r, -(i * i + j * j)};
  double GA = 0.0;
#pragma unroll
  for (int t = 0; t < 9; ++t) GA += G[t] * A[t];
  const double dr = -k * G[1] + j * G[2] + k * G[3] - i * G[5] - j * G[6] + i * G[7];
  const double di = j * G[1] + k * G[2] + j * G[3] - 2.0 * i * G[4] - r * G[5] + k * G[6] + r * G[7] - 2.0 * i * G[8];
  const double dj = -2.0 * j * G[0] + i * G[1] + r * G[2] + i * G[3] + k * G[5] - r * G[6] + k * G[7] - 2.0 * j * G[8];
  const double dk = -2.0 * k * G[0] - r * G[1] + i * G[2] + r * G[3] - 2.0 * k * G[4] + j * G[5] + i * G[6] + j * G[7];
  const double ss = s * s * GA;
  float* out = d_quadt + 7 * b;
  out[0] = (float)(s * dr - ss * r);
  out[1] = (float)(s * di - ss * i);
  out[2] = (float)(s * dj - ss * j);
  out[3] = (float)(s * dk - ss * k);
  out[4] = (float)G[9];
  out[5] = (float)G[10];
  out[6] = (float)G[11];
}

// Rt_to_quaternion(c2w, Tquad=False) per matrix: Shepperd's method in f64 (the largest of 1 + trace and the three
// 1 + 2 R_aa - trace takes the square root, so rotations near 180 degrees keep their accuracy), normalised, sign fixed
// to w >= 0, rounded to f32; then the translation
__global__ void __launch_bounds__(kRayThreads) c2w_to_quadt_kernel(const float* __restrict__ c2w, int n,
                                                                    float* __restrict__ quadt) {
  const int b = blockIdx.x * kRayThreads + threadIdx.x;
  if (b >= n) return;
  const float* m = c2w + 16 * (size_t)b;
  double R[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) R[a][c] = (double)__ldg(m + 4 * a + c);
  const double tr = R[0][0] + R[1][1] + R[2][2];
  double w, x, y, z;
  if (tr >= R[0][0] && tr >= R[1][1] && tr >= R[2][2]) {
    const double h = sqrt(1.0 + tr), f = 0.5 / h;
    w = 0.5 * h; x = (R[2][1] - R[1][2]) * f; y = (R[0][2] - R[2][0]) * f; z = (R[1][0] - R[0][1]) * f;
  } else if (R[0][0] >= R[1][1] && R[0][0] >= R[2][2]) {
    const double h = sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]), f = 0.5 / h;
    x = 0.5 * h; w = (R[2][1] - R[1][2]) * f; y = (R[0][1] + R[1][0]) * f; z = (R[0][2] + R[2][0]) * f;
  } else if (R[1][1] >= R[2][2]) {
    const double h = sqrt(1.0 - R[0][0] + R[1][1] - R[2][2]), f = 0.5 / h;
    y = 0.5 * h; w = (R[0][2] - R[2][0]) * f; x = (R[0][1] + R[1][0]) * f; z = (R[1][2] + R[2][1]) * f;
  } else {
    const double h = sqrt(1.0 - R[0][0] - R[1][1] + R[2][2]), f = 0.5 / h;
    z = 0.5 * h; w = (R[1][0] - R[0][1]) * f; x = (R[0][2] + R[2][0]) * f; y = (R[1][2] + R[2][1]) * f;
  }
  const double nrm = sqrt(w * w + x * x + y * y + z * z);
  const double sg = (w < 0.0 ? -1.0 : 1.0) / nrm;
  float* out = quadt + 7 * (size_t)b;
  out[0] = (float)(w * sg);
  out[1] = (float)(x * sg);
  out[2] = (float)(y * sg);
  out[3] = (float)(z * sg);
  out[4] = __ldg(m + 3);
  out[5] = __ldg(m + 7);
  out[6] = __ldg(m + 11);
}

__global__ void __launch_bounds__(kRayThreads) all_rays_kernel(const float* __restrict__ c2w, int hw, int W, Intr in,
                                                                float* __restrict__ rays_o, float* __restrict__ rays_d) {
  const int i = blockIdx.x * kRayThreads + threadIdx.x;
  if (i >= hw) return;
  float m[12], o[3], d[3];
#pragma unroll
  for (int t = 0; t < 12; ++t) m[t] = __ldg(c2w + t);
  pixel_ray((float)(i % W), (float)(i / W), m, in, o, d);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    rays_o[3 * (size_t)i + c] = o[c];
    rays_d[3 * (size_t)i + c] = d[c];
  }
}

// the f32 values torch's CUDA kernels use for `(x - cx) / fx` with Python-float cx, fx: cx rounded to f32 (the
// subtraction), the reciprocal 1.0 / fx in double rounded to f32 (the division)
Intr make_intr(double fx, double fy, double cx, double cy) {
  Intr in;
  in.cx = (float)cx;
  in.cy = (float)cy;
  in.rfx = (float)(1.0 / fx);
  in.rfy = (float)(1.0 / fy);
  return in;
}

// the entry table's checks (before anything touches CUDA): sets R = the batch's rows and D = the draws it reads
int check_entries(int F, long long hw, int n_entries, const int* slots, const int* counts, const int* draw,
                  int64_t n_draws, int64_t max_rays, long long* R, long long* D) {
  if (n_entries < 0 || n_draws < 0 || max_rays < 0) return GOSLAM_EINVAL;
  if (n_entries > 0 && (!slots || !counts || !draw)) return GOSLAM_EINVAL;
  *R = *D = 0;
  for (int i = 0; i < n_entries; ++i) {
    if (slots[i] < 0 || slots[i] >= F || counts[i] < 0 || counts[i] > hw || draw[i] < 0 || (draw[i] > 0 && counts[i] == 0))
      return GOSLAM_EINVAL;
    *R += draw[i] > 0 ? draw[i] : counts[i];
    *D += draw[i];
  }
  if (*R > max_rays || *D > n_draws || *R > INT32_MAX) return GOSLAM_EINVAL;
  return GOSLAM_OK;
}

// the table of entries [b, b + 64) (fewer at the end); r, d = that chunk's rows and draws
RayEntries chunk_entries(int b, int n_entries, const int* slots, const int* counts, const int* draw, int* r, int* d) {
  RayEntries e;
  e.n = n_entries - b < kMaxEntries ? n_entries - b : kMaxEntries;
  *r = *d = 0;
  for (int i = 0; i < e.n; ++i) {
    e.slot[i] = slots[b + i];
    e.draw[i] = draw[b + i];
    e.count[i] = counts[b + i];
    e.out_off[i] = *r;
    e.rand_off[i] = *d;
    *r += e.draw[i] > 0 ? e.draw[i] : e.count[i];
    *d += e.draw[i];
  }
  return e;
}

// the ray batch of goslam_mapping_rays (kQuadt false: pose = c2w per slot) or goslam_mapping_pose_rays (true: pose =
// quadt per entry), after the checks
template <bool kQuadt>
int launch_ray_batch(const void* workspace, size_t workspace_bytes, int F, int H, int W, const float* pose,
                     const int64_t* draws, int64_t n_draws, int n_entries, const int* slots, const int* counts,
                     const int* draw, double fx, double fy, double cx, double cy, float* rays_o, float* rays_d,
                     float* depth, float* color, int64_t max_rays, void* stream) {
  if (!snap_shape_ok(F, H, W) || F == 0) return GOSLAM_EINVAL;
  const long long hw = (long long)H * W;
  long long R, D;
  const int rc = check_entries(F, hw, n_entries, slots, counts, draw, n_draws, max_rays, &R, &D);
  if (rc != GOSLAM_OK) return rc;
  if (R == 0) return GOSLAM_OK;
  if (!pose || !rays_o || !rays_d || !depth || !color || (D > 0 && !draws)) return GOSLAM_EINVAL;
  SnapWork w;
  if (!workspace || workspace_bytes < snap_layout(F, hw, workspace, &w)) return GOSLAM_EWORKSPACE;
  const Intr in = make_intr(fx, fy, cx, cy);
  cudaStream_t st = (cudaStream_t)stream;
  long long out = 0, rnd = 0;
  for (int b = 0; b < n_entries; b += kMaxEntries) {
    int r, d;
    const RayEntries e = chunk_entries(b, n_entries, slots, counts, draw, &r, &d);
    if (r > 0) {
      ray_batch_kernel<kQuadt><<<gs_cdiv(r, kRayThreads), kRayThreads, 0, st>>>(
          e, r, (int)hw, W, w.pix, w.rec, kQuadt ? pose + 7 * (size_t)b : pose, (const long long*)draws + rnd, in,
          rays_o + 3 * out, rays_d + 3 * out, depth + out, color + 3 * out);
      GS_CHECK_LAUNCH();
    }
    out += r;
    rnd += d;
  }
  return GOSLAM_OK;
}

}  // namespace

extern "C" {

size_t goslam_mapping_snapshot_workspace_bytes(int F, int H, int W) {
  if (!snap_shape_ok(F, H, W) || F == 0) return 0;
  SnapWork w;
  return snap_layout(F, (long long)H * W, nullptr, &w);
}

int goslam_mapping_snapshot(const float* images, const float* mask, const float* disps, float* update_priority, int buffer,
                            int H, int W, const int* frames, const int* occurrences, int F, float decay, void* workspace,
                            size_t workspace_bytes, int* counts, void* stream) {
  if (!snap_shape_ok(F, H, W) || buffer <= 0) return GOSLAM_EINVAL;
  if (F == 0) return GOSLAM_OK;
  if (!images || !mask || !disps || !update_priority || !frames || !occurrences || !counts) return GOSLAM_EINVAL;
  const long long hw = (long long)H * W;
  SnapWork w;
  if (!workspace || workspace_bytes < snap_layout(F, hw, workspace, &w)) return GOSLAM_EWORKSPACE;
  const int T = num_tiles(hw);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(T, F);
  snapshot_count_kernel<<<grid, kSnapThreads, 0, st>>>(mask, frames, buffer, (int)hw, T, w.tile_count);
  GS_CHECK_LAUNCH();
  snapshot_scan_kernel<<<F, kSnapThreads, 0, st>>>(w.tile_count, T, frames, occurrences, buffer, decay, update_priority,
                                                    w.tile_off, counts);
  GS_CHECK_LAUNCH();
  snapshot_emit_kernel<<<grid, kSnapThreads, 0, st>>>(images, mask, disps, frames, buffer, (int)hw, T, w.tile_off, w.pix,
                                                       w.rec);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_mapping_rays(const void* workspace, size_t workspace_bytes, int F, int H, int W, const float* c2w,
                        const int64_t* draws, int64_t n_draws, int n_entries, const int* slots, const int* counts,
                        const int* draw, double fx, double fy, double cx, double cy, float* rays_o, float* rays_d, float* depth,
                        float* color, int64_t max_rays, void* stream) {
  return launch_ray_batch<false>(workspace, workspace_bytes, F, H, W, c2w, draws, n_draws, n_entries, slots, counts, draw,
                                 fx, fy, cx, cy, rays_o, rays_d, depth, color, max_rays, stream);
}

int goslam_mapping_pose_rays(const void* workspace, size_t workspace_bytes, int F, int H, int W, const float* quadt,
                             const int64_t* draws, int64_t n_draws, int n_entries, const int* slots, const int* counts,
                             const int* draw, double fx, double fy, double cx, double cy, float* rays_o, float* rays_d,
                             float* depth, float* color, int64_t max_rays, void* stream) {
  return launch_ray_batch<true>(workspace, workspace_bytes, F, H, W, quadt, draws, n_draws, n_entries, slots, counts, draw,
                                fx, fy, cx, cy, rays_o, rays_d, depth, color, max_rays, stream);
}

int goslam_mapping_pose_rays_backward(const void* workspace, size_t workspace_bytes, int F, int H, int W,
                                      const float* quadt, const int64_t* draws, int64_t n_draws, int n_entries,
                                      const int* slots, const int* counts, const int* draw, double fx, double fy,
                                      double cx, double cy, const float* d_rays_o, const float* d_rays_d,
                                      int64_t max_rays, float* d_quadt, void* stream) {
  if (!snap_shape_ok(F, H, W) || F == 0) return GOSLAM_EINVAL;
  const long long hw = (long long)H * W;
  long long R, D;
  const int rc = check_entries(F, hw, n_entries, slots, counts, draw, n_draws, max_rays, &R, &D);
  if (rc != GOSLAM_OK) return rc;
  if (n_entries == 0) return GOSLAM_OK;
  if (!quadt || !d_quadt || (R > 0 && (!d_rays_o || !d_rays_d)) || (D > 0 && !draws)) return GOSLAM_EINVAL;
  SnapWork w;
  if (!workspace || workspace_bytes < snap_layout(F, hw, workspace, &w)) return GOSLAM_EWORKSPACE;
  const Intr in = make_intr(fx, fy, cx, cy);
  cudaStream_t st = (cudaStream_t)stream;
  long long out = 0, rnd = 0;
  for (int b = 0; b < n_entries; b += kMaxEntries) {
    int r, d;
    const RayEntries e = chunk_entries(b, n_entries, slots, counts, draw, &r, &d);
    pose_rays_backward_kernel<<<e.n, kPoseBwdThreads, 0, st>>>(
        e, (int)hw, W, w.pix, quadt + 7 * (size_t)b, (const long long*)draws + rnd, in, d_rays_o + 3 * out,
        d_rays_d + 3 * out, d_quadt + 7 * (size_t)b);
    GS_CHECK_LAUNCH();
    out += r;
    rnd += d;
  }
  return GOSLAM_OK;
}

int goslam_mapping_c2w_to_quadt(const float* c2w, int n, float* quadt, void* stream) {
  if (n < 0) return GOSLAM_EINVAL;
  if (n == 0) return GOSLAM_OK;
  if (!c2w || !quadt) return GOSLAM_EINVAL;
  c2w_to_quadt_kernel<<<gs_cdiv(n, kRayThreads), kRayThreads, 0, (cudaStream_t)stream>>>(c2w, n, quadt);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_mapping_all_rays(const float* c2w, int H, int W, double fx, double fy, double cx, double cy, float* rays_o,
                            float* rays_d, void* stream) {
  if (H <= 0 || W <= 0 || (long long)H * W > kMaxPixels) return GOSLAM_EINVAL;
  if (!c2w || !rays_o || !rays_d) return GOSLAM_EINVAL;
  const int hw = H * W;
  all_rays_kernel<<<gs_cdiv(hw, kRayThreads), kRayThreads, 0, (cudaStream_t)stream>>>(
      c2w, hw, W, make_intr(fx, fy, cx, cy), rays_o, rays_d);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
