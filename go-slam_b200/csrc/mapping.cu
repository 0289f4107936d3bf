// mapping.cu — the mapping process's frame hand-over and ray sampling (src/mapping.py:151-300,
// src/depth_video.py:153-173, src/nerf_func.py:115-221) for sm_90a.
//
// snapshot (once per Mapper.__call__, under the video's mapping lock):
//   count   one block per (1024-pixel tile, frame): the tile's number of masked pixels
//   scan    one block per frame: exclusive tile prefixes, N_f, and the update_priority decay
//   emit    one block per (tile, frame): the tile's masked pixels as compact records in raster order
// rays (once per training iteration): one launch for the whole concatenated batch.
// all rays (render_img): every pixel of one image in raster order, the same per-pixel arithmetic.
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

// the ray of pixel (x, y) under c2w (row-major 4x4, f32):
//   dirs = ((x - cx) * rfx, (y - cy) * rfy, 1) with cx = (float)cx and rfx = (float)(1.0 / fx) — torch's CUDA true
//   division by a Python scalar multiplies by the reciprocal, taken in double and rounded to f32 (measured on an H100
//   with torch 2.11: bit-identical, where 1.0f / (float)fx and a true f32 division both differ);
//   rays_d[r] = (dirs.x * R[r][0] + dirs.y * R[r][1]) + R[r][2], every product and sum rounded separately (no FMA),
//   the order documented in the header; rays_o = t(c2w).
__device__ __forceinline__ void pixel_ray(float x, float y, const float* __restrict__ c2w, const Intr& in,
                                          float* __restrict__ o, float* __restrict__ d) {
  const float dx = __fmul_rn(__fsub_rn(x, in.cx), in.rfx);
  const float dy = __fmul_rn(__fsub_rn(y, in.cy), in.rfy);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float* row = c2w + 4 * r;
    d[r] = __fadd_rn(__fadd_rn(__fmul_rn(dx, __ldg(row)), __fmul_rn(dy, __ldg(row + 1))), __ldg(row + 2));
    o[r] = __ldg(row + 3);
  }
}

struct RayEntries {
  int n;
  int slot[kMaxEntries];       // snapshot slot of the entry's frame
  int draw[kMaxEntries];       // > 0: that many random records (indices from `draws`); 0: all records in raster order
  int out_off[kMaxEntries];    // first output row, relative to the launch
  int rand_off[kMaxEntries];   // first index in `draws`
  int count[kMaxEntries];      // N_f of the slot
};

__global__ void __launch_bounds__(kRayThreads) ray_batch_kernel(const __grid_constant__ RayEntries e, int R, int hw, int W,
                                                                 const int* __restrict__ pix, const float4* __restrict__ rec,
                                                                 const float* __restrict__ c2w, const long long* __restrict__ draws,
                                                                 Intr in, float* __restrict__ rays_o, float* __restrict__ rays_d,
                                                                 float* __restrict__ depth, float* __restrict__ color) {
  const int i = blockIdx.x * kRayThreads + threadIdx.x;
  if (i >= R) return;
  // the last entry starting at or before i (empty entries share their successor's start)
  int lo = 0, hi = e.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (e.out_off[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  const int j = i - e.out_off[lo];
  long long k = j;
  if (e.draw[lo] > 0) {
    k = __ldg(draws + e.rand_off[lo] + j);              // torch.randint(N, (n_rays,)).clamp(0, N - 1)
    k = k < 0 ? 0 : (k > e.count[lo] - 1 ? e.count[lo] - 1 : k);
  }
  const size_t r = (size_t)e.slot[lo] * hw + k;
  const int p = __ldg(pix + r);
  const float4 v = __ldg(rec + r);
  float o[3], d[3];
  pixel_ray((float)(p % W), (float)(p / W), c2w + 16 * e.slot[lo], in, o, d);
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

__global__ void __launch_bounds__(kRayThreads) all_rays_kernel(const float* __restrict__ c2w, int hw, int W, Intr in,
                                                                float* __restrict__ rays_o, float* __restrict__ rays_d) {
  const int i = blockIdx.x * kRayThreads + threadIdx.x;
  if (i >= hw) return;
  float o[3], d[3];
  pixel_ray((float)(i % W), (float)(i / W), c2w, in, o, d);
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
  if (!snap_shape_ok(F, H, W) || F == 0 || n_entries < 0 || n_draws < 0 || max_rays < 0) return GOSLAM_EINVAL;
  if (n_entries > 0 && (!slots || !counts || !draw)) return GOSLAM_EINVAL;
  const long long hw = (long long)H * W;
  long long R = 0, D = 0;
  for (int i = 0; i < n_entries; ++i) {
    if (slots[i] < 0 || slots[i] >= F || counts[i] < 0 || counts[i] > hw || draw[i] < 0 || (draw[i] > 0 && counts[i] == 0))
      return GOSLAM_EINVAL;
    R += draw[i] > 0 ? draw[i] : counts[i];
    D += draw[i];
  }
  if (R > max_rays || D > n_draws || R > INT32_MAX) return GOSLAM_EINVAL;
  if (R == 0) return GOSLAM_OK;
  if (!c2w || !rays_o || !rays_d || !depth || !color || (D > 0 && !draws)) return GOSLAM_EINVAL;
  SnapWork w;
  if (!workspace || workspace_bytes < snap_layout(F, hw, workspace, &w)) return GOSLAM_EWORKSPACE;
  const Intr in = make_intr(fx, fy, cx, cy);
  cudaStream_t st = (cudaStream_t)stream;
  long long out = 0, rnd = 0;
  for (int b = 0; b < n_entries; b += kMaxEntries) {
    RayEntries e;
    e.n = n_entries - b < kMaxEntries ? n_entries - b : kMaxEntries;
    int r = 0, d = 0;
    for (int i = 0; i < e.n; ++i) {
      e.slot[i] = slots[b + i];
      e.draw[i] = draw[b + i];
      e.count[i] = counts[b + i];
      e.out_off[i] = r;
      e.rand_off[i] = d;
      r += e.draw[i] > 0 ? e.draw[i] : e.count[i];
      d += e.draw[i];
    }
    if (r > 0) {
      ray_batch_kernel<<<gs_cdiv(r, kRayThreads), kRayThreads, 0, st>>>(
          e, r, (int)hw, W, w.pix, w.rec, c2w, (const long long*)draws + rnd, in, rays_o + 3 * out, rays_d + 3 * out,
          depth + out, color + 3 * out);
      GS_CHECK_LAUNCH();
    }
    out += r;
    rnd += d;
  }
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
