// geom.cu — per-pixel reprojection kernels of the droid_backends boundary:
// frame_distance, projmap, iproj, depth_filter and the DepthVideo.reproject fusion.
// All are a few flops per 4-byte pixel => HBM/latency bound; one thread per pixel,
// coalesced along x, relative pose computed once per block into shared memory.
#include <cub/cub.cuh>

#include "common.cuh"
#include "se3.cuh"

#include <algorithm>
#include <climits>

namespace {

constexpr int kThreads = 256;

// ---------------------------------------------------------------------------------
// frame_distance  (reference: src/lib/droid_kernels.cu:518-657)
// One block per (i,j) pair.  The float summation order is part of the contract: the
// distances are sorted / thresholded into factor-graph edges, so we keep the reference's
// association exactly — thread t sums pixels t, t+256, ... serially, then a fixed
// 128 / 64 / 32 / 16 / 8 / 4 / 2 / 1 tree (src/lib/droid_kernels.cu:36-55).
// ---------------------------------------------------------------------------------
__device__ __forceinline__ float tree256(float v, float* s) {
  const int tid = threadIdx.x;
  s[tid] = v;
  __syncthreads();
  if (tid < 128) s[tid] += s[tid + 128];
  __syncthreads();
  if (tid < 64) s[tid] += s[tid + 64];
  __syncthreads();
  float r = 0.f;
  if (tid < 32) {
    r = s[tid] + s[tid + 32];
    r += __shfl_down_sync(0xffffffffu, r, 16);
    r += __shfl_down_sync(0xffffffffu, r, 8);
    r += __shfl_down_sync(0xffffffffu, r, 4);
    r += __shfl_down_sync(0xffffffffu, r, 2);
    r += __shfl_down_sync(0xffffffffu, r, 1);
  }
  __syncthreads();
  return r;  // valid in thread 0
}

// distance of the ordered pair (ix -> jx); the value is valid in thread 0.  NOT inlined: the one-way and the
// bidirectional kernel must run the very same instruction sequence (FMA contraction included) so that
// 0.5 * (d_ij + d_ji) is bit-identical in both forms.
__device__ __noinline__ float pair_distance(const float* __restrict__ poses, const float* __restrict__ disps,
                                               const float* __restrict__ intr, int ix, int jx, int ht, int wd,
                                               float beta, float* red) {
  const float fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];

  // NB: no stereo special case here — the reference calls relSE3 unconditionally.
  GsSE3 G;
  {
    const float* pi = poses + 7 * (size_t)ix;
    const float* pj = poses + 7 * (size_t)jx;
    gs_rel(pi, pi + 3, pj, pj + 3, G);
  }

  float accum = 0.f, valid = 0.f, total = 0.f;
  const float* dsp = disps + (size_t)ix * ht * wd;
  const float omb = 1 - beta;
  for (int k = threadIdx.x; k < ht * wd; k += kThreads) {
    const float u = (float)(k % wd);
    const float v = (float)(k / wd);
    float Xi[4], Xj[4];
    Xi[0] = (u - cx) / fx;
    Xi[1] = (v - cy) / fy;
    Xi[2] = 1.f;
    Xi[3] = dsp[k];
    gs_act4(G, Xi, Xj);

    float du = fx * (Xj[0] / Xj[2]) + cx - u;
    float dv = fy * (Xj[1] / Xj[2]) + cy - v;
    float d = sqrtf(du * du + dv * dv);
    total += beta;
    if (Xj[2] > GS_MIN_DEPTH) {
      accum += beta * d;
      valid += beta;
    }

    // translation-only term
    Xj[0] = Xi[0] + Xi[3] * G.t[0];
    Xj[1] = Xi[1] + Xi[3] * G.t[1];
    Xj[2] = Xi[2] + Xi[3] * G.t[2];
    du = fx * (Xj[0] / Xj[2]) + cx - u;
    dv = fy * (Xj[1] / Xj[2]) + cy - v;
    d = sqrtf(du * du + dv * dv);
    total += omb;
    if (Xj[2] > GS_MIN_DEPTH) {
      accum += omb * d;
      valid += omb;
    }
  }
  const float a = tree256(accum, red);
  const float t = tree256(total, red);
  const float w = tree256(valid, red);
  return (w / (t + 1e-8f) < 0.75f) ? 1000.0f : a / w;
}

__global__ void __launch_bounds__(kThreads)
frame_distance_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                      const float* __restrict__ intr, const int64_t* __restrict__ ii,
                      const int64_t* __restrict__ jj, float* __restrict__ dist,
                      int ht, int wd, float beta) {
  __shared__ float red[kThreads];
  const float d = pair_distance(poses, disps, intr, (int)ii[blockIdx.x], (int)jj[blockIdx.x], ht, wd, beta, red);
  if (threadIdx.x == 0) dist[blockIdx.x] = d;
}

// DepthVideo.distance(bidirectional=True) (src/depth_video.py:233-245): 0.5 * (d(i->j) + d(j->i)) in one
// launch; each direction keeps the reduction tree above, so the result equals the two-launch form bit for bit.
__global__ void __launch_bounds__(kThreads)
frame_distance_bidir_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                            const float* __restrict__ intr, const int64_t* __restrict__ ii,
                            const int64_t* __restrict__ jj, float* __restrict__ dist,
                            int ht, int wd, float beta) {
  __shared__ float red[kThreads];
  const int ix = (int)ii[blockIdx.x], jx = (int)jj[blockIdx.x];
  const float d1 = pair_distance(poses, disps, intr, ix, jx, ht, wd, beta, red);
  const float d2 = pair_distance(poses, disps, intr, jx, ix, ht, wd, beta, red);
  if (threadIdx.x == 0) dist[blockIdx.x] = __fmul_rn(0.5f, __fadd_rn(d1, d2));
}

// ---------------------------------------------------------------------------------
// Banded frame-distance grid: the bidirectional distance over rows [r0, r1) x columns [c0, c1), computed only where
// j - i <= k (Backend.ba reads nothing else, DESIGN.md §3.18) and +inf elsewhere, straight from the ranges.
// Row i of the band holds n(i) = clamp(i + k + 1 - c0, 0, W) entries (W = c1 - c0), so the band's first entry of row
// i sits at S(i) = T(i + a) - T(r0 + a) with a = k + 1 - c0 and T(m) = sum_{t < m} clamp(t, 0, W), and a block finds
// its row by bisection on S.  Blocks [0, P) each own one band entry (P = S(r1)); blocks [P, P + F) write the +inf.
// When the mirror (j, i) is in the band too, the block with i < j computes the pair once and writes both entries
// (0.5 * (d1 + d2) with IEEE addition, which commutes) and the block with i > j has nothing to do.
// ---------------------------------------------------------------------------------
struct GridBand {
  int r0, r1, c0, c1, k;
  __device__ long long tri(long long m) const {           // T(m)
    const long long W = c1 - c0;
    if (m <= 0) return 0;
    if (m <= W + 1) return m * (m - 1) / 2;
    return W * (W + 1) / 2 + (m - W - 1) * W;
  }
  __device__ long long start(int i) const {               // S(i): band entries in rows [r0, i)
    const long long a = (long long)k + 1 - c0;
    return tri(i + a) - tri(r0 + a);
  }
  __device__ bool has(int i, int j) const { return i >= r0 && i < r1 && j >= c0 && j < c1 && j - i <= k; }
};

__global__ void __launch_bounds__(kThreads)
frame_distance_grid_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                           const float* __restrict__ intr, GridBand band, long long n_band, int fill_blocks,
                           float* __restrict__ dist, int ht, int wd, float beta) {
  __shared__ float red[kThreads];
  const long long W = band.c1 - band.c0;
  const long long b = blockIdx.x;
  if (b >= n_band) {                                      // +inf outside the band, grid-stride over the matrix
    const long long n = (long long)(band.r1 - band.r0) * W;
    const float inf = __int_as_float(0x7f800000);
    for (long long q = (b - n_band) * kThreads + threadIdx.x; q < n; q += (long long)fill_blocks * kThreads) {
      const int i = band.r0 + (int)(q / W), j = band.c0 + (int)(q % W);
      if (j - i > band.k) dist[q] = inf;
    }
    return;
  }
  int lo = band.r0, hi = band.r1 - 1;                     // largest row i with S(i) <= b (uniform over the block)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (band.start(mid) <= b) lo = mid; else hi = mid - 1;
  }
  const int i = lo, j = band.c0 + (int)(b - band.start(i));
  const bool mirrored = i != j && band.has(j, i);
  if (mirrored && i > j) return;
  const float d1 = pair_distance(poses, disps, intr, i, j, ht, wd, beta, red);
  const float d2 = pair_distance(poses, disps, intr, j, i, ht, wd, beta, red);
  if (threadIdx.x == 0) {
    const float d = __fmul_rn(0.5f, __fadd_rn(d1, d2));
    dist[(i - band.r0) * W + (j - band.c0)] = d;
    if (mirrored) dist[(j - band.r0) * W + (i - band.c0)] = d;
  }
}

// ---------------------------------------------------------------------------------
// projmap  (reference: src/lib/droid_kernels.cu:427-516)
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
projmap_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
               const float* __restrict__ intr, const int64_t* __restrict__ ii,
               const int64_t* __restrict__ jj, float* __restrict__ coords,
               float* __restrict__ valid, int ht, int wd) {
  const int e = blockIdx.y;
  const int k = blockIdx.x * kThreads + threadIdx.x;
  const int ix = (int)ii[e], jx = (int)jj[e];
  __shared__ GsSE3 G;
  if (threadIdx.x == 0) {
    const float* pi = poses + 7 * (size_t)ix;
    const float* pj = poses + 7 * (size_t)jx;
    gs_rel(pi, pi + 3, pj, pj + 3, G);
  }
  __syncthreads();
  if (k >= ht * wd) return;
  const float fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];
  const float u = (float)(k % wd), v = (float)(k / wd);
  float Xi[4] = {(u - cx) / fx, (v - cy) / fy, 1.f, disps[(size_t)ix * ht * wd + k]};
  float Xj[4];
  gs_act4(G, Xi, Xj);
  float cu = u, cv = v;
  if (Xj[2] > 0.01f) {
    cu = fx * (Xj[0] / Xj[2]) + cx;
    cv = fy * (Xj[1] / Xj[2]) + cy;
  }
  float* c = coords + ((size_t)e * ht * wd + k) * 3;
  c[0] = cu; c[1] = cv; c[2] = 0.f;
  valid[(size_t)e * ht * wd + k] = (Xj[2] > GS_MIN_DEPTH) ? 1.0f : 0.0f;
}

// ---------------------------------------------------------------------------------
// reproject: DepthVideo.reproject -> pops.projective_transform(jacobian=False)
// (src/depth_video.py:207-217, src/geom/projective_ops.py:26-44,54-57,88-99,114-144).
// Python-side constants: MIN_DEPTH = 0.2, Z < 0.1 replaced by 1 before dividing.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
reproject_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                 const float* __restrict__ intr_all, const int64_t* __restrict__ ii,
                 const int64_t* __restrict__ jj, float* __restrict__ coords,
                 float* __restrict__ valid, const float* __restrict__ target,
                 float* __restrict__ motion, int ht, int wd) {
  const int e = blockIdx.y;
  const int k = blockIdx.x * kThreads + threadIdx.x;
  const int ix = (int)ii[e], jx = (int)jj[e];
  __shared__ GsSE3 G;
  if (threadIdx.x == 0) gs_edge_pose(poses, ix, jx, G);
  __syncthreads();
  if (k >= ht * wd) return;
  const float* Ki = intr_all + 4 * (size_t)ix;
  const float* Kj = intr_all + 4 * (size_t)jx;
  const float u = (float)(k % wd), v = (float)(k / wd);
  float X0[4] = {(u - Ki[2]) / Ki[0], (v - Ki[3]) / Ki[1], 1.f,
                 disps[(size_t)ix * ht * wd + k]};
  float X1[4];
  gs_act4(G, X0, X1);
  const float Z = (X1[2] < 0.5f * 0.2f) ? 1.0f : X1[2];
  float2 c;
  c.x = Kj[0] * (X1[0] / Z) + Kj[2];
  c.y = Kj[1] * (X1[1] / Z) + Kj[3];
  reinterpret_cast<float2*>(coords)[(size_t)e * ht * wd + k] = c;
  if (valid) valid[(size_t)e * ht * wd + k] = (X1[2] > 0.2f) ? 1.0f : 0.0f;
  if (motion) {
    // FactorGraph.update's motion features (src/factor_graph.py:204-206):
    // cat([coords1 - coords0, target - coords1], -1).permute(0,1,4,2,3).clamp(-64, 64)
    const float2 t = reinterpret_cast<const float2*>(target)[(size_t)e * ht * wd + k];
    float* m = motion + (size_t)e * 4 * ht * wd + k;
    const size_t hw = (size_t)ht * wd;
    m[0] = fminf(fmaxf(c.x - u, -64.f), 64.f);
    m[hw] = fminf(fmaxf(c.y - v, -64.f), 64.f);
    m[2 * hw] = fminf(fmaxf(t.x - c.x, -64.f), 64.f);
    m[3 * hw] = fminf(fmaxf(t.y - c.y, -64.f), 64.f);
  }
}

// ---------------------------------------------------------------------------------
// iproj  (reference: src/lib/droid_kernels.cu:779-850)
// ---------------------------------------------------------------------------------
// world point of pixel (u, v) with inverse depth d under pose p = (t, q); shared with the multiview filter so that
// its points are iproj's, bit for bit.  d = 0 gives inf / NaN components, as in the reference.
__device__ __forceinline__ void iproj_point(const float* __restrict__ p, float fx, float fy, float cx, float cy,
                                            float u, float v, float d, float* o) {
  GsSE3 G;
  G.t[0] = p[0]; G.t[1] = p[1]; G.t[2] = p[2];
  G.q[0] = p[3]; G.q[1] = p[4]; G.q[2] = p[5]; G.q[3] = p[6];
  float Xi[4] = {(u - cx) / fx, (v - cy) / fy, 1.f, d};
  float Xj[4];
  gs_act4(G, Xi, Xj);
  o[0] = Xj[0] / Xj[3];
  o[1] = Xj[1] / Xj[3];
  o[2] = Xj[2] / Xj[3];
}

__global__ void __launch_bounds__(kThreads)
iproj_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
             const float* __restrict__ intr, float* __restrict__ points, int ht, int wd) {
  const int f = blockIdx.y;
  const int k = blockIdx.x * kThreads + threadIdx.x;
  if (k >= ht * wd) return;
  const float fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];
  float* o = points + ((size_t)f * ht * wd + k) * 3;
  iproj_point(poses + 7 * (size_t)f, fx, fy, cx, cy, (float)(k % wd), (float)(k / wd), disps[(size_t)f * ht * wd + k],
              o);
}

// ---------------------------------------------------------------------------------
// depth_filter  (reference: src/lib/droid_kernels.cu:661-775).  The reference scatters
// atomicAdd over a (frame, neighbour, tile) grid; each output pixel only ever receives
// its own 6 neighbour votes, so we loop the 6 neighbours inside one thread instead:
// same counts, no atomics, no memset.
// ---------------------------------------------------------------------------------
// relative poses frame ix -> its 6 neighbours ix-1, ix-2, ix-3, ix+3, ix+4, ix+5 (threads 0..5 of the block)
__device__ __forceinline__ void vote_neighbours(const float* __restrict__ poses, int ix, int num, GsSE3* G, int* jxs) {
  if (threadIdx.x < 6) {
    const int nb = threadIdx.x;
    const int jx = (nb < 3) ? ix - nb - 1 : ix + nb;
    jxs[nb] = jx;
    if (jx >= 0 && jx < num) {
      const float* pi = poses + 7 * (size_t)ix;
      const float* pj = poses + 7 * (size_t)jx;
      gs_rel(pi, pi + 3, pj, pj + 3, G[nb]);
    }
  }
}

// number of neighbours whose inverse depth agrees with pixel k = (i, j) of a frame with inverse depth d
__device__ __forceinline__ float depth_votes(const GsSE3* G, const int* jxs, const float* __restrict__ disps,
                                             float fx, float fy, float cx, float cy, float t, float d, int i, int j,
                                             int num, int ht, int wd) {
  const float ui = (float)j, vi = (float)i;
  float Xi[4] = {(ui - cx) / fx, (vi - cy) / fy, 1.f, d};
  float count = 0.f;
#pragma unroll
  for (int nb = 0; nb < 6; ++nb) {
    const int jx = jxs[nb];
    if (jx < 0 || jx >= num) continue;
    float Xj[4];
    gs_act4(G[nb], Xi, Xj);
    const float uj = fx * (Xj[0] / Xj[2]) + cx;
    const float vj = fy * (Xj[1] / Xj[2]) + cy;
    const float dj = Xj[3] / Xj[2];
    const int u0 = (int)floorf(uj);
    const int v0 = (int)floorf(vj);
    if (u0 >= 0 && v0 >= 0 && u0 < wd - 1 && v0 < ht - 1) {
      const float* dj_map = disps + (size_t)jx * ht * wd;
      const float d00 = dj_map[(v0 + 0) * wd + u0 + 0];
      const float d01 = dj_map[(v0 + 0) * wd + u0 + 1];
      const float d10 = dj_map[(v0 + 1) * wd + u0 + 0];
      const float d11 = dj_map[(v0 + 1) * wd + u0 + 1];
      // the reference evaluates these in double (1.0/dj literals), then compares to float t
      const double inv = 1.0 / dj;
      if (fabs(inv - 1.0 / d00) < t) count += 1.0f;
      else if (fabs(inv - 1.0 / d01) < t) count += 1.0f;
      else if (fabs(inv - 1.0 / d10) < t) count += 1.0f;
      else if (fabs(inv - 1.0 / d11) < t) count += 1.0f;
    }
  }
  return count;
}

__global__ void __launch_bounds__(kThreads)
depth_filter_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                    const float* __restrict__ intr, const int64_t* __restrict__ inds,
                    const float* __restrict__ thresh, float* __restrict__ counter,
                    int num, int ht, int wd) {
  const int b = blockIdx.y;
  const int k = blockIdx.x * kThreads + threadIdx.x;
  const int ix = (int)inds[b];
  __shared__ GsSE3 G[6];
  __shared__ int jxs[6];
  vote_neighbours(poses, ix, num, G, jxs);
  __syncthreads();
  if (k >= ht * wd) return;
  const float t = thresh[b];
  const float fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];
  const int i = k / wd, j = k % wd;
  counter[(size_t)b * ht * wd + k] =
      depth_votes(G, jxs, disps, fx, fy, cx, cy, t, disps[(size_t)ix * ht * wd + k], i, j, num, ht, wd);
}

// ---------------------------------------------------------------------------------
// Multiview filter  (reference: src/multiview_filter.py:98-170, one pass of MultiviewFilter.forward).
// Four launches over T frames at full resolution, no host synchronisation:
//   mv_mean_kernel    per-frame mean inverse depth (fp64 sum in a fixed order, rounded to fp32);
//                     block 0 also resets the reduction state of the pass.
//   mv_vote_kernel    depth_filter's vote + mask1 = count >= visible_num && d > 0.01 * mean, mask1 bytes,
//                     count and min / max of the mask1 world points (the first bound).
//   mv_extend_kernel  extended mask (all / mask1 / box dilation of mask1), AND the strict in-bound test against
//                     the first bound, final mask bytes, counts and min / max of the final points (second bound).
//   mv_commit_kernel  (separate entry point, called under the mapping lock) gated on the device: priority,
//                     poses / disps / mask / bound / filtered_id of the video, and a status record.
// Min / max / counts are integer atomics (floats mapped to order-preserving ints), so the bounds are exact and the
// pass is deterministic whatever the block order.  Points are recomputed in the extend pass, not stored.
// ---------------------------------------------------------------------------------
constexpr int kMvPerThread = 8;                      // pixels per thread of the vote / extend passes
constexpr int kMvTile = kThreads * kMvPerThread;
constexpr int kMvMeanThreads = 512;
constexpr int kMvMaxRadius = 15;

struct MvState {
  int mn1[3], mx1[3];                 // first bound (mask1 points), order-preserving ints
  int mn2[3], mx2[3];                 // second bound (final points)
  unsigned long long n1, n_ext, n_fin;
};
struct MvWork { MvState* st; float* mean; unsigned char* mask1; unsigned char* fin; };   // mean [T], masks [T, hw]

size_t mv_layout(int T, size_t hw, const void* base, MvWork* w) {
  GsArena ar(base);
  w->st = ar.take<MvState>(1);
  w->mean = ar.take<float>(T);
  w->mask1 = ar.take<unsigned char>((size_t)T * hw);
  w->fin = ar.take<unsigned char>((size_t)T * hw);
  return ar.off;
}

// float -> int with the same order (-0 sorts below +0); the map is its own inverse
__device__ __forceinline__ int mv_ord(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float mv_unord(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// get_bound_from_pointcloud(pts) with its default enlarge_scale = 1.0, in torch's fp32 op order
// (src/multiview_filter.py:82-96): len = (max - min) * 0, bound = [min - len / 2, max + len / 2]
__device__ __forceinline__ void mv_bound(const int* omn, const int* omx, float* lo, float* hi) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float mn = mv_unord(omn[c]), mx = mv_unord(omx[c]);
    const float len = __fmul_rn(__fsub_rn(mx, mn), 0.0f);
    lo[c] = __fadd_rn(mn, __fdiv_rn(-len, 2.0f));
    hi[c] = __fadd_rn(mx, __fdiv_rn(len, 2.0f));
  }
}

// per-thread partial of one pass: points (count + min / max per axis) and, in the extend pass, extended pixels
struct MvAcc {
  int mn[3], mx[3];
  unsigned n, e;
  __device__ MvAcc() : mn{INT_MAX, INT_MAX, INT_MAX}, mx{INT_MIN, INT_MIN, INT_MIN}, n(0), e(0) {}
  __device__ void add(const float* p) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int o = mv_ord(p[c]);
      mn[c] = min(mn[c], o);
      mx[c] = max(mx[c], o);
    }
    ++n;
  }
};

// block reduction of MvAcc, then one set of atomics per block (skipped when the block saw nothing).
// Every thread of the block must call it.
__device__ __forceinline__ void mv_flush(MvAcc& a, int* gmn, int* gmx, unsigned long long* gn,
                                         unsigned long long* ge) {
  __shared__ MvAcc part[kThreads / 32];
  const unsigned full = 0xffffffffu;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    a.mn[c] = __reduce_min_sync(full, a.mn[c]);
    a.mx[c] = __reduce_max_sync(full, a.mx[c]);
  }
  a.n = __reduce_add_sync(full, a.n);
  a.e = __reduce_add_sync(full, a.e);
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) part[warp] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    MvAcc b = part[0];
    for (int w = 1; w < kThreads / 32; ++w) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        b.mn[c] = min(b.mn[c], part[w].mn[c]);
        b.mx[c] = max(b.mx[c], part[w].mx[c]);
      }
      b.n += part[w].n;
      b.e += part[w].e;
    }
    if (b.n) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        atomicMin(gmn + c, b.mn[c]);
        atomicMax(gmx + c, b.mx[c]);
      }
      atomicAdd(gn, (unsigned long long)b.n);
    }
    if (ge && b.e) atomicAdd(ge, (unsigned long long)b.e);
  }
}

__global__ void __launch_bounds__(kMvMeanThreads)
mv_mean_kernel(const float* __restrict__ disps, float* __restrict__ mean, MvState* __restrict__ st, int T, int hw) {
  const int f = blockIdx.x;
  if (f == 0 && threadIdx.x == 0) {
    for (int c = 0; c < 3; ++c) {
      st->mn1[c] = st->mn2[c] = INT_MAX;
      st->mx1[c] = st->mx2[c] = INT_MIN;
    }
    st->n1 = st->n_ext = st->n_fin = 0ull;
  }
  if (f >= T) return;
  // fixed order: thread t sums pixels t, t + 512, ... in fp64, then a fixed shuffle tree and a warp-0 tree
  const float* d = disps + (size_t)f * hw;
  double s = 0.0;
  for (int k = threadIdx.x; k < hw; k += kMvMeanThreads) s += (double)d[k];
  __shared__ double red[kMvMeanThreads / 32];
#pragma unroll
  for (int off = 16; off; off >>= 1) s += __shfl_down_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < kMvMeanThreads / 32 ? red[threadIdx.x] : 0.0;
#pragma unroll
    for (int off = 8; off; off >>= 1) s += __shfl_down_sync(0xffffffffu, s, off);
    if (threadIdx.x == 0) mean[f] = (float)(s / (double)hw);
  }
}

__global__ void __launch_bounds__(kThreads)
mv_vote_kernel(const float* __restrict__ poses, const float* __restrict__ poses_world,
               const float* __restrict__ disps, const float* __restrict__ intr, const float* __restrict__ mean,
               float thresh, float visible, unsigned char* __restrict__ mask1, MvState* __restrict__ st, int T,
               int ht, int wd) {
  const int f = blockIdx.y;
  const int hw = ht * wd;
  __shared__ GsSE3 G[6];
  __shared__ int jxs[6];
  vote_neighbours(poses, f, T, G, jxs);
  __syncthreads();
  const float fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];
  const float dmin = __fmul_rn(0.01f, mean[f]);       // torch: 0.01 * mean in fp32
  const float* dsp = disps + (size_t)f * hw;
  const float* pw = poses_world + 7 * (size_t)f;
  MvAcc acc;
  for (int r = 0; r < kMvPerThread; ++r) {
    const int k = blockIdx.x * kMvTile + r * kThreads + threadIdx.x;
    if (k >= hw) break;
    const int i = k / wd, j = k % wd;
    const float d = dsp[k];
    const float count = depth_votes(G, jxs, disps, fx, fy, cx, cy, thresh, d, i, j, T, ht, wd);
    const bool m = count >= visible && d > dmin;
    mask1[(size_t)f * hw + k] = m;
    if (m) {
      float p[3];
      iproj_point(pw, fx, fy, cx, cy, (float)j, (float)i, d, p);
      acc.add(p);
    }
  }
  mv_flush(acc, st->mn1, st->mx1, &st->n1, nullptr);
}

// radius < 0: every pixel ('inf'); 0: mask1; > 0: mask1 dilated by a (2r+1)^2 box with zero padding
// (F.conv2d(mask, ones(k, k), padding=k // 2).bool()).
__global__ void __launch_bounds__(kThreads)
mv_extend_kernel(const float* __restrict__ poses_world, const float* __restrict__ disps, const float* __restrict__ intr,
                 const unsigned char* __restrict__ mask1, unsigned char* __restrict__ fin, MvState* __restrict__ st,
                 int radius, int ht, int wd) {
  const int f = blockIdx.y;
  const int hw = ht * wd;
  float lo[3], hi[3];
  mv_bound(st->mn1, st->mx1, lo, hi);
  const float fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];
  const float* dsp = disps + (size_t)f * hw;
  const unsigned char* m1 = mask1 + (size_t)f * hw;
  const float* pw = poses_world + 7 * (size_t)f;
  MvAcc acc;
  for (int r = 0; r < kMvPerThread; ++r) {
    const int k = blockIdx.x * kMvTile + r * kThreads + threadIdx.x;
    if (k >= hw) break;
    const int i = k / wd, j = k % wd;
    bool e;
    if (radius < 0) {
      e = true;
    } else if (radius == 0) {
      e = m1[k];
    } else {
      e = false;
      const int y0 = max(i - radius, 0), y1 = min(i + radius, ht - 1);
      const int x0 = max(j - radius, 0), x1 = min(j + radius, wd - 1);
      for (int y = y0; y <= y1 && !e; ++y)
        for (int x = x0; x <= x1; ++x)
          if (m1[y * wd + x]) { e = true; break; }
    }
    bool keep = false;
    if (e) {
      ++acc.e;
      float p[3];
      iproj_point(pw, fx, fy, cx, cy, (float)j, (float)i, dsp[k], p);
      // strict, as in_bound (src/multiview_filter.py:64-79): inf / NaN points of d = 0 fail every comparison
      keep = p[0] > lo[0] && p[0] < hi[0] && p[1] > lo[1] && p[1] < hi[1] && p[2] > lo[2] && p[2] < hi[2];
      if (keep) acc.add(p);
    }
    fin[(size_t)f * hw + k] = keep;
  }
  mv_flush(acc, st->mn2, st->mx2, &st->n_fin, &st->n_ext);
}

// quaternion -> (roll, pitch, yaw) of MultiviewFilter.pose_dist, op for op in fp32 (src/multiview_filter.py:30-52);
// explicit roundings keep nvcc from contracting what torch evaluates as separate kernels
__device__ __forceinline__ void mv_euler(const float* p, float* e) {
  const float x = p[3], y = p[4], z = p[5], w = p[6];
  const float t0 = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(w, x), __fmul_rn(y, z)));
  const float t1 = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))));
  e[0] = atan2f(t0, t1);
  float t2 = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(w, y), __fmul_rn(z, x)));
  t2 = t2 < -1.0f ? -1.0f : (t2 > 1.0f ? 1.0f : t2);     // torch.clamp keeps NaN
  e[1] = asinf(t2);
  const float t3 = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(w, z), __fmul_rn(x, y)));
  const float t4 = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z))));
  e[2] = atan2f(t3, t4);
}

// 1 * |dt|_1 + 2 * |d euler|_1 (BundleFusion Sec. 5.3, src/multiview_filter.py:54-61)
__device__ __forceinline__ float mv_pose_dist(const float* p0, const float* p1) {
  float e0[3], e1[3];
  mv_euler(p0, e0);
  mv_euler(p1, e1);
  const float st = __fadd_rn(__fadd_rn(fabsf(__fsub_rn(p0[0], p1[0])), fabsf(__fsub_rn(p0[1], p1[1]))),
                             fabsf(__fsub_rn(p0[2], p1[2])));
  const float sr = __fadd_rn(__fadd_rn(fabsf(__fsub_rn(e0[0], e1[0])), fabsf(__fsub_rn(e0[1], e1[1]))),
                             fabsf(__fsub_rn(e0[2], e1[2])));
  return __fadd_rn(__fmul_rn(1.0f, st), __fmul_rn(2.0f, sr));
}

// The reference returns a second time when extended_masks.sum() < 100 (src/multiview_filter.py:142-143).  That
// cannot happen once masks.sum() >= 100: every extension mode contains mask1 (all pixels, mask1 itself, or a
// dilation whose box includes the centre pixel), so the gate below needs only the mask1 count.  An empty final
// point set is where the reference's torch.min raises; nothing is committed and the status says why.
__global__ void __launch_bounds__(kThreads)
mv_commit_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                 const unsigned char* __restrict__ fin, const MvState* __restrict__ st, int T, size_t n,
                 float* __restrict__ poses_filtered, float* __restrict__ disps_filtered,
                 float* __restrict__ mask_filtered, float* __restrict__ update_priority,
                 int* __restrict__ filtered_id, float* __restrict__ bound, int64_t* __restrict__ status) {
  const size_t gid = (size_t)blockIdx.x * kThreads + threadIdx.x;
  const bool commit = st->n1 >= 100ull && st->n_fin > 0ull;
  if (gid == 0) {
    status[0] = (int64_t)st->n1;
    status[1] = (int64_t)st->n_ext;
    status[2] = (int64_t)st->n_fin;
    status[3] = commit ? 1 : 0;
  }
  if (!commit) return;
  if (gid < (size_t)T) {
    float* pf = poses_filtered + 7 * gid;
    const float* p = poses + 7 * gid;
    update_priority[gid] = __fadd_rn(update_priority[gid], mv_pose_dist(pf, p));
#pragma unroll
    for (int c = 0; c < 7; ++c) pf[c] = p[c];
  }
  if (gid == 0) {
    float lo[3], hi[3];
    mv_bound(st->mn2, st->mx2, lo, hi);
    for (int c = 0; c < 3; ++c) {
      bound[2 * c] = lo[c];
      bound[2 * c + 1] = hi[c];
    }
    *filtered_id = T;
  }
  // mask and inverse depth of the T frames: 4 pixels per thread, grid-stride, scalar tail
  const size_t n4 = n / 4;
  const size_t stride = (size_t)gridDim.x * kThreads;
  for (size_t q = gid; q < n4; q += stride) {
    const uchar4 m = reinterpret_cast<const uchar4*>(fin)[q];
    reinterpret_cast<float4*>(mask_filtered)[q] =
        make_float4(m.x ? 1.f : 0.f, m.y ? 1.f : 0.f, m.z ? 1.f : 0.f, m.w ? 1.f : 0.f);
    reinterpret_cast<float4*>(disps_filtered)[q] = reinterpret_cast<const float4*>(disps)[q];
  }
  for (size_t q = 4 * n4 + gid; q < n; q += stride) {
    mask_filtered[q] = fin[q] ? 1.f : 0.f;
    disps_filtered[q] = disps[q];
  }
}

// ---------------------------------------------------------------------------------
// Mapping point selection  (Mesher.update_param_from_mapping, src/mesher.py:256-276): the world points of the
// keyframes' full-resolution inverse depths with count >= 3 votes (depth_filter, thresh 0.01) and d > 0.01 * the
// frame's mean, i.e. mask1 of the multiview filter with visible_num = 3.  mv_mean_kernel + mv_vote_kernel count them
// (MvState::n1); the emit is an ordered CUB select of iproj_point over mask1, [b, h, w] row-major, widened to f64.
// ---------------------------------------------------------------------------------
struct MapPoint3 {
  double x, y, z;
};

struct MapPointOp {
  const float* pw;
  const float* disps;
  const float* intr;
  int hw, wd;
  __device__ MapPoint3 operator()(long long g) const {
    const int f = (int)(g / hw), k = (int)(g - (long long)f * hw);
    float p[3];
    iproj_point(pw + 7 * (size_t)f, intr[0], intr[1], intr[2], intr[3], (float)(k % wd), (float)(k / wd), disps[g], p);
    return MapPoint3{(double)p[0], (double)p[1], (double)p[2]};
  }
};

using MapIter = cub::TransformInputIterator<MapPoint3, MapPointOp, cub::CountingInputIterator<long long>>;

struct MapWork { MvState* st; float* mean; unsigned char* mask1; long long* nsel; void* tmp; size_t tmp_bytes; };

size_t map_layout(int T, size_t hw, void* base, MapWork* w) {
  GsArena ar(base);
  w->st = ar.take<MvState>(1);
  w->mean = ar.take<float>(T);
  w->mask1 = ar.take<unsigned char>((size_t)T * hw);
  w->nsel = ar.take<long long>(1);
  // a failed size query is reported by the select call itself (GS_CUDA)
  size_t t = 0;
  cub::DeviceSelect::Flagged(nullptr, t, MapIter(cub::CountingInputIterator<long long>(0), MapPointOp{}),
                             (const unsigned char*)nullptr, (MapPoint3*)nullptr, (long long*)nullptr,
                             (long long)(T * hw));
  w->tmp_bytes = std::max<size_t>(t, 1);
  w->tmp = ar.take<char>(w->tmp_bytes);
  return ar.off;
}

struct GridWork { float* poses; size_t pose_bytes; };   // the poses [max(r1, c1), 7] the grid kernel reads

size_t grid_layout(int r1, int c1, void* base, GridWork* w) {
  const size_t n = (size_t)7 * std::max(r1, c1);
  GsArena ar(base);
  w->poses = ar.take<float>(n);
  w->pose_bytes = n * sizeof(float);
  return ar.off;
}

constexpr float kMapThresh = 0.01f;          // src/mesher.py:252-253
constexpr float kMapVisible = 3.0f;

}  // namespace

extern "C" {

int goslam_frame_distance(const float* poses, const float* disps, const float* intrinsics,
                          const int64_t* ii, const int64_t* jj, float* dist, int K, int ht,
                          int wd, float beta, void* stream) {
  if (K < 0 || ht <= 0 || wd <= 0) return GOSLAM_EINVAL;
  if (K == 0) return GOSLAM_OK;
  frame_distance_kernel<<<K, kThreads, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, ii,
                                                                  jj, dist, ht, wd, beta);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_frame_distance_bidir(const float* poses, const float* disps, const float* intrinsics,
                                const int64_t* ii, const int64_t* jj, float* dist, int K, int ht, int wd,
                                float beta, void* stream) {
  if (K < 0 || ht <= 0 || wd <= 0) return GOSLAM_EINVAL;
  if (K == 0) return GOSLAM_OK;
  frame_distance_bidir_kernel<<<K, kThreads, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, ii, jj, dist, ht,
                                                                        wd, beta);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

size_t goslam_frame_distance_grid_workspace_bytes(int r0, int r1, int c0, int c1) {
  if (r0 < 0 || c0 < 0 || r1 <= r0 || c1 <= c0) return 0;
  GridWork w;
  return grid_layout(r1, c1, nullptr, &w);
}

int goslam_frame_distance_grid(const float* poses, const float* disps, const float* intrinsics, int r0, int r1, int c0,
                               int c1, int k, int ht, int wd, float beta, float* dist, void* workspace,
                               size_t workspace_bytes, void* stream) {
  if (r0 < 0 || c0 < 0 || r1 < r0 || c1 < c0 || ht <= 0 || wd <= 0) return GOSLAM_EINVAL;
  if ((long long)(r1 - r0) * (c1 - c0) > (long long)INT_MAX) return GOSLAM_EINVAL;
  if (r1 == r0 || c1 == c0) return GOSLAM_OK;
  if (poses == nullptr || disps == nullptr || intrinsics == nullptr || dist == nullptr) return GOSLAM_EINVAL;
  GridWork w;
  if (!workspace || workspace_bytes < grid_layout(r1, c1, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  // the poses of frames [0, max(r1, c1)) as they are when this call reaches the stream: other processes write the
  // shared pose buffer while a backend pass runs, and every pair must see one consistent set
  GS_CUDA(cudaMemcpyAsync(w.poses, poses, w.pose_bytes, cudaMemcpyDeviceToDevice, s));
  // band size S(r1) on the host (same closed form as GridBand::start)
  const long long W = c1 - c0, a = (long long)k + 1 - c0;
  auto tri = [W](long long m) -> long long {
    if (m <= 0) return 0;
    if (m <= W + 1) return m * (m - 1) / 2;
    return W * (W + 1) / 2 + (m - W - 1) * W;
  };
  const long long n_band = tri(r1 + a) - tri(r0 + a);
  const long long n_all = (long long)(r1 - r0) * W;
  const int fill_blocks = n_band == n_all ? 0 : (int)std::min<long long>((n_all + 4 * kThreads - 1) / (4 * kThreads), 1024);
  const GridBand band{r0, r1, c0, c1, k};
  frame_distance_grid_kernel<<<(unsigned)(n_band + fill_blocks), kThreads, 0, s>>>(w.poses, disps, intrinsics, band, n_band,
                                                                                  fill_blocks, dist, ht, wd, beta);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_projmap(const float* poses, const float* disps, const float* intrinsics,
                   const int64_t* ii, const int64_t* jj, float* coords, float* valid, int K,
                   int ht, int wd, void* stream) {
  if (K < 0 || K > 65535 || ht <= 0 || wd <= 0) return GOSLAM_EINVAL;
  if (K == 0) return GOSLAM_OK;
  dim3 grid(gs_cdiv(ht * wd, kThreads), K);
  projmap_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, ii, jj,
                                                              coords, valid, ht, wd);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_reproject(const float* poses, const float* disps, const float* intrinsics_all,
                     const int64_t* ii, const int64_t* jj, float* coords, float* valid, int K,
                     int ht, int wd, void* stream) {
  if (K < 0 || K > 65535 || ht <= 0 || wd <= 0) return GOSLAM_EINVAL;
  if (K == 0) return GOSLAM_OK;
  dim3 grid(gs_cdiv(ht * wd, kThreads), K);
  reproject_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics_all, ii,
                                                                jj, coords, valid, nullptr, nullptr, ht, wd);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_reproject_motion(const float* poses, const float* disps, const float* intrinsics_all,
                            const int64_t* ii, const int64_t* jj, const float* target, float* coords,
                            float* valid, float* motion, int K, int ht, int wd, void* stream) {
  if (K < 0 || K > 65535 || ht <= 0 || wd <= 0 || target == nullptr || motion == nullptr) return GOSLAM_EINVAL;
  if (K == 0) return GOSLAM_OK;
  dim3 grid(gs_cdiv(ht * wd, kThreads), K);
  reproject_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics_all, ii,
                                                                jj, coords, valid, target, motion, ht, wd);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_iproj(const float* poses, const float* disps, const float* intrinsics, float* points,
                 int num, int ht, int wd, void* stream) {
  if (num < 0 || num > 65535 || ht <= 0 || wd <= 0) return GOSLAM_EINVAL;
  if (num == 0) return GOSLAM_OK;
  dim3 grid(gs_cdiv(ht * wd, kThreads), num);
  iproj_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, points, ht,
                                                            wd);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_depth_filter(const float* poses, const float* disps, const float* intrinsics,
                        const int64_t* ix, const float* thresh, float* counter, int K, int num,
                        int ht, int wd, void* stream) {
  if (K < 0 || K > 65535 || ht <= 0 || wd <= 0) return GOSLAM_EINVAL;
  if (K == 0) return GOSLAM_OK;
  dim3 grid(gs_cdiv(ht * wd, kThreads), K);
  depth_filter_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, ix,
                                                                   thresh, counter, num, ht, wd);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

size_t goslam_mvfilter_workspace_bytes(int T, int ht, int wd) {
  if (T < 0 || T > 65535 || ht <= 0 || wd <= 0) return 0;
  MvWork w;
  return mv_layout(T, (size_t)ht * wd, nullptr, &w);
}

int goslam_mvfilter_compute(const float* poses, const float* poses_world, const float* disps,
                            const float* intrinsic, float filter_thresh, int visible_num, int kernel_size, int T,
                            int ht, int wd, void* workspace, size_t workspace_bytes, void* stream) {
  if (T < 0 || T > 65535 || ht <= 0 || wd <= 0 || kernel_size < 0) return GOSLAM_EINVAL;
  if ((size_t)ht * wd > (size_t)INT_MAX / 2) return GOSLAM_EINVAL;
  const int radius = kernel_size == 0 ? -1 : (kernel_size < 2 ? 0 : kernel_size / 2);
  if (radius > kMvMaxRadius) return GOSLAM_EINVAL;
  const int hw = ht * wd;
  MvWork w;
  if (!workspace || workspace_bytes < mv_layout(T, (size_t)hw, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  mv_mean_kernel<<<T > 0 ? T : 1, kMvMeanThreads, 0, s>>>(disps, w.mean, w.st, T, hw);
  GS_CHECK_LAUNCH();
  if (T == 0) return GOSLAM_OK;
  const dim3 grid(gs_cdiv(hw, kMvTile), T);
  mv_vote_kernel<<<grid, kThreads, 0, s>>>(poses, poses_world, disps, intrinsic, w.mean, filter_thresh,
                                           (float)visible_num, w.mask1, w.st, T, ht, wd);
  GS_CHECK_LAUNCH();
  mv_extend_kernel<<<grid, kThreads, 0, s>>>(poses_world, disps, intrinsic, w.mask1, w.fin, w.st, radius, ht, wd);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_mvfilter_commit(const float* poses, const float* disps, const void* workspace, size_t workspace_bytes,
                           int T, int ht, int wd, float* poses_filtered, float* disps_filtered, float* mask_filtered,
                           float* update_priority, int* filtered_id, float* bound, int64_t* status, void* stream) {
  if (T < 0 || T > 65535 || ht <= 0 || wd <= 0) return GOSLAM_EINVAL;
  if ((size_t)ht * wd > (size_t)INT_MAX / 2) return GOSLAM_EINVAL;
  MvWork w;
  if (!workspace || workspace_bytes < mv_layout(T, (size_t)ht * wd, workspace, &w)) return GOSLAM_EWORKSPACE;
  const size_t n = (size_t)T * ht * wd;
  const size_t want = std::max<size_t>((n / 4 + kThreads - 1) / kThreads, (size_t)gs_cdiv(T, kThreads));
  const int blocks = (int)std::min<size_t>(std::max<size_t>(want, 1), 4096);
  mv_commit_kernel<<<blocks, kThreads, 0, (cudaStream_t)stream>>>(
      poses, disps, w.fin, w.st, T, n, poses_filtered, disps_filtered, mask_filtered, update_priority, filtered_id,
      bound, status);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

size_t goslam_mapping_points_workspace_bytes(int T, int ht, int wd) {
  if (T < 1 || T > 65535 || ht <= 0 || wd <= 0 || (size_t)ht * wd > (size_t)INT_MAX / 2) return 0;
  MapWork w;
  return map_layout(T, (size_t)ht * wd, nullptr, &w);
}

int goslam_mapping_points_count(const float* poses, const float* poses_world, const float* disps,
                                const float* intrinsic, int T, int ht, int wd, void* workspace, size_t workspace_bytes,
                                int64_t* count, void* stream) {
  if (T < 1 || T > 65535 || ht <= 0 || wd <= 0 || count == nullptr) return GOSLAM_EINVAL;
  if ((size_t)ht * wd > (size_t)INT_MAX / 2) return GOSLAM_EINVAL;
  const int hw = ht * wd;
  MapWork w;
  if (!workspace || workspace_bytes < map_layout(T, (size_t)hw, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  mv_mean_kernel<<<T, kMvMeanThreads, 0, s>>>(disps, w.mean, w.st, T, hw);
  GS_CHECK_LAUNCH();
  mv_vote_kernel<<<dim3(gs_cdiv(hw, kMvTile), T), kThreads, 0, s>>>(poses, poses_world, disps, intrinsic, w.mean,
                                                                     kMapThresh, kMapVisible, w.mask1, w.st, T, ht, wd);
  GS_CHECK_LAUNCH();
  GS_CUDA(cudaMemcpyAsync(count, &w.st->n1, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
  return GOSLAM_OK;
}

int goslam_mapping_points_emit(const float* poses_world, const float* disps, const float* intrinsic, int T, int ht,
                               int wd, void* workspace, size_t workspace_bytes, double* points, int64_t n_points,
                               void* stream) {
  if (T < 1 || T > 65535 || ht <= 0 || wd <= 0 || n_points < 0 || (n_points > 0 && points == nullptr))
    return GOSLAM_EINVAL;
  if ((size_t)ht * wd > (size_t)INT_MAX / 2) return GOSLAM_EINVAL;
  const int hw = ht * wd;
  const long long n = (long long)T * hw;
  if (n_points > n) return GOSLAM_EINVAL;
  MapWork w;
  if (!workspace || workspace_bytes < map_layout(T, (size_t)hw, workspace, &w)) return GOSLAM_EWORKSPACE;
  if (n_points == 0) return GOSLAM_OK;
  size_t tb = w.tmp_bytes;
  const MapIter it(cub::CountingInputIterator<long long>(0), MapPointOp{poses_world, disps, intrinsic, hw, wd});
  GS_CUDA(cub::DeviceSelect::Flagged(w.tmp, tb, it, (const unsigned char*)w.mask1, reinterpret_cast<MapPoint3*>(points),
                                     w.nsel, n, (cudaStream_t)stream));
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
