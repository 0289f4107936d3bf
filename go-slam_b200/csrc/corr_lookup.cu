// corr_lookup.cu — radius-r bilinear window lookup into the 4D correlation volume.
//
// Reference: corr_index_forward_kernel (src/lib/correlation_kernels.cu:19-70) driven once
// per pyramid level by CorrBlock.__call__ (src/modules/corr.py:43-53).
//
// Layout/roofline: volume[n][y][x] is one (h2 x w2) plane per SOURCE pixel, so the 8x8
// tap windows of neighbouring source pixels live in different planes — a pure gather of
// 8 rows x 8 contiguous elements per (pixel, level).  Work decomposition:
//   * 8 lanes per source pixel, one lane per window row; fp16 rows are fetched as two
//     aligned 128-bit loads (the 8 taps start at an arbitrary element) and re-aligned in
//     registers with a 2-level mux + funnel shift;
//   * the row below comes from lane+1 by warp shuffle (4 x 32-bit for fp16);
//   * results for a tile of kTile consecutive source pixels are staged in shared memory
//     and written channel-major with full-sector coalesced stores (out[n][c][k]).
// The fused entry point does all pyramid levels for a tile in one block, reading the
// coordinates once.
//
// Arithmetic contract (bit-exact with the reference instantiations):
//   f32: acc = fma(s11,w11, fma(s10,w10, fma(s01,w01, s00*w00)))   in the reference's
//        tap order (x outer, y inner);
//   f16: every product and every add is rounded to half, weights rounded to half first —
//        what `corr += s * scalar_t(w)` does for c10::Half (src/lib/correlation_kernels.cu:53-63).
// A tap outside the level adds nothing, as the reference's within_bounds test has it.  With a finite
// coordinate the zeroed taps give the same sums.  A NaN or infinite one makes every weight NaN, so a
// rarely taken branch gives the outside taps weight 0: an output whose four taps all lie outside is 0,
// the others NaN, as in the reference (float-to-int conversion takes NaN to 0 and saturates).  Window
// origins are clamped to +-2^30 first, so that the tap indices of a huge or infinite coordinate cannot
// overflow; every tap of a clamped origin is outside the level.
#include "common.cuh"

namespace {

constexpr int kTile = 64;       // source pixels per block
constexpr int kThreadsL = 256;  // 8 warps x 4 pixels x 8 row-lanes
constexpr int kMaxLevels = 4;

struct LookupArgs {
  const void* vol[kMaxLevels];
  int h2[kMaxLevels], w2[kMaxLevels];
  float inv_scale[kMaxLevels];
  int num_levels;
  const float* coords;   // planar [N,2,h1,w1] or interleaved [N,h1,w1,2]
  int interleaved;
  void* out;             // [N, num_levels*rd*rd, h1*w1]
  int N, hw1, radius;
  const int* slot;       // optional edge -> volume slot table (CorrPool); nullptr = identity
  int cap;               // slots in the volume allocation (N when slot == nullptr)
  int w4[kMaxLevels];    // > 0: the level is stored as 4x4 tiles, w4 tiles per tile-row (f16 only)
  long long plane[kMaxLevels];   // elements per source-pixel plane
  // otherwise row y starts at element (y >> rsh) * pitch + (y & rsh) * wrow   (rsh in {0, 1};
  // reference layout: rsh = 0, pitch = w2)
  int rsh[kMaxLevels], pitch[kMaxLevels], wrow[kMaxLevels];
  const int* alias;      // optional level-0 alias table, 4 words per slot (goslam_corr_pool_lookup_aliased)
};

// ---- row fetch: 8 consecutive elements starting at absolute element index e0 ----------
// Returns taps as 4 packed half2 words (fp16 path).
__device__ __forceinline__ void fetch_row8_h(const __half* __restrict__ base, long long e0,
                                             long long total, uint32_t (&w)[4]) {
  const long long c0 = e0 >> 3;               // 16-byte chunk index (8 halves)
  const int s = (int)(e0 & 7);
  uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
  const long long nchunk = total >> 3;        // full chunks only
  if (c0 >= 0 && c0 < nchunk) {
    a = __ldg(reinterpret_cast<const uint4*>(base) + c0);
  } else if (c0 >= 0 && c0 * 8 < total) {     // ragged tail of the allocation
    __half t[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) t[i] = (c0 * 8 + i < total) ? base[c0 * 8 + i] : __half(0.f);
    a = *reinterpret_cast<uint4*>(t);
  }
  if (s != 0) {
    const long long c1 = c0 + 1;
    if (c1 >= 0 && c1 < nchunk) {
      b = __ldg(reinterpret_cast<const uint4*>(base) + c1);
    } else if (c1 >= 0 && c1 * 8 < total) {
      __half t[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) t[i] = (c1 * 8 + i < total) ? base[c1 * 8 + i] : __half(0.f);
      b = *reinterpret_cast<uint4*>(t);
    }
  }
  // 8 words = 16 halves; want halves [s, s+8)
  const uint32_t v0 = a.x, v1 = a.y, v2 = a.z, v3 = a.w, v4 = b.x, v5 = b.y, v6 = b.z, v7 = b.w;
  const int q = s >> 1;
  const bool q2 = (q & 2) != 0, q1 = (q & 1) != 0;
  const uint32_t t0 = q2 ? v2 : v0, t1 = q2 ? v3 : v1, t2 = q2 ? v4 : v2, t3 = q2 ? v5 : v3,
                 t4 = q2 ? v6 : v4, t5 = q2 ? v7 : v5;
  const uint32_t u0 = q1 ? t1 : t0, u1 = q1 ? t2 : t1, u2 = q1 ? t3 : t2, u3 = q1 ? t4 : t3,
                 u4 = q1 ? t5 : t4;
  const uint32_t sh = (s & 1) * 16;
  w[0] = __funnelshift_r(u0, u1, sh);
  w[1] = __funnelshift_r(u1, u2, sh);
  w[2] = __funnelshift_r(u2, u3, sh);
  w[3] = __funnelshift_r(u3, u4, sh);
}

// Tiled level (4x4-element tiles, tile-row-major): the 8 taps of window row y1 starting at column
// x1 are sub-row (y1 & 3) of tiles tx0, tx0+1, tx0+2 of tile-row (y1 >> 2): three aligned 8-byte
// loads, re-aligned in registers.  Tiles outside [0, w4) read as zero.
__device__ __forceinline__ void fetch_row8_tiled_h(const __half* __restrict__ plane, int y1, int x1,
                                                   int w4, uint32_t (&w)[4]) {
  const int ty = y1 >> 2, r = y1 & 3;
  const int tx0 = x1 >> 2;                    // floor, also for negative x1
  const int a = x1 & 3;
  const uint2* rowp = reinterpret_cast<const uint2*>(plane + ((size_t)ty * w4) * 16 + r * 4);
  uint2 t[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int tx = tx0 + i;
    t[i] = (tx >= 0 && tx < w4 && (i < 2 || a != 0)) ? __ldg(rowp + (size_t)tx * 4) : make_uint2(0u, 0u);
  }
  const uint32_t v0 = t[0].x, v1 = t[0].y, v2 = t[1].x, v3 = t[1].y, v4 = t[2].x, v5 = t[2].y;
  const bool q = (a & 2) != 0;
  const uint32_t u0 = q ? v1 : v0, u1 = q ? v2 : v1, u2 = q ? v3 : v2, u3 = q ? v4 : v3, u4 = q ? v5 : v4;
  const uint32_t sh = (a & 1) * 16;
  w[0] = __funnelshift_r(u0, u1, sh);
  w[1] = __funnelshift_r(u1, u2, sh);
  w[2] = __funnelshift_r(u2, u3, sh);
  w[3] = __funnelshift_r(u3, u4, sh);
}

// Transposed level 0 (a reader edge, goslam_corr_pool_lookup_aliased): tap (y1, x1 + t) of source pixel q is
// element q (tiled offset qoff) of plane y1 * w2 + x1 + t of the holder slot.  Columns outside [0, w2) read as
// zero; the taps fill the words fetch_row8_tiled_h fills.
__device__ __forceinline__ void fetch_row8_transposed_h(const __half* __restrict__ vol, long long plane_base, int y1,
                                                        int x1, int w2, long long plane, int qoff, uint32_t (&w)[4]) {
  const unsigned short* row = reinterpret_cast<const unsigned short*>(vol) + plane_base +
                              (long long)y1 * w2 * plane + qoff;
  uint32_t t[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int x = x1 + i;
    t[i] = (x >= 0 && x < w2) ? (uint32_t)__ldg(row + (long long)x * plane) : 0u;
  }
#pragma unroll
  for (int m = 0; m < 4; ++m) w[m] = t[2 * m] | (t[2 * m + 1] << 16);
}

__device__ __forceinline__ __half2 u2h2(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }
__device__ __forceinline__ uint32_t h22u(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

// floor(x) as the device converts it (NaN -> 0, saturating), clamped so that the taps' indices cannot overflow
constexpr int kFarOrigin = 1 << 30;
__device__ __forceinline__ int origin(float f) { return min(max((int)f, -kFarOrigin), kFarOrigin); }

// zero the taps whose column x1+t is outside [0,w2)
__device__ __forceinline__ void mask_cols_h(uint32_t (&w)[4], int x1, int w2) {
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    const bool lo = (x1 + 2 * m >= 0) && (x1 + 2 * m < w2);
    const bool hi = (x1 + 2 * m + 1 >= 0) && (x1 + 2 * m + 1 < w2);
    w[m] &= (lo ? 0x0000ffffu : 0u) | (hi ? 0xffff0000u : 0u);
  }
}

// ------------------------------------------------------------------------------------
// One (level, 32-pixel half-tile) pass for a warp-group: every lane owns window row `row`
// of pixel `p`; writes rd*rd results for its pixel into the smem stage.
// ------------------------------------------------------------------------------------
template <int R>
__device__ __forceinline__ void lookup_pass_h(const __half* __restrict__ vol, long long total,
                                              long long plane_base, int h2, int w2, int w4, int rsh,
                                              int pitch, int wrow, float x0,
                                              float y0, int row, bool active, __half* stage,
                                              int stage_ld, int px_in_tile, long long plane, int qoff) {
  constexpr int RD = 2 * R + 1;
  static_assert(RD + 1 == 8, "row-lane mapping assumes radius 3 (8-tap windows)");
  const float fx0 = floorf(x0), fy0 = floorf(y0);
  const float dx = x0 - fx0, dy = y0 - fy0;
  const int x1 = origin(fx0) - R;
  const int y1 = origin(fy0) - R + row;

  uint32_t own[4] = {0, 0, 0, 0};
  if (active && y1 >= 0 && y1 < h2 && x1 > -8 && x1 < w2) {
    if (qoff >= 0) fetch_row8_transposed_h(vol, plane_base, y1, x1, w2, plane, qoff, own);
    else if (w4 > 0) fetch_row8_tiled_h(vol + plane_base, y1, x1, w4, own);
    else fetch_row8_h(vol, plane_base + (long long)(y1 >> rsh) * pitch + (y1 & rsh) * wrow + x1, total, own);
    mask_cols_h(own, x1, w2);
  }
  uint32_t dn[4];
#pragma unroll
  for (int m = 0; m < 4; ++m) dn[m] = __shfl_down_sync(0xffffffffu, own[m], 1);

  // weights, rounded to half exactly like scalar_t(dx*dy) etc.
  const __half2 w00 = __float2half2_rn((1.0f - dx) * (1.0f - dy));
  const __half2 w01 = __float2half2_rn((1.0f - dx) * dy);
  const __half2 w10 = __float2half2_rn(dx * (1.0f - dy));
  const __half2 w11 = __float2half2_rn(dx * dy);

  if (row < RD && active) {
    if (__builtin_expect(dx == dx && dy == dy, 1)) {       // dx, dy are NaN iff x0 or y0 is not finite
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        // P = taps (2m, 2m+1), Q = taps (2m+1, 2m+2)
        const uint32_t ownn = (m < 3) ? own[m + 1] : 0u;
        const uint32_t dnn = (m < 3) ? dn[m + 1] : 0u;
        const __half2 P = u2h2(own[m]), Pd = u2h2(dn[m]);
        const __half2 Q = u2h2(__funnelshift_r(own[m], ownn, 16));
        const __half2 Qd = u2h2(__funnelshift_r(dn[m], dnn, 16));
        __half2 acc = __hmul2_rn(P, w00);
        acc = __hadd2_rn(acc, __hmul2_rn(Pd, w01));
        acc = __hadd2_rn(acc, __hmul2_rn(Q, w10));
        acc = __hadd2_rn(acc, __hmul2_rn(Qd, w11));
        // outputs i = 2m (low), 2m+1 (high); channel = i*RD + row
        stage[(2 * m * RD + row) * stage_ld + px_in_tile] = __low2half(acc);
        if (2 * m + 1 < RD) stage[((2 * m + 1) * RD + row) * stage_ld + px_in_tile] = __high2half(acc);
      }
    } else {
      // non-finite coordinate: the same sums with each outside tap's weight masked to 0
      uint32_t cp[4] = {~0u, ~0u, ~0u, ~0u}, cq[4] = {~0u, ~0u, ~0u, ~0u};
      mask_cols_h(cp, x1, w2);                              // columns of taps (2m, 2m+1)
      mask_cols_h(cq, x1 + 1, w2);                          // columns of taps (2m+1, 2m+2)
      const uint32_t r0 = (y1 >= 0 && y1 < h2) ? ~0u : 0u, r1 = (y1 + 1 >= 0 && y1 + 1 < h2) ? ~0u : 0u;
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const uint32_t ownn = (m < 3) ? own[m + 1] : 0u;
        const uint32_t dnn = (m < 3) ? dn[m + 1] : 0u;
        const __half2 P = u2h2(own[m]), Pd = u2h2(dn[m]);
        const __half2 Q = u2h2(__funnelshift_r(own[m], ownn, 16));
        const __half2 Qd = u2h2(__funnelshift_r(dn[m], dnn, 16));
        __half2 acc = __hmul2_rn(P, u2h2(h22u(w00) & cp[m] & r0));
        acc = __hadd2_rn(acc, __hmul2_rn(Pd, u2h2(h22u(w01) & cp[m] & r1)));
        acc = __hadd2_rn(acc, __hmul2_rn(Q, u2h2(h22u(w10) & cq[m] & r0)));
        acc = __hadd2_rn(acc, __hmul2_rn(Qd, u2h2(h22u(w11) & cq[m] & r1)));
        stage[(2 * m * RD + row) * stage_ld + px_in_tile] = __low2half(acc);
        if (2 * m + 1 < RD) stage[((2 * m + 1) * RD + row) * stage_ld + px_in_tile] = __high2half(acc);
      }
    }
  }
}

template <int R>
__device__ __forceinline__ void lookup_pass_f(const float* __restrict__ vol, long long plane_base,
                                              int h2, int w2, float x0, float y0, int row,
                                              bool active, float* stage, int stage_ld,
                                              int px_in_tile) {
  constexpr int RD = 2 * R + 1;
  const float fx0 = floorf(x0), fy0 = floorf(y0);
  const float dx = x0 - fx0, dy = y0 - fy0;
  const int x1 = origin(fx0) - R;
  const int y1 = origin(fy0) - R + row;
  float own[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) own[t] = 0.f;
  if (active && y1 >= 0 && y1 < h2) {
    const float* rowp = vol + plane_base + (long long)y1 * w2;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int xx = x1 + t;
      if (xx >= 0 && xx < w2) own[t] = __ldg(rowp + xx);
    }
  }
  float dn[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) dn[t] = __shfl_down_sync(0xffffffffu, own[t], 1);
  const float w00 = (1.0f - dx) * (1.0f - dy), w01 = (1.0f - dx) * dy;
  const float w10 = dx * (1.0f - dy), w11 = dx * dy;
  if (row < RD && active) {
    if (__builtin_expect(dx == dx && dy == dy, 1)) {       // dx, dy are NaN iff x0 or y0 is not finite
#pragma unroll
      for (int i = 0; i < RD; ++i) {
        float acc = __fmul_rn(own[i], w00);
        acc = __fmaf_rn(dn[i], w01, acc);
        acc = __fmaf_rn(own[i + 1], w10, acc);
        acc = __fmaf_rn(dn[i + 1], w11, acc);
        stage[(i * RD + row) * stage_ld + px_in_tile] = acc;
      }
    } else {
      // non-finite coordinate: the same sums with each outside tap's weight masked to 0
      const bool r0 = y1 >= 0 && y1 < h2, r1 = y1 + 1 >= 0 && y1 + 1 < h2;
#pragma unroll
      for (int i = 0; i < RD; ++i) {
        const bool c0 = x1 + i >= 0 && x1 + i < w2, c1 = x1 + i + 1 >= 0 && x1 + i + 1 < w2;
        float acc = __fmul_rn(own[i], c0 && r0 ? w00 : 0.f);
        acc = __fmaf_rn(dn[i], c0 && r1 ? w01 : 0.f, acc);
        acc = __fmaf_rn(own[i + 1], c1 && r0 ? w10 : 0.f, acc);
        acc = __fmaf_rn(dn[i + 1], c1 && r1 ? w11 : 0.f, acc);
        stage[(i * RD + row) * stage_ld + px_in_tile] = acc;
      }
    }
  }
}

template <typename T, int R>
__global__ void __launch_bounds__(kThreadsL)
corr_lookup_kernel(const LookupArgs a) {
  constexpr int RD = 2 * R + 1;
  constexpr int CH = RD * RD;
  constexpr int LD = kTile + 8;   // padded leading dim of the stage (elements)
  __shared__ __align__(16) T stage[CH * LD];

  const int n = blockIdx.y;
  const int nv = a.slot ? __ldg(a.slot + n) : n;      // where this edge's volume lives
  const int al = a.alias ? __ldg(a.alias + 4 * (size_t)nv) : 2 * nv;   // ... and its level 0 (holder slot, transposed)
  const int k0 = blockIdx.x * kTile;
  const int lane8 = threadIdx.x & 7;          // window row
  const int pslot = threadIdx.x >> 3;         // 0..31 pixel slot within a pass

  // coordinates of the (up to) two pixels this thread serves
  float cx[2], cy[2];
  bool act[2];
#pragma unroll
  for (int ps = 0; ps < 2; ++ps) {
    const int k = k0 + ps * 32 + pslot;
    act[ps] = k < a.hw1;
    cx[ps] = 0.f; cy[ps] = 0.f;
    if (act[ps]) {
      if (a.interleaved) {
        const float2 c = __ldg(reinterpret_cast<const float2*>(a.coords) + (size_t)n * a.hw1 + k);
        cx[ps] = c.x; cy[ps] = c.y;
      } else {
        cx[ps] = __ldg(a.coords + ((size_t)n * 2 + 0) * a.hw1 + k);
        cy[ps] = __ldg(a.coords + ((size_t)n * 2 + 1) * a.hw1 + k);
      }
    }
  }

  for (int lvl = 0; lvl < a.num_levels; ++lvl) {
    const int h2 = a.h2[lvl], w2 = a.w2[lvl];
    const long long plane = a.plane[lvl];
    const long long total = (long long)a.cap * a.hw1 * plane;
    const T* vol = reinterpret_cast<const T*>(a.vol[lvl]);
    const float sc = a.inv_scale[lvl];
    // per edge (blockIdx.y), so no divergence: a transposed level 0 is read as element k of the holder's planes
    const bool tr = lvl == 0 && (al & 1);
#pragma unroll
    for (int ps = 0; ps < 2; ++ps) {
      const int k = k0 + ps * 32 + pslot;
      const long long pbase = tr ? (long long)(al >> 1) * a.hw1 * plane
                                 : ((long long)(lvl == 0 ? al >> 1 : nv) * a.hw1 + k) * plane;
      if constexpr (sizeof(T) == 2) {
        const int qy = k / w2, qx = k - qy * w2;
        const int qoff = tr ? ((qy >> 2) * a.w4[0] + (qx >> 2)) * 16 + (qy & 3) * 4 + (qx & 3) : -1;
        lookup_pass_h<R>(reinterpret_cast<const __half*>(vol), total, pbase, h2, w2, a.w4[lvl], a.rsh[lvl],
                         a.pitch[lvl], a.wrow[lvl], cx[ps] * sc,
                         cy[ps] * sc, lane8, act[ps], reinterpret_cast<__half*>(stage), LD,
                         ps * 32 + pslot, plane, qoff);
      } else {
        lookup_pass_f<R>(reinterpret_cast<const float*>(vol), pbase, h2, w2, cx[ps] * sc,
                         cy[ps] * sc, lane8, act[ps], reinterpret_cast<float*>(stage), LD,
                         ps * 32 + pslot);
      }
    }
    __syncthreads();
    // coalesced channel-major store of the [CH][kTile] stage
    T* outp = reinterpret_cast<T*>(a.out) +
              ((size_t)n * a.num_levels * CH + (size_t)lvl * CH) * a.hw1 + k0;
    const int npx = min(kTile, a.hw1 - k0);
    if (sizeof(T) == 2 && (a.hw1 & 7) == 0) {
      // 16-byte pieces: channel rows start 16-byte aligned in both the stage (LD*2 = 144 B) and the output
      for (int idx = threadIdx.x; idx < CH * (kTile / 8); idx += kThreadsL) {
        const int c = idx / (kTile / 8), p = (idx % (kTile / 8)) * 8;
        if (p < npx)
          *reinterpret_cast<uint4*>(outp + (size_t)c * a.hw1 + p) = *reinterpret_cast<const uint4*>(stage + c * LD + p);
      }
    } else {
      for (int idx = threadIdx.x; idx < CH * kTile; idx += kThreadsL) {
        const int c = idx / kTile, p = idx % kTile;
        if (p < npx) outp[(size_t)c * a.hw1 + p] = stage[c * LD + p];
      }
    }
    __syncthreads();
  }
}

template <typename T>
int launch_lookup(const LookupArgs& a, cudaStream_t st) {
  if (a.radius != 3) return GOSLAM_EINVAL;   // the reference only ever uses r = 3
  dim3 grid(gs_cdiv(a.hw1, kTile), a.N);
  corr_lookup_kernel<T, 3><<<grid, kThreadsL, 0, st>>>(a);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // namespace

extern "C" {

int goslam_corr_index_forward(const void* volume, int dtype, const float* coords, void* corr,
                              int N, int h1, int w1, int h2, int w2, int radius, void* stream) {
  if (N < 0 || h1 <= 0 || w1 <= 0 || h2 <= 0 || w2 <= 0) return GOSLAM_EINVAL;
  if (N == 0) return GOSLAM_OK;
  LookupArgs a{};
  a.vol[0] = volume; a.h2[0] = h2; a.w2[0] = w2; a.inv_scale[0] = 1.0f;
  a.w4[0] = 0; a.plane[0] = (long long)h2 * w2; a.rsh[0] = 0; a.pitch[0] = w2; a.wrow[0] = w2;
  a.num_levels = 1; a.coords = coords; a.interleaved = 0; a.out = corr;
  a.N = N; a.hw1 = h1 * w1; a.radius = radius; a.slot = nullptr; a.cap = N;
  if (dtype == GOSLAM_F16) return launch_lookup<__half>(a, (cudaStream_t)stream);
  if (dtype == GOSLAM_F32) return launch_lookup<float>(a, (cudaStream_t)stream);
  return GOSLAM_EINVAL;
}

int goslam_corr_pyramid_lookup(const void* const* pyramid, int dtype, int num_levels,
                               const float* coords_hw2, void* out, int N, int h1, int w1, int h2,
                               int w2, int radius, void* stream) {
  return goslam_corr_pool_lookup(pyramid, dtype, num_levels, nullptr, N, GOSLAM_LAYOUT_ROWMAJOR, coords_hw2,
                                 out, N, h1, w1, h2, w2, radius, stream);
}

int goslam_corr_pool_lookup(const void* const* pyramid, int dtype, int num_levels, const int* slots,
                            int capacity, int layout, const float* coords_hw2, void* out, int N, int h1,
                            int w1, int h2, int w2, int radius, void* stream) {
  return goslam_corr_pool_lookup_aliased(pyramid, dtype, num_levels, slots, nullptr, capacity, layout, coords_hw2,
                                         out, N, h1, w1, h2, w2, radius, stream);
}

int goslam_corr_pool_lookup_aliased(const void* const* pyramid, int dtype, int num_levels, const int* slots,
                                    const int* alias, int capacity, int layout, const float* coords_hw2,
                                    void* out, int N, int h1, int w1, int h2, int w2, int radius,
                                    void* stream) {
  if (N < 0 || h1 <= 0 || w1 <= 0 || num_levels < 1 || num_levels > kMaxLevels || capacity < N)
    return GOSLAM_EINVAL;
  if (layout != GOSLAM_LAYOUT_ROWMAJOR && layout != GOSLAM_LAYOUT_TILED) return GOSLAM_EINVAL;
  if (layout == GOSLAM_LAYOUT_TILED && dtype != GOSLAM_F16) return GOSLAM_EINVAL;
  if (alias != nullptr && (layout != GOSLAM_LAYOUT_TILED || h1 != h2 || w1 != w2)) return GOSLAM_EINVAL;
  if (N == 0) return GOSLAM_OK;
  LookupArgs a{};
  for (int i = 0; i < num_levels; ++i) {
    a.vol[i] = pyramid[i];
    a.h2[i] = h2 >> i; a.w2[i] = w2 >> i;          // floor, as F.avg_pool2d(2,2) produces
    a.inv_scale[i] = 1.0f / (float)(1 << i);       // coords / 2**i (exact)
    if (a.h2[i] <= 0 || a.w2[i] <= 0) return GOSLAM_EINVAL;
    a.plane[i] = (long long)goslam_corr_level_plane_elems(i, layout, h2, w2);
    a.w4[i] = 0; a.rsh[i] = 0; a.pitch[i] = a.w2[i]; a.wrow[i] = a.w2[i];
    if (layout == GOSLAM_LAYOUT_TILED) {
      const int n_xb = gs_cdiv(w2, 16);
      if (i < 2) a.w4[i] = gs_cdiv(a.w2[i], 4);
      else if (i == 2) { a.rsh[i] = 1; a.wrow[i] = n_xb * 4; a.pitch[i] = (n_xb * 8 + 15) / 16 * 16; }
      else { a.pitch[i] = 16; a.wrow[i] = 16; }
    }
  }
  a.num_levels = num_levels; a.coords = coords_hw2; a.interleaved = 1; a.out = out;
  a.N = N; a.hw1 = h1 * w1; a.radius = radius; a.slot = slots; a.cap = capacity; a.alias = alias;
  if (dtype == GOSLAM_F16) return launch_lookup<__half>(a, (cudaStream_t)stream);
  if (dtype == GOSLAM_F32) return launch_lookup<float>(a, (cudaStream_t)stream);
  return GOSLAM_EINVAL;
}

int goslam_corr_index_backward(void) { return GOSLAM_EUNSUPPORTED; }

}  // extern "C"
