// mesh_view.cu — the projection and component culls of Mesher.cull_mesh (src/mesher.py:56-240) on the device.
//
//  * depth rasterizer (extract_depth_from_mesh, :444-479): one thread per (face, view).  The face's vertices go to camera
//    space in fp64 (X = R^T (p - t), R and t the f32 entries of c2w), the triangle is clipped against z = znear (up to two
//    pieces), projected to pixels, and every pixel whose centre (c + 0.5, r + 0.5) lies inside or on the piece (inclusive
//    edge functions, either winding) gets the perspective-correct depth (1/z interpolated linearly in screen space).  The
//    nearest fragment wins through atomicMin on the float's bit pattern (positive floats order like their bits), so the
//    result does not depend on scheduling; pixels no fragment reaches hold 0.  A piece whose pixel box exceeds
//    kSmallPixels is not walked by its own thread: the warp takes the warp's large pieces one after another, 32 lanes
//    striding over the box (a full-screen quad is 2 x W*H / 32 pixels per lane instead of W*H for one thread).  Every
//    formula is evaluated operation by operation (__dmul_rn / __dadd_rn, no contraction) so that the numpy restatement
//    (oracle/mesh_view_oracle.py) reproduces the depth bit for bit.
//  * view masks (point_masks, :56-136): one thread per vertex loops over a chunk of views in f32, torch's order of
//    operations; grid_sample (bilinear, border, align_corners=True) restated from torch's CUDA kernel.  The thread ORs into
//    the caller's u8 masks and stops early once both bits are set (OR is monotone).
//  * component filter (get_connected_mesh, :139-153): faces are adjacent when they share an edge that belongs to exactly
//    two faces (sorted edge keys, CUB radix sort); union-find hooks the larger root under the smaller one, so every
//    component's label is its smallest face id.  Face areas (fp64) are sorted by label (stable: face order inside a
//    component) and summed per component by CUB's segmented reduction: fixed order, no float atomics.
#include <cub/cub.cuh>

#include "common.cuh"
#include "mesh_geom.cuh"

namespace {

typedef unsigned long long u64;

constexpr int kRasterThreads = 256;
constexpr int kSmallPixels = 64;          // pieces with a larger pixel box are rasterized by the whole warp
constexpr unsigned kFull = 0xffffffffu;
constexpr unsigned kInfBits = 0x7f800000u;

long long cdiv64(long long a, long long b) { return (a + b - 1) / b; }

// ---- depth rasterizer -------------------------------------------------------------------------------------------
struct Cam { double fx, fy, cx, cy, znear, zfar; int H, W; };

struct V3 { double x, y, z; };

// a screen-space triangle: pixel coordinates, 1/z per vertex, twice the signed area, and the pixel box
struct Piece {
  double x0, y0, x1, y1, x2, y2, iz0, iz1, iz2, area;
  int c0, r0, bw, bh;
};

__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }

// a + t (b - a) at z = znear for a inside (z >= znear) and b outside
__device__ __forceinline__ V3 clip_point(const V3& a, const V3& b, double znear) {
  const double t = __ddiv_rn(dsub(znear, a.z), dsub(b.z, a.z));
  return V3{dadd(a.x, dmul(t, dsub(b.x, a.x))), dadd(a.y, dmul(t, dsub(b.y, a.y))), znear};
}

// the s-th (0 or 1) piece of the triangle a, b, c after the near clip, projected; false if there is none or it is empty
__device__ bool make_piece(V3 a, V3 b, V3 c, int s, const Cam& cam, Piece* p) {
  const bool ia = a.z >= cam.znear, ib = b.z >= cam.znear, ic = c.z >= cam.znear;
  const int nin = (int)ia + (int)ib + (int)ic;
  V3 q0, q1, q2;
  if (nin == 3) {
    if (s) return false;
    q0 = a; q1 = b; q2 = c;
  } else if (nin == 1) {
    if (s) return false;
    // rotate so that the inside vertex comes first (keeps the winding)
    V3 i = a, j = b, k = c;
    if (ib) { i = b; j = c; k = a; }
    if (ic) { i = c; j = a; k = b; }
    q0 = i; q1 = clip_point(i, j, cam.znear); q2 = clip_point(i, k, cam.znear);
  } else if (nin == 2) {
    // rotate so that the outside vertex comes first: o, i, j; the quad i, j, Q(j,o), Q(i,o)
    V3 o = a, i = b, j = c;
    if (!ib) { o = b; i = c; j = a; }
    if (!ic) { o = c; i = a; j = b; }
    if (s == 0) { q0 = i; q1 = j; q2 = clip_point(j, o, cam.znear); }
    else { q0 = i; q1 = clip_point(j, o, cam.znear); q2 = clip_point(i, o, cam.znear); }
  } else {
    return false;
  }
  p->x0 = dadd(dmul(cam.fx, __ddiv_rn(q0.x, q0.z)), cam.cx); p->y0 = dadd(dmul(cam.fy, __ddiv_rn(q0.y, q0.z)), cam.cy);
  p->x1 = dadd(dmul(cam.fx, __ddiv_rn(q1.x, q1.z)), cam.cx); p->y1 = dadd(dmul(cam.fy, __ddiv_rn(q1.y, q1.z)), cam.cy);
  p->x2 = dadd(dmul(cam.fx, __ddiv_rn(q2.x, q2.z)), cam.cx); p->y2 = dadd(dmul(cam.fy, __ddiv_rn(q2.y, q2.z)), cam.cy);
  p->iz0 = __drcp_rn(q0.z); p->iz1 = __drcp_rn(q1.z); p->iz2 = __drcp_rn(q2.z);
  p->area = dsub(dmul(dsub(p->x1, p->x0), dsub(p->y2, p->y0)), dmul(dsub(p->y1, p->y0), dsub(p->x2, p->x0)));
  if (!(p->area != 0.0) || !isfinite(p->area)) return false;
  // pixel box: centres c + 0.5 within [min x, max x], clamped to the image (in fp64 before any integer conversion)
  const double xmin = fmin(fmin(p->x0, p->x1), p->x2), xmax = fmax(fmax(p->x0, p->x1), p->x2);
  const double ymin = fmin(fmin(p->y0, p->y1), p->y2), ymax = fmax(fmax(p->y0, p->y1), p->y2);
  const double c0 = fmax(0.0, ceil(dsub(xmin, 0.5))), c1 = fmin((double)(cam.W - 1), floor(dsub(xmax, 0.5)));
  const double r0 = fmax(0.0, ceil(dsub(ymin, 0.5))), r1 = fmin((double)(cam.H - 1), floor(dsub(ymax, 0.5)));
  if (!(c0 <= c1) || !(r0 <= r1)) return false;
  p->c0 = (int)c0; p->r0 = (int)r0;
  p->bw = (int)c1 - p->c0 + 1; p->bh = (int)r1 - p->r0 + 1;
  return true;
}

__device__ __forceinline__ void shade(const Piece& p, int r, int c, const Cam& cam, float* depth) {
  const double px = (double)c + 0.5, py = (double)r + 0.5;
  const double e0 = dsub(dmul(dsub(p.x2, p.x1), dsub(py, p.y1)), dmul(dsub(p.y2, p.y1), dsub(px, p.x1)));
  const double e1 = dsub(dmul(dsub(p.x0, p.x2), dsub(py, p.y2)), dmul(dsub(p.y0, p.y2), dsub(px, p.x2)));
  const double e2 = dsub(dmul(dsub(p.x1, p.x0), dsub(py, p.y0)), dmul(dsub(p.y1, p.y0), dsub(px, p.x0)));
  const bool in = (e0 >= 0.0 && e1 >= 0.0 && e2 >= 0.0) || (e0 <= 0.0 && e1 <= 0.0 && e2 <= 0.0);
  if (!in) return;
  const double iz = dadd(dadd(dmul(__ddiv_rn(e0, p.area), p.iz0), dmul(__ddiv_rn(e1, p.area), p.iz1)),
                         dmul(__ddiv_rn(e2, p.area), p.iz2));
  const double z = __drcp_rn(iz);
  if (!(z > 0.0) || z > cam.zfar) return;
  atomicMin((unsigned*)depth + (long long)r * cam.W + c, __float_as_uint(__double2float_rn(z)));
}

__device__ __forceinline__ V3 to_camera(const double* verts, long long v, const double* R, const double* t) {
  const double d0 = dsub(verts[3 * v], t[0]), d1 = dsub(verts[3 * v + 1], t[1]), d2 = dsub(verts[3 * v + 2], t[2]);
  V3 q;
  q.x = dadd(dadd(dmul(R[0], d0), dmul(R[3], d1)), dmul(R[6], d2));
  q.y = dadd(dadd(dmul(R[1], d0), dmul(R[4], d1)), dmul(R[7], d2));
  q.z = dadd(dadd(dmul(R[2], d0), dmul(R[5], d1)), dmul(R[8], d2));
  return q;
}

// grid (ceil(F / 256), K); every thread of a warp reaches the ballots (no early return)
__global__ void __launch_bounds__(kRasterThreads) raster_kernel(const double* verts, long long nv, const long long* faces,
                                                                long long nf, const float* c2w, const Cam cam, float* depth) {
  const long long f = (long long)blockIdx.x * kRasterThreads + threadIdx.x;
  const int k = blockIdx.y;
  const int lane = threadIdx.x & 31;
  float* img = depth + (long long)k * cam.H * cam.W;
  double R[9], t[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) R[3 * i + j] = (double)__ldg(c2w + 16 * k + 4 * i + j);
    t[i] = (double)__ldg(c2w + 16 * k + 4 * i + 3);
  }
  bool valid = f < nf;
  long long ia = 0, ib = 0, ic = 0;
  if (valid) {
    ia = faces[3 * f]; ib = faces[3 * f + 1]; ic = faces[3 * f + 2];
    valid = ia >= 0 && ia < nv && ib >= 0 && ib < nv && ic >= 0 && ic < nv;
  }
  V3 a{0, 0, 1}, b{0, 0, 1}, c{0, 0, 1};
  if (valid) { a = to_camera(verts, ia, R, t); b = to_camera(verts, ib, R, t); c = to_camera(verts, ic, R, t); }
  for (int s = 0; s < 2; ++s) {
    Piece p;
    const bool ok = valid && make_piece(a, b, c, s, cam, &p);
    const bool big = ok && (long long)p.bw * p.bh > kSmallPixels;
    if (ok && !big) {
      for (int r = 0; r < p.bh; ++r)
        for (int q = 0; q < p.bw; ++q) shade(p, p.r0 + r, p.c0 + q, cam, img);
    }
    unsigned m = __ballot_sync(kFull, big);
    while (m) {
      const int src = __ffs(m) - 1;
      m &= m - 1;
      Piece g;
      g.x0 = __shfl_sync(kFull, p.x0, src); g.y0 = __shfl_sync(kFull, p.y0, src);
      g.x1 = __shfl_sync(kFull, p.x1, src); g.y1 = __shfl_sync(kFull, p.y1, src);
      g.x2 = __shfl_sync(kFull, p.x2, src); g.y2 = __shfl_sync(kFull, p.y2, src);
      g.iz0 = __shfl_sync(kFull, p.iz0, src); g.iz1 = __shfl_sync(kFull, p.iz1, src);
      g.iz2 = __shfl_sync(kFull, p.iz2, src); g.area = __shfl_sync(kFull, p.area, src);
      g.c0 = __shfl_sync(kFull, p.c0, src); g.r0 = __shfl_sync(kFull, p.r0, src);
      g.bw = __shfl_sync(kFull, p.bw, src); g.bh = __shfl_sync(kFull, p.bh, src);
      const int n = g.bw * g.bh;                       // at most H * W
      for (int i = lane; i < n; i += 32) {
        const int r = i / g.bw;
        shade(g, g.r0 + r, g.c0 + (i - r * g.bw), cam, img);
      }
    }
  }
}

__global__ void fill_kernel(unsigned* p, long long n, unsigned v) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

// +inf (no fragment) -> 0
__global__ void finalize_depth_kernel(unsigned* p, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (p[i] == kInfBits) p[i] = 0u;
}

// ---- view masks -------------------------------------------------------------------------------------------------
struct MaskCam { float fx, fy, cx, cy, radius, eps; int H, W; };

__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }

// F.grid_sample(depth[1,1,H,W], grid, 'bilinear', padding_mode='border', align_corners=True) at one grid point, as torch's
// CUDA kernel computes it: unnormalise ((g + 1) / 2) * (size - 1), clip to [0, size - 1], four taps in nw, ne, sw, se order
__device__ __forceinline__ float sample_border(const float* img, int H, int W, float gx, float gy) {
  float ix = fmul(__fdiv_rn(fadd(gx, 1.f), 2.f), (float)(W - 1));
  float iy = fmul(__fdiv_rn(fadd(gy, 1.f), 2.f), (float)(H - 1));
  ix = fminf((float)(W - 1), fmaxf(ix, 0.f));
  iy = fminf((float)(H - 1), fmaxf(iy, 0.f));
  const int x0 = (int)floorf(ix), y0 = (int)floorf(iy);
  const float x1f = (float)(x0 + 1), y1f = (float)(y0 + 1), x0f = (float)x0, y0f = (float)y0;
  const float nw = fmul(fsub(x1f, ix), fsub(y1f, iy));
  const float ne = fmul(fsub(ix, x0f), fsub(y1f, iy));
  const float sw = fmul(fsub(x1f, ix), fsub(iy, y0f));
  const float se = fmul(fsub(ix, x0f), fsub(iy, y0f));
  const bool xin = x0 + 1 < W, yin = y0 + 1 < H;
  float out = 0.f;
  out = fadd(out, fmul(__ldg(img + y0 * W + x0), nw));
  if (xin) out = fadd(out, fmul(__ldg(img + y0 * W + x0 + 1), ne));
  if (yin) out = fadd(out, fmul(__ldg(img + (y0 + 1) * W + x0), sw));
  if (xin && yin) out = fadd(out, fmul(__ldg(img + (y0 + 1) * W + x0 + 1), se));
  return out;
}

__global__ void __launch_bounds__(256) mask_kernel(const double* verts, long long nv, const float* w2c, const float* depth,
                                                   int K, const MaskCam cam, unsigned char* seen, unsigned char* forecast) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  bool s = seen[i] != 0, fc = forecast[i] != 0;
  if (s && fc) return;
  const float x = (float)verts[3 * i], y = (float)verts[3 * i + 1], z = (float)verts[3 * i + 2];
  const float wm1 = (float)(cam.W - 1), hm1 = (float)(cam.H - 1), r = cam.radius;
  const long long hw = (long long)cam.H * cam.W;
  for (int k = 0; k < K && !(s && fc); ++k) {
    const float* m = w2c + 16 * k;
    const float X = fadd(fadd(fadd(fmul(__ldg(m + 0), x), fmul(__ldg(m + 1), y)), fmul(__ldg(m + 2), z)), __ldg(m + 3));
    const float Y = fadd(fadd(fadd(fmul(__ldg(m + 4), x), fmul(__ldg(m + 5), y)), fmul(__ldg(m + 6), z)), __ldg(m + 7));
    const float Z = fadd(fadd(fadd(fmul(__ldg(m + 8), x), fmul(__ldg(m + 9), y)), fmul(__ldg(m + 10), z)), __ldg(m + 11));
    const float zz = fadd(Z, 1e-8f);
    const float u = __fdiv_rn(fadd(fmul(cam.fx, X), fmul(cam.cx, Z)), zz);
    const float v = __fdiv_rn(fadd(fmul(cam.fy, Y), fmul(cam.cy, Z)), zz);
    const bool in_f = u >= 0.f && u <= wm1 && v >= 0.f && v <= hm1 && zz > 0.f;
    const bool fc_f = u >= -r && u <= fadd(wm1, r) && v >= -r && v <= fadd(hm1, r) && zz > 0.f;
    if (!in_f && !fc_f) continue;
    const float gx = fsub(fmul(__fdiv_rn(u, wm1), 2.f), 1.f), gy = fsub(fmul(__fdiv_rn(v, hm1), 2.f), 1.f);
    const float d = sample_border(depth + k * hw, cam.H, cam.W, gx, gy);
    const bool front = d > 0.f ? zz < fadd(d, cam.eps) : true;
    s = s || (in_f && front);
    fc = fc || (fc_f && front) || (in_f && front);
  }
  seen[i] = s ? 1 : 0;
  forecast[i] = fc ? 1 : 0;
}

// ---- component filter -------------------------------------------------------------------------------------------
struct CompWork {
  u64* keys[2];          // edge keys (double buffer of the radix sort)
  unsigned* efaces[2];   // face of each edge
  unsigned* parent;      // union-find forest; after the count pass, the component label (smallest face id) of each face
  unsigned* labels[2];   // labels, then sorted
  double* area[2];       // face areas, then sorted by label
  unsigned* seg_begin;   // first sorted position of each component, [n_comp + 1]
  unsigned* seg_of_label;
  double* comp_area;     // [n_comp]
  unsigned char* comp_keep;
  void* cub_tmp;
  size_t cub_bytes;
};

struct IsRunStart {
  const unsigned* lab;
  __device__ bool operator()(unsigned i) const { return i == 0 || lab[i] != lab[i - 1]; }
};

// CUB's temporary storage for the largest of the count pass's calls (needs a device to size)
int comp_cub_bytes(long long nf, size_t* bytes) {
  const int ne = (int)(3 * nf), n = (int)nf;
  size_t a = 0, b = 0, c = 0, d = 0;
  cub::DoubleBuffer<u64> k(nullptr, nullptr);
  cub::DoubleBuffer<unsigned> v(nullptr, nullptr), l(nullptr, nullptr);
  cub::DoubleBuffer<double> ar(nullptr, nullptr);
  GS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, a, k, v, ne));
  GS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, l, ar, n));
  GS_CUDA(cub::DeviceSelect::If(nullptr, c, cub::CountingInputIterator<unsigned>(0), (unsigned*)nullptr, (long long*)nullptr,
                                n, IsRunStart{nullptr}));
  GS_CUDA(cub::DeviceSegmentedReduce::Sum(nullptr, d, (const double*)nullptr, (double*)nullptr, n, (const unsigned*)nullptr,
                                          (const unsigned*)nullptr));
  *bytes = std::max(std::max(a, b), std::max(c, d));
  return GOSLAM_OK;
}

size_t comp_layout(long long nf, size_t cub_bytes, void* base, CompWork* w) {
  GsArena ar(base);
  const long long ne = 3 * nf > 0 ? 3 * nf : 1, n = nf > 0 ? nf : 1;
  for (int i = 0; i < 2; ++i) {
    w->keys[i] = ar.take<u64>(ne);
    w->efaces[i] = ar.take<unsigned>(ne);
    w->labels[i] = ar.take<unsigned>(n);
    w->area[i] = ar.take<double>(n);
  }
  w->parent = ar.take<unsigned>(n);
  w->seg_begin = ar.take<unsigned>(n + 1);
  w->seg_of_label = ar.take<unsigned>(n);
  w->comp_area = ar.take<double>(n);
  w->comp_keep = ar.take<unsigned char>(n);
  w->cub_tmp = ar.take<unsigned char>(cub_bytes > 0 ? cub_bytes : 1);
  w->cub_bytes = cub_bytes;
  return ar.off;
}

// edge keys min * nv + max of the three (sorted) edges of each face, areas 0.5 |(v1 - v0) x (v2 - v0)| in fp64; a face
// with an index outside [0, nv) gets area 0 and three edge keys no other edge has
__global__ void __launch_bounds__(256) edge_kernel(const double* verts, long long nv, const long long* faces, long long nf,
                                                   u64* keys, unsigned* efaces, unsigned* parent, double* area) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  long long v[3];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    v[j] = faces[3 * f + j];
    ok = ok && v[j] >= 0 && v[j] < nv;
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const long long a = v[j], b = v[(j + 1) % 3];
    keys[3 * f + j] = ok ? (u64)(a < b ? a : b) * (u64)nv + (u64)(a < b ? b : a) : ~0ull - (u64)(3 * f + j);
    efaces[3 * f + j] = (unsigned)f;
  }
  parent[f] = (unsigned)f;
  area[f] = ok ? gs_face_area(verts + 3 * v[0], verts + 3 * v[1], verts + 3 * v[2]) : 0.0;
}

__device__ __forceinline__ unsigned find_root(const unsigned* parent, unsigned x) {
  unsigned p = ((volatile const unsigned*)parent)[x];
  while (p != x) { x = p; p = ((volatile const unsigned*)parent)[x]; }
  return x;
}

// for every run of exactly two equal edge keys: union the two faces, hooking the larger root under the smaller
__global__ void __launch_bounds__(256) union_kernel(const u64* keys, const unsigned* efaces, long long ne, unsigned* parent) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i + 1 >= ne) return;
  const u64 k = keys[i];
  if (keys[i + 1] != k || (i > 0 && keys[i - 1] == k) || (i + 2 < ne && keys[i + 2] == k)) return;
  unsigned a = efaces[i], b = efaces[i + 1];
  while (true) {
    a = find_root(parent, a);
    b = find_root(parent, b);
    if (a == b) return;
    if (a < b) { const unsigned t = a; a = b; b = t; }
    if (atomicCAS(parent + a, a, b) == a) return;
  }
}

__global__ void __launch_bounds__(256) label_kernel(const unsigned* parent, long long nf, unsigned* labels) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f < nf) labels[f] = find_root(parent, (unsigned)f);
}

__global__ void __launch_bounds__(256) seg_kernel(const unsigned* lab_sorted, const long long* n_comp, long long nf,
                                                  unsigned* seg_begin, unsigned* seg_of_label) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = *n_comp;
  if (s < n) seg_of_label[lab_sorted[seg_begin[s]]] = (unsigned)s;
  if (s == 0) seg_begin[n] = (unsigned)nf;
}

// one block: total area (per-thread strided sums, fixed tree) and the first component of largest area, then the verdicts
constexpr int kDecideThreads = 1024;
__global__ void __launch_bounds__(kDecideThreads) decide_kernel(const double* comp_area, long long n, double threshold,
                                                                int largest, unsigned char* keep) {
  __shared__ double s_sum[kDecideThreads];
  __shared__ double s_max[kDecideThreads];
  __shared__ long long s_arg[kDecideThreads];
  double sum = 0.0, best = -1.0;
  long long arg = -1;
  for (long long i = threadIdx.x; i < n; i += kDecideThreads) {
    const double a = comp_area[i];
    sum = dadd(sum, a);
    if (a > best) { best = a; arg = i; }
  }
  s_sum[threadIdx.x] = sum; s_max[threadIdx.x] = best; s_arg[threadIdx.x] = arg;
  __syncthreads();
  for (int h = kDecideThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      const int o = threadIdx.x + h;
      s_sum[threadIdx.x] = dadd(s_sum[threadIdx.x], s_sum[o]);
      const double bm = s_max[o];
      const long long ba = s_arg[o];
      if (ba >= 0 && (bm > s_max[threadIdx.x] || (bm == s_max[threadIdx.x] && ba < s_arg[threadIdx.x]) || s_arg[threadIdx.x] < 0)) {
        s_max[threadIdx.x] = bm; s_arg[threadIdx.x] = ba;
      }
    }
    __syncthreads();
  }
  const double limit = dmul(threshold, s_sum[0]);
  const long long top = s_arg[0];
  for (long long i = threadIdx.x; i < n; i += kDecideThreads)
    keep[i] = largest ? (i == top) : (comp_area[i] > limit);
}

__global__ void __launch_bounds__(256) face_keep_kernel(const unsigned* labels, const unsigned* seg_of_label,
                                                        const unsigned char* comp_keep, long long nf, unsigned char* out) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f < nf) out[f] = comp_keep[seg_of_label[labels[f]]];
}

unsigned blocks_for(long long n, int threads) { return (unsigned)cdiv64(n, threads); }

// faces and vertices are counted in u32 inside the component filter
constexpr long long kMaxCompFaces = (1ll << 31) - 1;

}  // namespace

extern "C" {

int goslam_mesh_depth_render(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const float* c2w,
                             int K, int H, int W, double fx, double fy, double cx, double cy, double znear, double zfar,
                             float* depth, void* stream) {
  if (n_verts < 0 || n_faces < 0 || K < 0 || H < 1 || W < 1 || (long long)H * W > (1ll << 30) || K > 65535 ||
      (n_verts > 0 && !verts) || (n_faces > 0 && !faces) || (K > 0 && (!c2w || !depth)) || !(znear > 0.0) ||
      !(zfar > znear) || !(fx == fx && fy == fy && cx == cx && cy == cy))
    return GOSLAM_EINVAL;
  if (K == 0) return GOSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)K * H * W;
  const unsigned fill_blocks = (unsigned)std::min<long long>(cdiv64(n, 256), 4 * 1024);
  fill_kernel<<<fill_blocks, 256, 0, st>>>((unsigned*)depth, n, kInfBits);
  GS_CHECK_LAUNCH();
  if (n_faces > 0) {
    const Cam cam{fx, fy, cx, cy, znear, zfar, H, W};
    raster_kernel<<<dim3(blocks_for(n_faces, kRasterThreads), (unsigned)K), kRasterThreads, 0, st>>>(
        verts, n_verts, (const long long*)faces, n_faces, c2w, cam, depth);
    GS_CHECK_LAUNCH();
  }
  finalize_depth_kernel<<<fill_blocks, 256, 0, st>>>((unsigned*)depth, n);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_mesh_view_masks(const double* verts, int64_t n_verts, const float* w2c, const float* depth, int K, int H, int W,
                           float fx, float fy, float cx, float cy, float radius, float eps, unsigned char* seen,
                           unsigned char* forecast, void* stream) {
  if (n_verts < 0 || K < 0 || H < 2 || W < 2 || (long long)H * W > (1ll << 30) || (n_verts > 0 && (!verts || !seen || !forecast)) ||
      (K > 0 && (!w2c || !depth)) || !(radius >= 0.f))
    return GOSLAM_EINVAL;
  if (K == 0 || n_verts == 0) return GOSLAM_OK;
  const MaskCam cam{fx, fy, cx, cy, radius, eps, H, W};
  mask_kernel<<<blocks_for(n_verts, 256), 256, 0, (cudaStream_t)stream>>>(verts, n_verts, w2c, depth, K, cam, seen, forecast);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

size_t goslam_mesh_components_workspace_bytes(int64_t n_verts, int64_t n_faces) {
  if (n_verts < 0 || n_faces < 0 || n_faces > kMaxCompFaces) return 0;
  size_t cb = 0;
  if (n_faces > 0 && comp_cub_bytes(n_faces, &cb) != GOSLAM_OK) return 0;
  CompWork w;
  return comp_layout(n_faces, cb, nullptr, &w);
}

int goslam_mesh_components_count(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, void* workspace,
                                 size_t workspace_bytes, int64_t* counts, void* stream) {
  if (n_verts < 0 || n_faces < 0 || n_faces > kMaxCompFaces || (n_verts > 0 && !verts) || (n_faces > 0 && !faces) || !counts)
    return GOSLAM_EINVAL;
  if (!workspace) return GOSLAM_EWORKSPACE;     // refused before the empty-input return and the CUB size query
  cudaStream_t st = (cudaStream_t)stream;
  if (n_faces == 0) {
    GS_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t), st));
    return GOSLAM_OK;
  }
  size_t cb = 0;
  if (const int rc = comp_cub_bytes(n_faces, &cb)) return rc;
  CompWork w;
  if (workspace_bytes < comp_layout(n_faces, cb, workspace, &w)) return GOSLAM_EWORKSPACE;
  const long long ne = 3 * n_faces;
  edge_kernel<<<blocks_for(n_faces, 256), 256, 0, st>>>(verts, n_verts, (const long long*)faces, n_faces, w.keys[0], w.efaces[0],
                                                        w.parent, w.area[0]);
  GS_CHECK_LAUNCH();
  cub::DoubleBuffer<u64> kb(w.keys[0], w.keys[1]);
  cub::DoubleBuffer<unsigned> fb(w.efaces[0], w.efaces[1]);
  size_t tb = w.cub_bytes;
  GS_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, tb, kb, fb, (int)ne, 0, 64, st));
  union_kernel<<<blocks_for(ne, 256), 256, 0, st>>>(kb.Current(), fb.Current(), ne, w.parent);
  GS_CHECK_LAUNCH();
  label_kernel<<<blocks_for(n_faces, 256), 256, 0, st>>>(w.parent, n_faces, w.labels[0]);
  GS_CHECK_LAUNCH();
  // the labels stay in labels[0] for the face verdicts: sort copies of them
  GS_CUDA(cudaMemcpyAsync(w.labels[1], w.labels[0], n_faces * sizeof(unsigned), cudaMemcpyDeviceToDevice, st));
  cub::DoubleBuffer<unsigned> lb(w.labels[1], (unsigned*)w.keys[0]);
  cub::DoubleBuffer<double> ab(w.area[0], w.area[1]);
  tb = w.cub_bytes;
  GS_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, tb, lb, ab, (int)n_faces, 0, 32, st));
  // keep the sorted labels and areas where the emit pass finds them
  if (lb.Current() != w.labels[1])
    GS_CUDA(cudaMemcpyAsync(w.labels[1], lb.Current(), n_faces * sizeof(unsigned), cudaMemcpyDeviceToDevice, st));
  if (ab.Current() != w.area[1])
    GS_CUDA(cudaMemcpyAsync(w.area[1], ab.Current(), n_faces * sizeof(double), cudaMemcpyDeviceToDevice, st));
  tb = w.cub_bytes;
  GS_CUDA(cub::DeviceSelect::If(w.cub_tmp, tb, cub::CountingInputIterator<unsigned>(0), w.seg_begin, (long long*)counts,
                                (int)n_faces, IsRunStart{w.labels[1]}, st));
  seg_kernel<<<blocks_for(n_faces, 256), 256, 0, st>>>(w.labels[1], (const long long*)counts, n_faces, w.seg_begin,
                                                       w.seg_of_label);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_mesh_components_keep(int64_t n_faces, int64_t n_components, double threshold, int largest, void* workspace,
                                size_t workspace_bytes, unsigned char* face_keep, void* stream) {
  if (n_faces < 0 || n_faces > kMaxCompFaces || n_components < 0 || n_components > n_faces || (n_faces > 0 && !face_keep) ||
      (n_faces > 0 && n_components == 0) || threshold != threshold)
    return GOSLAM_EINVAL;
  if (!workspace) return GOSLAM_EWORKSPACE;     // refused before the empty-input return and the CUB size query
  if (n_faces == 0) return GOSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  size_t cb = 0;
  if (const int rc = comp_cub_bytes(n_faces, &cb)) return rc;
  CompWork w;
  if (workspace_bytes < comp_layout(n_faces, cb, workspace, &w)) return GOSLAM_EWORKSPACE;
  size_t tb = w.cub_bytes;
  GS_CUDA(cub::DeviceSegmentedReduce::Sum(w.cub_tmp, tb, w.area[1], w.comp_area, (int)n_components, w.seg_begin,
                                          w.seg_begin + 1, st));
  decide_kernel<<<1, kDecideThreads, 0, st>>>(w.comp_area, n_components, threshold, largest, w.comp_keep);
  GS_CHECK_LAUNCH();
  face_keep_kernel<<<blocks_for(n_faces, 256), 256, 0, st>>>(w.labels[0], w.seg_of_label, w.comp_keep, n_faces, face_keep);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
