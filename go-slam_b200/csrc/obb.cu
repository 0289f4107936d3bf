// obb.cu — the oriented bounding box of Mesher.update_param_from_mapping (src/mesher.py:242-281,
// src/oriented_bounding_box.py), i.e. Open3D 0.13's OrientedBoundingBox::CreateFromPoints and
// GetPointIndicesWithinBoundingBox, on the device.
//
// Convex-hull vertices of points [n,3] f64, as the exact extreme-point set (a point on a hull face or edge is not a
// vertex; among equal points only the lowest index can be one), with no host synchronisation:
//   extremes_kernel  one pass over the cloud: per-axis fp64 min / max, a non-finite count, and for each of kDirs fixed
//                    directions the point of largest projection (64-bit order-preserving keys, lowest index on ties).
//   winners_kernel   the distinct winners, sorted.
//   hull_kernel      (one block) the exact hull of the winners: the inner polytope.
//   cull_kernel      one bandwidth-bound pass: a point is dropped when every inner facet certifies it strictly inside,
//                    by an fp64 plane test with a proven error bound, so no extreme point is ever dropped.
//   (CUB select)     survivors in index order.
//   hull_kernel      (one block) quickhull of the survivors with a device-side loop: farthest point, visible facets,
//                    horizon, new facets, reassignment of the affected outside sets; then the extreme-point test of
//                    every hull vertex (its incident facets span at least three planes).
//   (CUB select)     the sorted vertex ids.
// Orientation tests are Shewchuk's orient3d filter with an exact expansion fallback, so the vertex set does not
// depend on rounding.  Every choice is a deterministic function of the input (ties go to the lowest index), so two
// runs are bit-identical.
//
// box_kernel restates CreateFromPoints on the hull vertices (fp64 cumulant covariance, one-thread Jacobi eigenvectors,
// descending order, sign convention, axis-aligned box in that frame); in_box_kernel is GetPointIndicesWithinBoundingBox
// (six determinant tests against the GetBoxPoints corners) reading the box from device memory.
#include <cub/cub.cuh>

#include <cfloat>
#include <cmath>

#include "common.cuh"
#include "mesh_geom.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kHullThreads = 256;          // the one-block hull kernel
constexpr int kDirs = 96;                  // directions of the extremes pass (3 per lane of a warp)
constexpr int kWinCap = 4 * kDirs + 16;    // facet slots of the winners' hull
constexpr long long kMaxPoints = 1ll << 28;
constexpr int kMaxFacets = 1 << 24;        // facet slots of the survivors' hull

enum { kHullOk = 0, kHullDegenerate = 1, kHullCapacity = 2, kHullNonFinite = 3, kHullInconsistent = 4 };

// ---- predicates ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void two_sum(double a, double b, double& x, double& y) {
  x = __dadd_rn(a, b);
  const double bv = __dsub_rn(x, a), av = __dsub_rn(x, bv);
  y = __dadd_rn(__dsub_rn(a, av), __dsub_rn(b, bv));
}

__device__ __forceinline__ void two_prod(double a, double b, double& x, double& y) {
  x = __dmul_rn(a, b);
  y = fma(a, b, -x);
}

// e (len components, nonoverlapping, increasing magnitude) += b, zero components eliminated (Shewchuk's Grow-Expansion)
__device__ __forceinline__ int grow(double* e, int len, double b) {
  double q = b;
  int k = 0;
  for (int i = 0; i < len; ++i) {
    double x, y;
    two_sum(q, e[i], x, y);
    if (y != 0.0) e[k++] = y;
    q = x;
  }
  if (q != 0.0) e[k++] = q;
  return k;
}

// exact sign of det[[a 1],[b 1],[c 1],[d 1]] = det[a - d; b - d; c - d]: 24 products of three coordinates, each an
// exact sum of four doubles, accumulated into one expansion whose largest component carries the sign
__device__ __forceinline__ int orient3d_exact(const double* a, const double* b, const double* c, const double* d) {
  const double* P[4] = {a, b, c, d};
  const int rows[4][3] = {{1, 2, 3}, {0, 2, 3}, {0, 1, 3}, {0, 1, 2}};
  const int perm[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
  const double msign[4] = {-1.0, 1.0, -1.0, 1.0};
  const double psign[6] = {1.0, -1.0, -1.0, 1.0, 1.0, -1.0};
  double e[100];
  int len = 0;
  for (int m = 0; m < 4; ++m)
    for (int t = 0; t < 6; ++t) {
      const double p = P[rows[m][0]][perm[t][0]], q = P[rows[m][1]][perm[t][1]];
      const double r = msign[m] * psign[t] * P[rows[m][2]][perm[t][2]];
      double x, y, p1, e1, p2, e2;
      two_prod(p, q, x, y);
      two_prod(x, r, p1, e1);
      two_prod(y, r, p2, e2);
      len = grow(e, len, e2);
      len = grow(e, len, e1);
      len = grow(e, len, p2);
      len = grow(e, len, p1);
    }
  return len == 0 ? 0 : (e[len - 1] > 0.0 ? 1 : -1);
}

// exact sign of the 2-d orientation of a, b, c projected on axes (i, j)
__device__ __forceinline__ int orient2d_exact(const double* a, const double* b, const double* c, int i, int j) {
  const double t[6][3] = {{a[i], b[j], 1.0}, {a[i], c[j], -1.0}, {a[j], b[i], -1.0},
                          {a[j], c[i], 1.0}, {b[i], c[j], 1.0}, {b[j], c[i], -1.0}};
  double e[16];
  int len = 0;
  for (int k = 0; k < 6; ++k) {
    double x, y;
    two_prod(t[k][0], t[k][2] * t[k][1], x, y);
    len = grow(e, len, y);
    len = grow(e, len, x);
  }
  return len == 0 ? 0 : (e[len - 1] > 0.0 ? 1 : -1);
}

__device__ __forceinline__ bool collinear_exact(const double* a, const double* b, const double* c) {
  return orient2d_exact(a, b, c, 0, 1) == 0 && orient2d_exact(a, b, c, 1, 2) == 0 && orient2d_exact(a, b, c, 2, 0) == 0;
}

// Shewchuk's orient3d: > 0 when d lies below the plane of a, b, c (a, b, c counter-clockwise seen from above).  The
// fp64 value with its static error bound (7 + 56 eps) eps * permanent; the exact expansion only when that is
// inconclusive.  det receives the fp64 value (for distances).
__device__ __forceinline__ int orient3d(const double* a, const double* b, const double* c, const double* d, double& det) {
  const double adx = __dsub_rn(a[0], d[0]), bdx = __dsub_rn(b[0], d[0]), cdx = __dsub_rn(c[0], d[0]);
  const double ady = __dsub_rn(a[1], d[1]), bdy = __dsub_rn(b[1], d[1]), cdy = __dsub_rn(c[1], d[1]);
  const double adz = __dsub_rn(a[2], d[2]), bdz = __dsub_rn(b[2], d[2]), cdz = __dsub_rn(c[2], d[2]);
  const double bdxcdy = __dmul_rn(bdx, cdy), cdxbdy = __dmul_rn(cdx, bdy);
  const double cdxady = __dmul_rn(cdx, ady), adxcdy = __dmul_rn(adx, cdy);
  const double adxbdy = __dmul_rn(adx, bdy), bdxady = __dmul_rn(bdx, ady);
  det = __dadd_rn(__dadd_rn(__dmul_rn(adz, __dsub_rn(bdxcdy, cdxbdy)), __dmul_rn(bdz, __dsub_rn(cdxady, adxcdy))),
                  __dmul_rn(cdz, __dsub_rn(adxbdy, bdxady)));
  const double perm = __dadd_rn(__dadd_rn(__dmul_rn(__dadd_rn(fabs(bdxcdy), fabs(cdxbdy)), fabs(adz)),
                                          __dmul_rn(__dadd_rn(fabs(cdxady), fabs(adxcdy)), fabs(bdz))),
                                __dmul_rn(__dadd_rn(fabs(adxbdy), fabs(bdxady)), fabs(cdz)));
  const double bound = 7.771561172376103e-16 * perm;     // (7 + 56 * 2^-53) * 2^-53
  if (det > bound) return 1;
  if (-det > bound) return -1;
  return orient3d_exact(a, b, c, d);
}

// ---- order-preserving integer keys ---------------------------------------------------------------------------------
__device__ __forceinline__ unsigned ord32(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ unsigned long long ord64(double f) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(f);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double unord64(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// ---- state and workspace -------------------------------------------------------------------------------------------
struct HullState {
  int status, bump, nfree, nact, nvis, nnew, stamp, p;
  long long n_vertices;
};

// one hull: facet slots (vertex ids, neighbour across edge (v[e], v[e+1]), visit stamp, 1 / |normal|, alive), the free
// stack, the visible / new-facet scratch of a round and the outside sets as an active list (point, facet, distance)
struct HullMem {
  int *fv, *fn, *fstamp, *freestk, *visl, *newl, *nstart, *nend;
  double* finv;
  unsigned char* falive;
  int *apt, *aown;
  float* adist;
  int cap;
  HullState* st;
};

struct ObbState {
  unsigned long long dir_key[kDirs];
  unsigned long long hi[3], lo_inv[3];      // ord64 of the per-axis max, ~ord64 of the per-axis min
  unsigned long long nonfinite;
  long long n_win, n_surv, n_vert;
  int win[kDirs];
  HullState wh, mh;
};

struct Dirs {
  float d[kDirs][3];
};

int facet_cap(long long n) { return (int)std::min<long long>(4 * n + 64, kMaxFacets); }

// what hull_mem carves: per facet slot 1 / |normal|, 12 ints (fv, fn, fstamp, freestk, visl, newl, nstart, nend)
// and the alive byte; then 256 bytes of alignment slack
size_t hull_bytes(int cap) { return gs_align((size_t)cap * (sizeof(double) + 12 * sizeof(int) + 1) + 256); }

struct ObbWork {
  ObbState* state;
  char *win, *main;                 // hull_mem's regions: the winners' hull with its active list, the survivors' hull
  unsigned char *keep, *vflag;      // [n]
  int *surv, *apt, *aown, *out;     // [n]; apt, aown, adist: the survivors' hull's active list; out: its vertices
  float* adist;                     // [n]
  char* tmp;                        // CUB's select storage
  size_t tmp_bytes;
};

size_t obb_layout(long long n, const void* base, ObbWork* w) {
  GsArena ar(base);
  w->state = ar.take<ObbState>(1);
  w->win = ar.take<char>(hull_bytes(kWinCap) + (size_t)kDirs * (2 * sizeof(int) + sizeof(float)));
  w->main = ar.take<char>(hull_bytes(facet_cap(n)));
  w->keep = ar.take<unsigned char>(n);
  w->vflag = ar.take<unsigned char>(n);
  w->surv = ar.take<int>(n);
  w->apt = ar.take<int>(n);
  w->aown = ar.take<int>(n);
  w->adist = ar.take<float>(n);
  w->out = ar.take<int>(n);
  size_t t1 = 0;   // a failed size query is reported by the select calls themselves (GS_CUDA)
  cub::DeviceSelect::Flagged(nullptr, t1, cub::CountingInputIterator<int>(0), (const unsigned char*)nullptr,
                             (int*)nullptr, (long long*)nullptr, (int)std::max<long long>(n, 1));
  w->tmp_bytes = std::max<size_t>(t1, 1);
  w->tmp = ar.take<char>(w->tmp_bytes);
  return ar.off;
}

HullMem hull_mem(char* base, int cap, int act_cap, HullState* st, int* apt, int* aown, float* adist) {
  HullMem h;
  size_t o = 0;
  auto take = [&](size_t b) { char* r = base + o; o += b; return r; };
  h.finv = (double*)take((size_t)cap * sizeof(double));
  h.fv = (int*)take((size_t)cap * 3 * sizeof(int));
  h.fn = (int*)take((size_t)cap * 3 * sizeof(int));
  h.fstamp = (int*)take((size_t)cap * sizeof(int));
  h.freestk = (int*)take((size_t)cap * sizeof(int));
  h.visl = (int*)take((size_t)cap * sizeof(int));
  h.newl = (int*)take((size_t)cap * sizeof(int));
  h.nstart = (int*)take((size_t)cap * sizeof(int));
  h.nend = (int*)take((size_t)cap * sizeof(int));
  h.falive = (unsigned char*)take((size_t)cap);
  if (apt == nullptr) {          // the winners' hull keeps its small active list behind its facets
    o = gs_align(o);
    apt = (int*)take((size_t)act_cap * sizeof(int));
    aown = (int*)take((size_t)act_cap * sizeof(int));
    adist = (float*)take((size_t)act_cap * sizeof(float));
  }
  h.apt = apt;
  h.aown = aown;
  h.adist = adist;
  h.cap = cap;
  h.st = st;
  return h;
}

// ---- extremes pass -------------------------------------------------------------------------------------------------
constexpr int kExWarps = kThreads / 32;

__global__ void __launch_bounds__(kThreads) extremes_kernel(const double* __restrict__ P, long long n, Dirs dirs,
                                                            ObbState* __restrict__ gs) {
  __shared__ float stage[kExWarps][32][3];
  __shared__ unsigned long long best[kDirs];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = threadIdx.x; t < kDirs; t += kThreads) best[t] = 0ull;
  float dx[3], dy[3], dz[3];
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    dx[t] = dirs.d[lane + 32 * t][0];
    dy[t] = dirs.d[lane + 32 * t][1];
    dz[t] = dirs.d[lane + 32 * t][2];
  }
  unsigned long long key[3] = {0ull, 0ull, 0ull};
  unsigned long long hi[3] = {0ull, 0ull, 0ull}, lo_inv[3] = {0ull, 0ull, 0ull};
  unsigned nonfinite = 0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long base = ((long long)blockIdx.x * kExWarps + warp) * 32; base < n; base += stride) {
    const long long j = base + lane;
    if (j < n) {
      const double x = P[3 * j], y = P[3 * j + 1], z = P[3 * j + 2];
      if (!isfinite(x) || !isfinite(y) || !isfinite(z)) ++nonfinite;
      const double c[3] = {x, y, z};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const unsigned long long o = ord64(c[a]);
        hi[a] = max(hi[a], o);
        lo_inv[a] = max(lo_inv[a], ~o);
      }
      stage[warp][lane][0] = (float)x;
      stage[warp][lane][1] = (float)y;
      stage[warp][lane][2] = (float)z;
    }
    __syncwarp();
    const int m = (int)min(32ll, n - base);
    for (int q = 0; q < m; ++q) {
      const float x = stage[warp][q][0], y = stage[warp][q][1], z = stage[warp][q][2];
      const unsigned long long low = 0xffffffffull - (unsigned long long)(base + q);
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const float pr = fmaf(dz[t], z, fmaf(dy[t], y, dx[t] * x));
        key[t] = max(key[t], ((unsigned long long)ord32(pr) << 32) | low);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int t = 0; t < 3; ++t) atomicMax(&best[lane + 32 * t], key[t]);
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      hi[a] = max(hi[a], __shfl_down_sync(0xffffffffu, hi[a], off));
      lo_inv[a] = max(lo_inv[a], __shfl_down_sync(0xffffffffu, lo_inv[a], off));
    }
  nonfinite = __reduce_add_sync(0xffffffffu, nonfinite);
  if (lane == 0) {
    for (int a = 0; a < 3; ++a) {
      if (hi[a]) atomicMax(&gs->hi[a], hi[a]);
      if (lo_inv[a]) atomicMax(&gs->lo_inv[a], lo_inv[a]);
    }
    if (nonfinite) atomicAdd(&gs->nonfinite, (unsigned long long)nonfinite);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kDirs; t += kThreads)
    if (best[t]) atomicMax(&gs->dir_key[t], best[t]);
}

__global__ void winners_kernel(ObbState* gs) {
  if (threadIdx.x != 0) return;
  int w[kDirs], m = 0;
  for (int t = 0; t < kDirs; ++t)
    if (gs->dir_key[t]) w[m++] = (int)(0xffffffffull - (gs->dir_key[t] & 0xffffffffull));
  for (int a = 1; a < m; ++a)        // insertion sort, then drop repeats
    for (int b = a; b > 0 && w[b - 1] > w[b]; --b) { const int t = w[b]; w[b] = w[b - 1]; w[b - 1] = t; }
  int k = 0;
  for (int a = 0; a < m; ++a)
    if (k == 0 || w[a] != gs->win[k - 1]) gs->win[k++] = w[a];
  gs->n_win = k;
}

// ---- the one-block hull --------------------------------------------------------------------------------------------
__device__ __forceinline__ const double* pt(const double* P, int i) { return P + 3 * (size_t)i; }

// > 0 when point i is strictly above (outside) facet f; dist gets the fp64 distance estimate
__device__ __forceinline__ bool above(const double* P, const HullMem& h, int f, int i, float& dist) {
  double det;
  const int s = orient3d(pt(P, h.fv[3 * f]), pt(P, h.fv[3 * f + 1]), pt(P, h.fv[3 * f + 2]), pt(P, i), det);
  dist = (float)fmax(-det * h.finv[f], 0.0);
  return s < 0;
}

__device__ void set_finv(const double* P, HullMem& h, int f) {
  const double* a = pt(P, h.fv[3 * f]);
  const double* b = pt(P, h.fv[3 * f + 1]);
  const double* c = pt(P, h.fv[3 * f + 2]);
  const double u[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, v[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
  const double nx = u[1] * v[2] - u[2] * v[1], ny = u[2] * v[0] - u[0] * v[2], nz = u[0] * v[1] - u[1] * v[0];
  const double len = sqrt(nx * nx + ny * ny + nz * nz);
  h.finv[f] = len > 0.0 ? 1.0 / len : 0.0;
}

__device__ __forceinline__ bool lex_less(const double* P, int i, int j) {
  const double* a = pt(P, i);
  const double* b = pt(P, j);
  if (a[0] != b[0]) return a[0] < b[0];
  if (a[1] != b[1]) return a[1] < b[1];
  if (a[2] != b[2]) return a[2] < b[2];
  return i < j;
}

// block-wide best candidate (-1 = none) under better(i, j); every thread gets the result
template <class Better>
__device__ int block_best(int cand, Better better, int* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off; off >>= 1) {
    const int o = __shfl_down_sync(0xffffffffu, cand, off);
    if (o >= 0 && (cand < 0 || better(o, cand))) cand = o;
  }
  if (lane == 0) sh[warp] = cand;
  __syncthreads();
  if (threadIdx.x == 0) {
    int b = sh[0];
    for (int w = 1; w < kHullThreads / 32; ++w)
      if (sh[w] >= 0 && (b < 0 || better(sh[w], b))) b = sh[w];
    sh[32] = b;
  }
  __syncthreads();
  const int r = sh[32];
  __syncthreads();
  return r;
}

// exclusive position of this thread's flag among the block's and the block total
__device__ __forceinline__ int block_scan(int flag, int& total) {
  using Scan = cub::BlockScan<int, kHullThreads>;
  __shared__ typename Scan::TempStorage tmp;
  int pos;
  Scan(tmp).ExclusiveSum(flag, pos, total);
  __syncthreads();
  return pos;
}

// ids == nullptr: points 0 .. n-1, else ids[0 .. n-1] (ascending).  vflag != nullptr: after the hull, mark its extreme
// vertices (vflag[id] = 1); vf is scratch indexed by point id.
__global__ void __launch_bounds__(kHullThreads, 1)
hull_kernel(const double* __restrict__ P, const int* __restrict__ ids, const long long* n_ids, HullMem h,
            const unsigned long long* nonfinite, int* __restrict__ vf, unsigned char* __restrict__ vflag) {
  __shared__ int sh[33];
  __shared__ int s_simplex[4];
  HullState* st = h.st;
  const int tid = threadIdx.x;
  const int n = (int)*n_ids;
  if (*nonfinite) {
    if (tid == 0) st->status = kHullNonFinite;
    return;
  }
  if (n < 4) {
    if (tid == 0) st->status = kHullDegenerate;
    return;
  }
  auto id = [&](int j) { return ids ? ids[j] : j; };

  // ---- initial simplex: lexicographic minimum a, farthest b, then the points farthest from line ab and plane abc,
  // each checked exactly (a linear search for any qualifying point when the fp64 choice is degenerate)
  int cand = -1;
  for (int j = tid; j < n; j += kHullThreads) {
    const int i = id(j);
    if (cand < 0 || lex_less(P, i, cand)) cand = i;
  }
  const int a = block_best(cand, [&](int i, int k) { return lex_less(P, i, k); }, sh);
  const double* A = pt(P, a);
  auto d2a = [&](int i) {
    const double* p = pt(P, i);
    const double x = p[0] - A[0], y = p[1] - A[1], z = p[2] - A[2];
    return x * x + y * y + z * z;
  };
  auto far_a = [&](int i, int k) { const double u = d2a(i), v = d2a(k); return u > v || (u == v && i < k); };
  cand = -1;
  for (int j = tid; j < n; j += kHullThreads) {
    const int i = id(j);
    if (cand < 0 || far_a(i, cand)) cand = i;
  }
  const int b = block_best(cand, far_a, sh);
  const double* B = pt(P, b);
  if (B[0] == A[0] && B[1] == A[1] && B[2] == A[2]) {
    if (tid == 0) st->status = kHullDegenerate;
    return;
  }
  auto cr2 = [&](int i) {
    const double* p = pt(P, i);
    const double u[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]}, v[3] = {p[0] - A[0], p[1] - A[1], p[2] - A[2]};
    const double x = u[1] * v[2] - u[2] * v[1], y = u[2] * v[0] - u[0] * v[2], z = u[0] * v[1] - u[1] * v[0];
    return x * x + y * y + z * z;
  };
  auto far_l = [&](int i, int k) { const double u = cr2(i), v = cr2(k); return u > v || (u == v && i < k); };
  cand = -1;
  for (int j = tid; j < n; j += kHullThreads) {
    const int i = id(j);
    if (cand < 0 || far_l(i, cand)) cand = i;
  }
  int c = block_best(cand, far_l, sh);
  if (collinear_exact(A, B, pt(P, c))) {
    cand = -1;
    for (int j = tid; j < n && cand < 0; j += kHullThreads)
      if (!collinear_exact(A, B, pt(P, id(j)))) cand = id(j);
    c = block_best(cand, [](int i, int k) { return i < k; }, sh);
    if (c < 0) {
      if (tid == 0) st->status = kHullDegenerate;
      return;
    }
  }
  const double* C = pt(P, c);
  auto vol = [&](int i) {
    double det;
    orient3d(A, B, C, pt(P, i), det);
    return fabs(det);
  };
  auto far_p = [&](int i, int k) { const double u = vol(i), v = vol(k); return u > v || (u == v && i < k); };
  cand = -1;
  for (int j = tid; j < n; j += kHullThreads) {
    const int i = id(j);
    if (cand < 0 || far_p(i, cand)) cand = i;
  }
  int d = block_best(cand, far_p, sh);
  if (orient3d_exact(A, B, C, pt(P, d)) == 0) {
    cand = -1;
    for (int j = tid; j < n && cand < 0; j += kHullThreads)
      if (orient3d_exact(A, B, C, pt(P, id(j))) != 0) cand = id(j);
    d = block_best(cand, [](int i, int k) { return i < k; }, sh);
    if (d < 0) {
      if (tid == 0) st->status = kHullDegenerate;
      return;
    }
  }

  // ---- the tetrahedron: facet k omits vertex k and is oriented so that vertex k lies below it
  if (tid == 0) {
    s_simplex[0] = a; s_simplex[1] = b; s_simplex[2] = c; s_simplex[3] = d;
    for (int k = 0; k < 4; ++k) {
      int t[3], m = 0;
      for (int q = 0; q < 4; ++q)
        if (q != k) t[m++] = s_simplex[q];
      double det;
      if (orient3d(pt(P, t[0]), pt(P, t[1]), pt(P, t[2]), pt(P, s_simplex[k]), det) < 0) {
        const int x = t[1]; t[1] = t[2]; t[2] = x;
      }
      for (int q = 0; q < 3; ++q) h.fv[3 * k + q] = t[q];
      h.fstamp[k] = 0;
      h.falive[k] = 1;
    }
    for (int f = 0; f < 4; ++f)
      for (int e = 0; e < 3; ++e) {
        const int x = h.fv[3 * f + e], y = h.fv[3 * f + (e + 1) % 3];
        for (int g = 0; g < 4; ++g)
          for (int q = 0; q < 3; ++q)
            if (g != f && h.fv[3 * g + q] == y && h.fv[3 * g + (q + 1) % 3] == x) h.fn[3 * f + e] = g;
      }
    for (int f = 0; f < 4; ++f) set_finv(P, h, f);
    st->status = kHullOk;
    st->bump = 4;
    st->nfree = 0;
    st->stamp = 0;
    st->n_vertices = 0;
  }
  __syncthreads();

  // ---- outside sets of the tetrahedron (the first facet a point is strictly above), in input order
  int nact = 0;
  for (int base = 0; base < n; base += kHullThreads) {
    const int j = base + tid;
    int keep = 0, i = -1, own = -1;
    float dist = 0.f;
    if (j < n) {
      i = id(j);
      for (int f = 0; f < 4; ++f)
        if (above(P, h, f, i, dist)) { own = f; keep = 1; break; }
    }
    int total;
    const int pos = block_scan(keep, total);
    if (keep) {
      h.apt[nact + pos] = i;
      h.aown[nact + pos] = own;
      h.adist[nact + pos] = dist;
    }
    nact += total;
  }
  __syncthreads();

  // ---- quickhull rounds
  __shared__ int s_p, s_fail;
  while (nact > 0) {
    // farthest outside point (largest distance, lowest index on ties)
    float bd = -1.f;
    int bp = -1, bf = -1;
    for (int j = tid; j < nact; j += kHullThreads) {
      const float dd = h.adist[j];
      const int pp = h.apt[j];
      if (dd > bd || (dd == bd && pp < bp)) { bd = dd; bp = pp; bf = h.aown[j]; }
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      const float od = __shfl_down_sync(0xffffffffu, bd, off);
      const int op = __shfl_down_sync(0xffffffffu, bp, off);
      const int of = __shfl_down_sync(0xffffffffu, bf, off);
      if (op >= 0 && (bp < 0 || od > bd || (od == bd && op < bp))) { bd = od; bp = op; bf = of; }
    }
    __shared__ float rd[kHullThreads / 32];
    __shared__ int rp[kHullThreads / 32], rf[kHullThreads / 32];
    if ((tid & 31) == 0) { rd[tid >> 5] = bd; rp[tid >> 5] = bp; rf[tid >> 5] = bf; }
    __syncthreads();
    if (tid == 0) {
      float xd = rd[0];
      int xp = rp[0], xf = rf[0];
      for (int w = 1; w < kHullThreads / 32; ++w)
        if (rp[w] >= 0 && (xp < 0 || rd[w] > xd || (rd[w] == xd && rp[w] < xp))) { xd = rd[w]; xp = rp[w]; xf = rf[w]; }
      s_p = xp;
      s_fail = 0;
      // visible facets (breadth first from the owner), horizon, new facets
      const int p = xp;
      const int stamp = ++st->stamp;
      int nvis = 0, nnew = 0;
      h.visl[nvis++] = xf;
      h.fstamp[xf] = stamp;
      for (int q = 0; q < nvis; ++q) {
        const int f = h.visl[q];
        for (int e = 0; e < 3; ++e) {
          const int g = h.fn[3 * f + e];
          if (h.fstamp[g] == stamp || h.fstamp[g] == -stamp) continue;
          float dd;
          if (above(P, h, g, p, dd)) {
            h.fstamp[g] = stamp;
            h.visl[nvis++] = g;
          } else {
            h.fstamp[g] = -stamp;
          }
        }
      }
      for (int q = 0; q < nvis && !s_fail; ++q) {
        const int f = h.visl[q];
        for (int e = 0; e < 3; ++e) {
          const int g = h.fn[3 * f + e];
          if (h.fstamp[g] == stamp) continue;
          int nf;
          if (st->nfree > 0) nf = h.freestk[--st->nfree];
          else if (st->bump < h.cap) nf = st->bump++;
          else { s_fail = 1; st->status = kHullCapacity; break; }
          const int u = h.fv[3 * f + e], v = h.fv[3 * f + (e + 1) % 3];
          h.fv[3 * nf] = u; h.fv[3 * nf + 1] = v; h.fv[3 * nf + 2] = p;
          h.fn[3 * nf] = g; h.fn[3 * nf + 1] = -1; h.fn[3 * nf + 2] = -1;
          for (int s = 0; s < 3; ++s)
            if (h.fv[3 * g + s] == v && h.fv[3 * g + (s + 1) % 3] == u) h.fn[3 * g + s] = nf;
          h.fstamp[nf] = 0;
          h.falive[nf] = 1;
          set_finv(P, h, nf);
          h.newl[nnew] = nf; h.nstart[nnew] = u; h.nend[nnew] = v;
          ++nnew;
        }
      }
      st->nvis = nvis;
      st->nnew = nnew;
    }
    __syncthreads();
    if (s_fail) return;
    const int p = s_p, nnew = st->nnew;
    const int stamp = st->stamp;
    // the new facets around p: facet k's edge (end_k, p) meets the facet whose horizon edge starts at end_k
    for (int k = tid; k < nnew; k += kHullThreads) {
      const int e = h.nend[k];
      int j = 0;
      while (j < nnew && h.nstart[j] != e) ++j;
      if (j == nnew) {           // the horizon is not a cycle: cannot happen with exact predicates
        s_fail = 1;
        st->status = kHullInconsistent;
        continue;
      }
      h.fn[3 * h.newl[k] + 1] = h.newl[j];
      h.fn[3 * h.newl[j] + 2] = h.newl[k];
    }
    __syncthreads();
    if (s_fail) return;
    // outside sets of the visible facets move to the first new facet they are strictly above, or leave
    int kept = 0;
    for (int base = 0; base < nact; base += kHullThreads) {
      const int j = base + tid;
      int keep = 0, i = -1, own = -1;
      float dist = 0.f;
      if (j < nact) {
        i = h.apt[j];
        own = h.aown[j];
        dist = h.adist[j];
        if (h.fstamp[own] != stamp) {
          keep = 1;
        } else if (i != p) {
          for (int k = 0; k < nnew; ++k)
            if (above(P, h, h.newl[k], i, dist)) { own = h.newl[k]; keep = 1; break; }
        }
      }
      int total;
      const int pos = block_scan(keep, total);
      if (keep) {
        h.apt[kept + pos] = i;
        h.aown[kept + pos] = own;
        h.adist[kept + pos] = dist;
      }
      kept += total;
    }
    nact = kept;
    if (tid == 0) {
      for (int q = 0; q < st->nvis; ++q) {
        const int f = h.visl[q];
        h.falive[f] = 0;
        h.freestk[st->nfree++] = f;
      }
    }
    __syncthreads();
  }
  if (vflag == nullptr) return;

  // ---- extreme-point test: a hull vertex is a vertex of the polytope iff its incident facets span >= 3 planes
  const int bump = st->bump;
  for (int f = tid; f < bump; f += kHullThreads)
    if (h.falive[f])
      for (int e = 0; e < 3; ++e) vf[h.fv[3 * f + e]] = f;
  __syncthreads();
  auto coplanar = [&](int f, int g) {
    for (int e = 0; e < 3; ++e) {
      double det;
      if (orient3d(pt(P, h.fv[3 * f]), pt(P, h.fv[3 * f + 1]), pt(P, h.fv[3 * f + 2]), pt(P, h.fv[3 * g + e]), det))
        return false;
    }
    return true;
  };
  unsigned long long found = 0;
  for (int f = tid; f < bump; f += kHullThreads) {
    if (!h.falive[f]) continue;
    for (int e = 0; e < 3; ++e) {
      const int v = h.fv[3 * f + e];
      if (vf[v] != f) continue;
      int p2 = -1, cur = f;
      bool extreme = false;
      for (int guard = 0; guard < bump && !extreme; ++guard) {
        int s = 0;
        while (s < 3 && h.fv[3 * cur + s] != v) ++s;
        if (s == 3) break;       // not a closed fan: cannot happen on a consistent hull
        if (cur != f && !coplanar(f, cur)) {
          if (p2 < 0) p2 = cur;
          else if (!coplanar(p2, cur)) extreme = true;
        }
        cur = h.fn[3 * cur + s];
        if (cur == f) break;
      }
      if (extreme) {
        vflag[v] = 1;
        ++found;
      }
    }
  }
  found = __reduce_add_sync(0xffffffffu, (unsigned)found);
  if ((tid & 31) == 0 && found) atomicAdd((unsigned long long*)&st->n_vertices, found);
}

// ---- the cull pass -------------------------------------------------------------------------------------------------
// For the winners' facet (a, b, c), interior points p have N.(p - a) < 0 with N = (b - a) x (c - a).  With u, v, w the
// rounded b - a, c - a, p - a, n = fl(u x v) and s = fl(n.w):  |s - N.(p - a)| <= 4.1 eps sum_i (|n_i| + m_i) |w_i|,
// m_i = |u_j v_k| + |u_k v_j|, and |w_i| <= the largest axis span W of the cloud.  margin = 16 eps sum_i (|n_i| + m_i) W
// (twice the bound, rounding of the bound itself included), so s < -margin proves p strictly inside that facet.
__global__ void __launch_bounds__(kThreads) cull_kernel(const double* __restrict__ P, long long n, HullMem h,
                                                        const ObbState* __restrict__ gs,
                                                        unsigned char* __restrict__ keep) {
  __shared__ double pl[kWinCap][7];
  __shared__ int nf;
  const bool all = h.st->status != kHullOk;
  if (threadIdx.x == 0) nf = 0;
  __syncthreads();
  if (!all) {
    double W = 0.0;
    for (int a = 0; a < 3; ++a) W = fmax(W, unord64(gs->hi[a]) - unord64(~gs->lo_inv[a]));
    W *= 1.0 + 0x1p-50;
    for (int f = threadIdx.x; f < h.st->bump; f += kThreads) {
      if (!h.falive[f]) continue;
      const double* A = pt(P, h.fv[3 * f]);
      const double* B = pt(P, h.fv[3 * f + 1]);
      const double* C = pt(P, h.fv[3 * f + 2]);
      double u[3], v[3], nn[3], m[3];
      for (int i = 0; i < 3; ++i) { u[i] = __dsub_rn(B[i], A[i]); v[i] = __dsub_rn(C[i], A[i]); }
      for (int i = 0; i < 3; ++i) {
        const int j = (i + 1) % 3, k = (i + 2) % 3;
        const double x = __dmul_rn(u[j], v[k]), y = __dmul_rn(u[k], v[j]);
        nn[i] = __dsub_rn(x, y);
        m[i] = fabs(x) + fabs(y);
      }
      const double M = fabs(nn[0]) + fabs(nn[1]) + fabs(nn[2]) + m[0] + m[1] + m[2];
      const int k = atomicAdd(&nf, 1);
      pl[k][0] = nn[0]; pl[k][1] = nn[1]; pl[k][2] = nn[2];
      pl[k][3] = A[0]; pl[k][4] = A[1]; pl[k][5] = A[2];
      pl[k][6] = 0x1p-49 * M * W;
    }
  }
  __syncthreads();
  const int nfac = nf;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
    bool k = all;
    if (!k) {
      const double x = P[3 * i], y = P[3 * i + 1], z = P[3 * i + 2];
      for (int f = 0; f < nfac; ++f) {
        const double s = pl[f][0] * (x - pl[f][3]) + pl[f][1] * (y - pl[f][4]) + pl[f][2] * (z - pl[f][5]);
        if (!(s < -pl[f][6])) { k = true; break; }
      }
    }
    keep[i] = k;
  }
}

__global__ void info_kernel(const ObbState* gs, int64_t* info) {
  info[0] = gs->mh.status;
  info[1] = gs->mh.status == kHullOk ? gs->n_vert : 0;
  info[2] = gs->n_surv;
  info[3] = gs->n_win;
}

// ---- the box -------------------------------------------------------------------------------------------------------
// Open3D 0.13 OrientedBoundingBox::CreateFromPoints on the hull vertices: mean and covariance from fp64 cumulants / h
// (PointCloud::ComputeMeanAndCovariance), eigenvectors by descending eigenvalue, then the axis-aligned box of
// R^T (v - mean): center = R c' + mean, extent = max - min (+ extend).  Sign convention: each of columns 0 and 1 has its
// largest-magnitude component positive, column 2 = column 0 x column 1.
__global__ void __launch_bounds__(kThreads) box_kernel(const double* __restrict__ P, const int* __restrict__ vid,
                                                       const ObbState* __restrict__ gs, double extend,
                                                       double* __restrict__ box) {
  __shared__ double red[kThreads / 32][9];
  __shared__ double sR[9], smean[3];
  if (gs->mh.status != kHullOk) return;
  const int h = (int)gs->n_vert;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int k = threadIdx.x; k < h; k += kThreads) {
    const double* p = pt(P, vid[k]);
    s[0] = __dadd_rn(s[0], p[0]);
    s[1] = __dadd_rn(s[1], p[1]);
    s[2] = __dadd_rn(s[2], p[2]);
    s[3] = __dadd_rn(s[3], __dmul_rn(p[0], p[0]));
    s[4] = __dadd_rn(s[4], __dmul_rn(p[0], p[1]));
    s[5] = __dadd_rn(s[5], __dmul_rn(p[0], p[2]));
    s[6] = __dadd_rn(s[6], __dmul_rn(p[1], p[1]));
    s[7] = __dadd_rn(s[7], __dmul_rn(p[1], p[2]));
    s[8] = __dadd_rn(s[8], __dmul_rn(p[2], p[2]));
  }
#pragma unroll
  for (int q = 0; q < 9; ++q) {
#pragma unroll
    for (int off = 16; off; off >>= 1) s[q] = __dadd_rn(s[q], __shfl_down_sync(0xffffffffu, s[q], off));
    if (lane == 0) red[warp][q] = s[q];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double c[9];
    for (int q = 0; q < 9; ++q) {
      double t = red[0][q];
      for (int w = 1; w < kThreads / 32; ++w) t = __dadd_rn(t, red[w][q]);
      c[q] = __ddiv_rn(t, (double)h);
    }
    const double cxx = c[3] - c[0] * c[0], cyy = c[6] - c[1] * c[1], czz = c[8] - c[2] * c[2];
    const double cxy = c[4] - c[0] * c[1], cxz = c[5] - c[0] * c[2], cyz = c[7] - c[1] * c[2];
    const double cov[9] = {cxx, cxy, cxz, cxy, cyy, cyz, cxz, cyz, czz};
    double B[9], V[9];
    gs_jacobi3(cov, B, V);
    double ev[3];
    int ord[3] = {0, 1, 2};
    for (int j = 0; j < 3; ++j) ev[j] = sqrt(B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j]);
    for (int x = 0; x < 3; ++x)
      for (int y = x + 1; y < 3; ++y)
        if (ev[ord[y]] > ev[ord[x]]) { const int t = ord[x]; ord[x] = ord[y]; ord[y] = t; }
    double col[3][3];
    for (int j = 0; j < 2; ++j) {
      double nrm = 0.0;
      for (int r = 0; r < 3; ++r) nrm += V[3 * r + ord[j]] * V[3 * r + ord[j]];
      nrm = sqrt(nrm);
      int big = 0;
      for (int r = 0; r < 3; ++r) {
        col[j][r] = V[3 * r + ord[j]] / nrm;
        if (fabs(col[j][r]) > fabs(col[j][big])) big = r;
      }
      if (col[j][big] < 0.0)
        for (int r = 0; r < 3; ++r) col[j][r] = -col[j][r];
    }
    col[2][0] = col[0][1] * col[1][2] - col[0][2] * col[1][1];
    col[2][1] = col[0][2] * col[1][0] - col[0][0] * col[1][2];
    col[2][2] = col[0][0] * col[1][1] - col[0][1] * col[1][0];
    for (int r = 0; r < 3; ++r)
      for (int j = 0; j < 3; ++j) sR[3 * r + j] = col[j][r];
    smean[0] = c[0]; smean[1] = c[1]; smean[2] = c[2];
  }
  __syncthreads();
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  for (int k = threadIdx.x; k < h; k += kThreads) {
    const double* p = pt(P, vid[k]);
    const double d[3] = {p[0] - smean[0], p[1] - smean[1], p[2] - smean[2]};
    for (int j = 0; j < 3; ++j) {
      const double q = sR[j] * d[0] + sR[3 + j] * d[1] + sR[6 + j] * d[2];
      lo[j] = fmin(lo[j], q);
      hi[j] = fmax(hi[j], q);
    }
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 3; ++j) {
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      lo[j] = fmin(lo[j], __shfl_down_sync(0xffffffffu, lo[j], off));
      hi[j] = fmax(hi[j], __shfl_down_sync(0xffffffffu, hi[j], off));
    }
    if (lane == 0) { red[warp][j] = lo[j]; red[warp][3 + j] = hi[j]; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double c[3], e[3];
    for (int j = 0; j < 3; ++j) {
      double l = red[0][j], u = red[0][3 + j];
      for (int w = 1; w < kThreads / 32; ++w) { l = fmin(l, red[w][j]); u = fmax(u, red[w][3 + j]); }
      c[j] = (l + u) * 0.5;
      e[j] = u - l;
    }
    for (int r = 0; r < 3; ++r)
      box[r] = sR[3 * r] * c[0] + sR[3 * r + 1] * c[1] + sR[3 * r + 2] * c[2] + smean[r];
    for (int k = 0; k < 9; ++k) box[3 + k] = sR[k];
    for (int j = 0; j < 3; ++j) box[12 + j] = e[j] + extend;
  }
}

// det[b - a, c - a, x - a] (columns) in Eigen's 3x3 cofactor order, every operation rounded
__device__ __forceinline__ double plane_test(const double* a, const double* b, const double* c, const double* x) {
  const double u[3] = {__dsub_rn(b[0], a[0]), __dsub_rn(b[1], a[1]), __dsub_rn(b[2], a[2])};
  const double v[3] = {__dsub_rn(c[0], a[0]), __dsub_rn(c[1], a[1]), __dsub_rn(c[2], a[2])};
  const double w[3] = {__dsub_rn(x[0], a[0]), __dsub_rn(x[1], a[1]), __dsub_rn(x[2], a[2])};
  const double t0 = __dmul_rn(u[0], __dsub_rn(__dmul_rn(v[1], w[2]), __dmul_rn(v[2], w[1])));
  const double t1 = __dmul_rn(v[0], __dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1])));
  const double t2 = __dmul_rn(w[0], __dsub_rn(__dmul_rn(u[1], v[2]), __dmul_rn(u[2], v[1])));
  return __dadd_rn(__dsub_rn(t0, t1), t2);
}

// OrientedBoundingBox::GetBoxPoints: center -/+ R (e0/2, 0, 0) -/+ R (0, e1/2, 0) -/+ R (0, 0, e2/2), Open3D's order
__global__ void __launch_bounds__(kThreads) in_box_kernel(const double* __restrict__ box, const double* __restrict__ P,
                                                          long long n, unsigned char* __restrict__ mask) {
  __shared__ double cp[8][3];
  if (threadIdx.x < 8) {
    const int k = threadIdx.x;
    // signs of (x, y, z) per corner
    const int sg[8][3] = {{-1, -1, -1}, {1, -1, -1}, {-1, 1, -1}, {-1, -1, 1},
                          {1, 1, 1},    {-1, 1, 1},  {1, -1, 1},  {1, 1, -1}};
    double ax[3][3];
    for (int j = 0; j < 3; ++j) {
      const double hlf = __dmul_rn(box[12 + j], 0.5);
      for (int r = 0; r < 3; ++r) ax[j][r] = __dmul_rn(box[3 + 3 * r + j], hlf);
    }
    for (int r = 0; r < 3; ++r) {
      double v = box[r];
      for (int j = 0; j < 3; ++j) v = sg[k][j] > 0 ? __dadd_rn(v, ax[j][r]) : __dsub_rn(v, ax[j][r]);
      cp[k][r] = v;
    }
  }
  __syncthreads();
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
    const double* x = P + 3 * i;
    const bool in = plane_test(cp[0], cp[1], cp[3], x) <= 0.0 && plane_test(cp[0], cp[5], cp[3], x) >= 0.0 &&
                    plane_test(cp[2], cp[5], cp[7], x) <= 0.0 && plane_test(cp[1], cp[4], cp[7], x) >= 0.0 &&
                    plane_test(cp[3], cp[4], cp[5], x) <= 0.0 && plane_test(cp[0], cp[1], cp[7], x) >= 0.0;
    mask[i] = in;
  }
}

__global__ void __launch_bounds__(kThreads) widen_kernel(const int* __restrict__ src, int64_t* __restrict__ dst,
                                                         long long n) {
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads)
    dst[i] = src[i];
}

Dirs make_dirs() {
  Dirs d;
  const double ax[6][3] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
  for (int k = 0; k < 6; ++k)
    for (int c = 0; c < 3; ++c) d.d[k][c] = (float)ax[k][c];
  const int m = kDirs - 6;                     // a Fibonacci sphere for the rest
  const double golden = M_PI * (3.0 - std::sqrt(5.0));
  for (int k = 0; k < m; ++k) {
    const double z = 1.0 - (2.0 * k + 1.0) / m, r = std::sqrt(1.0 - z * z), t = golden * k;
    d.d[6 + k][0] = (float)(r * std::cos(t));
    d.d[6 + k][1] = (float)(r * std::sin(t));
    d.d[6 + k][2] = (float)z;
  }
  return d;
}

int grid_for(long long n) {
  return (int)std::max<long long>(1, std::min<long long>((n + kThreads - 1) / kThreads, (long long)kNumSms * 16));
}

}  // namespace

extern "C" {

size_t goslam_hull_workspace_bytes(int64_t n) {
  if (n < 1 || n > kMaxPoints) return 0;
  ObbWork w;
  return obb_layout(n, nullptr, &w);
}

int goslam_hull_vertices(const double* points, int64_t n, void* workspace, size_t workspace_bytes, int64_t* info,
                         void* stream) {
  if (points == nullptr || info == nullptr || n < 1 || n > kMaxPoints) return GOSLAM_EINVAL;
  ObbWork w;
  if (!workspace || workspace_bytes < obb_layout(n, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  ObbState* gs = w.state;
  const HullMem wh = hull_mem(w.win, kWinCap, kDirs, &gs->wh, nullptr, nullptr, nullptr);
  const HullMem mh = hull_mem(w.main, facet_cap(n), 0, &gs->mh, w.apt, w.aown, w.adist);
  GS_CUDA(cudaMemsetAsync(gs, 0, sizeof(ObbState), s));
  GS_CUDA(cudaMemsetAsync(w.vflag, 0, (size_t)n, s));
  extremes_kernel<<<grid_for(n), kThreads, 0, s>>>(points, n, make_dirs(), gs);
  GS_CHECK_LAUNCH();
  winners_kernel<<<1, 32, 0, s>>>(gs);
  GS_CHECK_LAUNCH();
  hull_kernel<<<1, kHullThreads, 0, s>>>(points, gs->win, &gs->n_win, wh, &gs->nonfinite, nullptr, nullptr);
  GS_CHECK_LAUNCH();
  cull_kernel<<<grid_for(n), kThreads, 0, s>>>(points, n, wh, gs, w.keep);
  GS_CHECK_LAUNCH();
  size_t tb = w.tmp_bytes;
  GS_CUDA(cub::DeviceSelect::Flagged(w.tmp, tb, cub::CountingInputIterator<int>(0), w.keep, w.surv, &gs->n_surv, (int)n,
                                     s));
  hull_kernel<<<1, kHullThreads, 0, s>>>(points, w.surv, &gs->n_surv, mh, &gs->nonfinite, w.surv, w.vflag);
  GS_CHECK_LAUNCH();
  tb = w.tmp_bytes;
  GS_CUDA(cub::DeviceSelect::Flagged(w.tmp, tb, cub::CountingInputIterator<int>(0), w.vflag, w.out, &gs->n_vert, (int)n,
                                     s));
  info_kernel<<<1, 1, 0, s>>>(gs, info);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_hull_vertices_emit(const void* workspace, size_t workspace_bytes, int64_t n, int64_t* out, int64_t count,
                              void* stream) {
  if (n < 1 || n > kMaxPoints || count < 0 || count > n || (count > 0 && out == nullptr)) return GOSLAM_EINVAL;
  ObbWork w;
  if (!workspace || workspace_bytes < obb_layout(n, workspace, &w)) return GOSLAM_EWORKSPACE;
  if (count == 0) return GOSLAM_OK;
  widen_kernel<<<grid_for(count), kThreads, 0, (cudaStream_t)stream>>>(w.out, out, count);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_obb_from_hull(const double* points, int64_t n, const void* workspace, size_t workspace_bytes, double extend,
                         double* box, void* stream) {
  if (points == nullptr || box == nullptr || n < 1 || n > kMaxPoints) return GOSLAM_EINVAL;
  ObbWork w;
  if (!workspace || workspace_bytes < obb_layout(n, workspace, &w)) return GOSLAM_EWORKSPACE;
  box_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>(points, w.out, w.state, extend, box);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_obb_in_bound(const double* box, const double* points, int64_t n, uint8_t* mask, void* stream) {
  if (n < 0 || (n > 0 && (box == nullptr || points == nullptr || mask == nullptr))) return GOSLAM_EINVAL;
  if (n == 0) return GOSLAM_OK;
  in_box_kernel<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(box, points, n, mask);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
