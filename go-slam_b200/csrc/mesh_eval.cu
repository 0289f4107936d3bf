// mesh_eval.cu — the evaluation step of Mesher.__call__(the_end=True) (src/mesher.py:310-327) on the device: surface
// sampling (trimesh.sample.sample_surface), exact nearest-neighbour search (scipy's cKDTree, Open3D's SearchHybrid) and
// point-to-point ICP (Open3D's registration_icp with TransformationEstimationPointToPoint).
//
//  * sampling: fp64 face areas (gs_face_area, the component filter's formula), an fp64 inclusive scan (CUB), then one
//    thread per sample: face = the first f with cum[f] >= u * cum[F-1] (searchsorted side='left'), and trimesh's point
//    rule ((v1 - v0) l0 + (v2 - v0) l1) + v0 with (l0, l1) folded to |l - 1| when l0 + l1 > 1.  Operation by operation,
//    no contraction; the uniforms are the caller's.
//  * nearest-neighbour index: a uniform grid over the target points.  Origin = the points' box minimum, cell size h =
//    max(min_cell, cbrt(box volume / n)), grown by 1.25x until the grid has at most 2n + 64 cells; cell keys (x fastest),
//    a CUB radix sort of (key, point id), the points gathered in key order and cell_start[c] = first sorted position
//    with key >= c.
//  * query: one thread per query walks shells of cells (Chebyshev rings) around its cell, clamped to the grid.  After
//    shell k every unvisited point lies in the box of all points but beyond one of the six faces of the visited cube;
//    the distance from q to the nearest such region is a lower bound L_k.  The walk stops once the best squared
//    distance is below (L_k - slack)^2, slack = 1e-12 x the coordinate scale (covers the rounding of the cell
//    assignment), or when nothing is left.  With a radius r only d2 < r * r counts (nanoflann's strict rule) and the
//    walk also stops at L_k >= r.  d2 = (dx^2 + dy^2) + dz^2 rounded operation by operation, which is what cKDTree
//    computes, so distances are sqrt(d2) bit for bit; among equal d2 the smallest point id wins.
//  * ICP: every iteration is enqueued up front (cov, solve, transform, correspond, reduce); the reduce kernel sets a
//    device flag on convergence and every later kernel returns at once.  Reductions are fp64 per-block partials summed
//    in block order (deterministic); the 3x3 Umeyama solve is one thread (one-sided Jacobi SVD).
#include <cub/cub.cuh>

#include "common.cuh"
#include "mesh_geom.cuh"

namespace {

constexpr int kThreads = 256;
constexpr long long kMaxPoints = 1ll << 28;          // point ids and cell keys are u32
constexpr long long kMaxFaces = (1ll << 31) - 1;     // CUB item counts are int
constexpr int kBoxBlocks = 4 * kNumSms;

__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }

unsigned blocks_for(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// ---- surface sampling ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) area_kernel(const double* verts, long long nv, const long long* faces,
                                                        long long nf, double* area) {
  const long long f = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (f >= nf) return;
  const long long a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
  const bool ok = a >= 0 && a < nv && b >= 0 && b < nv && c >= 0 && c < nv;
  area[f] = ok ? gs_face_area(verts + 3 * a, verts + 3 * b, verts + 3 * c) : 0.0;
}

__global__ void __launch_bounds__(kThreads) sample_kernel(const double* verts, long long nv, const long long* faces,
                                                          long long nf, const double* cum, const double* uniforms,
                                                          long long count, double* samples, long long* face_index) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= count) return;
  const double target = dmul(uniforms[3 * i], cum[nf - 1]);
  long long lo = 0, hi = nf - 1;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (cum[mid] >= target) hi = mid;
    else lo = mid + 1;
  }
  double l0 = uniforms[3 * i + 1], l1 = uniforms[3 * i + 2];
  if (dadd(l0, l1) > 1.0) { l0 = fabs(dsub(l0, 1.0)); l1 = fabs(dsub(l1, 1.0)); }
  const long long a = faces[3 * lo], b = faces[3 * lo + 1], c = faces[3 * lo + 2];
  const bool ok = a >= 0 && a < nv && b >= 0 && b < nv && c >= 0 && c < nv;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    double s = nan("");
    if (ok) {
      const double v0 = verts[3 * a + j];
      s = dadd(dadd(dmul(dsub(verts[3 * b + j], v0), l0), dmul(dsub(verts[3 * c + j], v0), l1)), v0);
    }
    samples[3 * i + j] = s;
  }
  if (face_index) face_index[i] = lo;
}

int sample_cub_bytes(long long nf, size_t* b) {
  GS_CUDA(cub::DeviceScan::InclusiveSum(nullptr, *b, (const double*)nullptr, (double*)nullptr, (int)nf));
  return GOSLAM_OK;
}

struct SampleWork { double* area; double* cum; void* cub_tmp; size_t cub_bytes; };

size_t sample_layout(long long nf, size_t cub_bytes, void* base, SampleWork* w) {
  GsArena ar(base);
  w->area = ar.take<double>(nf);
  w->cum = ar.take<double>(nf);
  w->cub_tmp = ar.take<unsigned char>(cub_bytes);
  w->cub_bytes = cub_bytes;
  return ar.off;
}

// ---- nearest-neighbour grid ---------------------------------------------------------------------------------------
struct NnParams {
  double o[3];      // grid origin = the points' box minimum
  double hi[3];     // the points' box maximum
  double h, inv_h;  // cell size and its reciprocal
  double slack;     // absolute margin of the shell bound
  int d[3];         // cells per axis
};

struct NnIndex {
  NnParams* params;
  unsigned* cell_start;  // [max_cells + 1]
  unsigned* keys[2];
  unsigned* vals[2];
  unsigned* ids;         // point id of each sorted position
  double* pts;           // [n,3] in sorted order
  double* box;           // per-block box partials [kBoxBlocks, 6]
  void* cub_tmp;
  size_t cub_bytes;
};

__host__ __device__ inline long long max_cells(long long n) { return 2 * n + 64; }

int key_bits(long long n) {
  int b = 1;
  while ((1ll << b) <= max_cells(n)) ++b;
  return b;
}

int nn_cub_bytes(long long n, size_t* b) {
  cub::DoubleBuffer<unsigned> k(nullptr, nullptr), v(nullptr, nullptr);
  GS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, *b, k, v, (int)n));
  return GOSLAM_OK;
}

size_t nn_layout(long long n, size_t cub_bytes, const void* base, NnIndex* x) {
  GsArena ar(base);
  x->params = ar.take<NnParams>(1);
  x->cell_start = ar.take<unsigned>(max_cells(n) + 1);
  for (int i = 0; i < 2; ++i) {
    x->keys[i] = ar.take<unsigned>(n);
    x->vals[i] = ar.take<unsigned>(n);
  }
  x->ids = ar.take<unsigned>(n);
  x->pts = ar.take<double>(3 * n);
  x->box = ar.take<double>(6 * kBoxBlocks);
  x->cub_tmp = ar.take<unsigned char>(cub_bytes);
  x->cub_bytes = cub_bytes;
  return ar.off;
}

__global__ void __launch_bounds__(kThreads) box_kernel(const double* p, long long n, double* box) {
  __shared__ double sh[6][kThreads];
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double v = p[3 * i + j];
      lo[j] = fmin(lo[j], v);
      hi[j] = fmax(hi[j], v);
    }
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) { sh[j][threadIdx.x] = lo[j]; sh[3 + j][threadIdx.x] = hi[j]; }
  __syncthreads();
  for (int h = kThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        sh[j][threadIdx.x] = fmin(sh[j][threadIdx.x], sh[j][threadIdx.x + h]);
        sh[3 + j][threadIdx.x] = fmax(sh[3 + j][threadIdx.x], sh[3 + j][threadIdx.x + h]);
      }
    }
    __syncthreads();
  }
  if (threadIdx.x < 6) box[6 * blockIdx.x + threadIdx.x] = sh[threadIdx.x][0];
}

__device__ double grid_cells(const double* ext, double inv_h) {
  double c = 1.0;
  for (int j = 0; j < 3; ++j) c *= floor(ext[j] * inv_h) + 1.0;
  return c;
}

// one thread: the box from the partials, then the cell size
__global__ void params_kernel(const double* box, int nb, long long n, double min_cell, NnParams* P) {
  if (threadIdx.x != 0) return;
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int b = 0; b < nb; ++b)
    for (int j = 0; j < 3; ++j) { lo[j] = fmin(lo[j], box[6 * b + j]); hi[j] = fmax(hi[j], box[6 * b + 3 + j]); }
  double ext[3], emax = 0.0, scale = min_cell;
  for (int j = 0; j < 3; ++j) {
    ext[j] = isfinite(hi[j] - lo[j]) ? hi[j] - lo[j] : 0.0;
    emax = fmax(emax, ext[j]);
    scale = fmax(scale, fmax(fabs(lo[j]), fabs(hi[j])));
  }
  double h = 1.0;
  if (emax > 0.0) {
    double vol = 1.0;
    for (int j = 0; j < 3; ++j) vol *= fmax(ext[j], 1e-3 * emax);
    h = cbrt(vol / (double)n);
  }
  h = fmax(h, min_cell);
  const double limit = (double)max_cells(n);
  for (int g = 0; g < 512 && grid_cells(ext, 1.0 / h) > limit; ++g) h *= 1.25;
  const double inv_h = 1.0 / h;
  for (int j = 0; j < 3; ++j) {
    P->o[j] = lo[j];
    P->hi[j] = hi[j];
    P->d[j] = (int)(floor(ext[j] * inv_h) + 1.0);
  }
  P->h = h;
  P->inv_h = inv_h;
  P->slack = 1e-12 * (scale + emax + h);
}

__device__ __forceinline__ int cell_of(double v, double o, double inv_h, int d) {
  const double c = floor(dmul(dsub(v, o), inv_h));
  return c >= 0.0 ? (c > (double)(d - 1) ? d - 1 : (int)c) : 0;      // NaN -> 0
}

__global__ void __launch_bounds__(kThreads) key_kernel(const double* p, long long n, const NnParams* P, unsigned* keys,
                                                       unsigned* vals) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const double inv_h = P->inv_h;
  const int cx = cell_of(p[3 * i], P->o[0], inv_h, P->d[0]);
  const int cy = cell_of(p[3 * i + 1], P->o[1], inv_h, P->d[1]);
  const int cz = cell_of(p[3 * i + 2], P->o[2], inv_h, P->d[2]);
  keys[i] = ((unsigned)cz * (unsigned)P->d[1] + (unsigned)cy) * (unsigned)P->d[0] + (unsigned)cx;
  vals[i] = (unsigned)i;
}

__global__ void __launch_bounds__(kThreads) gather_kernel(const double* p, long long n, const unsigned* vals, unsigned* ids,
                                                          double* pts) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const unsigned id = vals[i];
  ids[i] = id;
  pts[3 * i] = p[3 * (long long)id];
  pts[3 * i + 1] = p[3 * (long long)id + 1];
  pts[3 * i + 2] = p[3 * (long long)id + 2];
}

// cell_start[c] = the first sorted position whose key is >= c
__global__ void __launch_bounds__(kThreads) cell_start_kernel(const unsigned* keys, long long n, long long nc,
                                                              unsigned* cell_start) {
  const long long c = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (c > nc) return;
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if ((long long)keys[mid] >= c) hi = mid;
    else lo = mid + 1;
  }
  cell_start[c] = (unsigned)lo;
}

struct Best { double d2; long long pos; unsigned id; };

__device__ __forceinline__ void scan_run(const double* pts, const unsigned* ids, unsigned b, unsigned e, double qx, double qy,
                                         double qz, Best& best) {
  for (unsigned j = b; j < e; ++j) {
    const double dx = dsub(qx, pts[3 * j]), dy = dsub(qy, pts[3 * j + 1]), dz = dsub(qz, pts[3 * j + 2]);
    const double d2 = dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz));
    if (d2 < best.d2 || (best.pos >= 0 && d2 == best.d2 && ids[j] < best.id)) {
      best.d2 = d2; best.pos = j; best.id = ids[j];
    }
  }
}

// the nearest point to q with d2 < r2 (r2 = +inf: unbounded); pos -1 if there is none
__device__ Best nn_search(const NnParams& P, const unsigned* cell_start, const double* pts, const unsigned* ids, double qx,
                          double qy, double qz, double r2) {
  const double q[3] = {qx, qy, qz};
  int c[3];
  double g2[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    c[j] = cell_of(q[j], P.o[j], P.inv_h, P.d[j]);
    const double g = fmax(0.0, fmax(dsub(P.o[j], q[j]), dsub(q[j], P.hi[j])));
    g2[j] = dmul(g, g);
  }
  Best best{r2, -1, 0u};
  for (int k = 0;; ++k) {
    const int z0 = max(c[2] - k, 0), z1 = min(c[2] + k, P.d[2] - 1);
    const int y0 = max(c[1] - k, 0), y1 = min(c[1] + k, P.d[1] - 1);
    const int x0 = max(c[0] - k, 0), x1 = min(c[0] + k, P.d[0] - 1);
    for (int z = z0; z <= z1; ++z) {
      for (int y = y0; y <= y1; ++y) {
        const unsigned row = ((unsigned)z * (unsigned)P.d[1] + (unsigned)y) * (unsigned)P.d[0];
        if (z == c[2] - k || z == c[2] + k || y == c[1] - k || y == c[1] + k) {
          // a whole row of the shell: its cells are consecutive keys, so their points are one sorted run
          scan_run(pts, ids, cell_start[row + x0], cell_start[row + x1 + 1], qx, qy, qz, best);
        } else {
          if (c[0] - k >= 0) scan_run(pts, ids, cell_start[row + c[0] - k], cell_start[row + c[0] - k + 1], qx, qy, qz, best);
          if (k > 0 && c[0] + k < P.d[0])
            scan_run(pts, ids, cell_start[row + c[0] + k], cell_start[row + c[0] + k + 1], qx, qy, qz, best);
        }
      }
    }
    // lower bound on the distance to every point outside the visited cube of cells
    double L2 = INFINITY;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double rest = dadd(g2[(j + 1) % 3], g2[(j + 2) % 3]);
      if (c[j] + k + 1 < P.d[j]) {
        const double b = dadd(P.o[j], dmul((double)(c[j] + k + 1), P.h));
        const double g = fmax(0.0, fmax(dsub(b, q[j]), dsub(q[j], P.hi[j])));
        L2 = fmin(L2, dadd(rest, dmul(g, g)));
      }
      if (c[j] - k - 1 >= 0) {
        const double b = dadd(P.o[j], dmul((double)(c[j] - k), P.h));
        const double g = fmax(0.0, fmax(dsub(q[j], b), dsub(P.o[j], q[j])));
        L2 = fmin(L2, dadd(rest, dmul(g, g)));
      }
    }
    if (L2 == INFINITY) break;
    const double L = sqrt(L2) - P.slack;
    if (L > 0.0) {
      const double LL = L * L;
      if (LL > best.d2 || (best.pos < 0 && LL >= best.d2)) break;
    }
  }
  return best;
}

__global__ void __launch_bounds__(kThreads) query_kernel(const NnParams* Pp, const unsigned* cell_start, const double* pts,
                                                         const unsigned* ids, const double* q, long long nq, double r2,
                                                         double* dist, long long* idx) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= nq) return;
  const NnParams P = *Pp;
  const Best b = nn_search(P, cell_start, pts, ids, q[3 * i], q[3 * i + 1], q[3 * i + 2], r2);
  if (dist) dist[i] = b.pos >= 0 ? __dsqrt_rn(b.d2) : INFINITY;
  if (idx) idx[i] = b.pos >= 0 ? (long long)b.id : -1;
}

// one block: sum of dist and count of dist < threshold (per-thread strided sums, fixed tree)
constexpr int kStatThreads = 1024;
__global__ void __launch_bounds__(kStatThreads) stats_kernel(const double* dist, long long n, double threshold, double* out) {
  __shared__ double s_sum[kStatThreads];
  __shared__ long long s_cnt[kStatThreads];
  double sum = 0.0;
  long long cnt = 0;
  for (long long i = threadIdx.x; i < n; i += kStatThreads) {
    const double d = dist[i];
    sum = dadd(sum, d);
    cnt += d < threshold;
  }
  s_sum[threadIdx.x] = sum; s_cnt[threadIdx.x] = cnt;
  __syncthreads();
  for (int h = kStatThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      s_sum[threadIdx.x] = dadd(s_sum[threadIdx.x], s_sum[threadIdx.x + h]);
      s_cnt[threadIdx.x] += s_cnt[threadIdx.x + h];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[0] = s_sum[0]; out[1] = (double)s_cnt[0]; }
}

// ---- ICP ----------------------------------------------------------------------------------------------------------
struct IcpState {
  double T[16];        // the accumulated transformation (row-major)
  double upd[16];      // the latest update
  double fitness, rmse;
  double mean_s[3], mean_d[3];
  double count;
  int iterations;
  int done;
};

struct IcpWork { IcpState* state; double* work; int* corr; double* part; };

size_t icp_layout(long long n, void* base, IcpWork* w) {
  GsArena ar(base);
  w->state = ar.take<IcpState>(1);
  w->work = ar.take<double>(3 * n);
  w->corr = ar.take<int>(n);
  w->part = ar.take<double>(9 * (size_t)blocks_for(n, kThreads));
  return ar.off;
}

__global__ void icp_init_kernel(const double* init, IcpState* s) {
  const int t = threadIdx.x;
  if (t < 16) { s->T[t] = init[t]; s->upd[t] = (t % 5 == 0) ? 1.0 : 0.0; }
  if (t == 0) { s->fitness = 0.0; s->rmse = 0.0; s->count = 0.0; s->iterations = 0; s->done = 0; }
}

// p <- M p as a general 4x4 (x' = ((m0 x + m1 y) + m2 z) + m3, divided by w'), on the working copy
__global__ void __launch_bounds__(kThreads) icp_transform_kernel(const double* src, long long n, const IcpState* s,
                                                                 int use_T, double* work) {
  if (s->done) return;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const double* M = use_T ? s->T : s->upd;
  const double* p = use_T ? src : work;
  const double x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
  double r[4];
#pragma unroll
  for (int a = 0; a < 4; ++a) r[a] = dadd(dadd(dadd(dmul(M[4 * a], x), dmul(M[4 * a + 1], y)), dmul(M[4 * a + 2], z)), M[4 * a + 3]);
  work[3 * i] = __ddiv_rn(r[0], r[3]);
  work[3 * i + 1] = __ddiv_rn(r[1], r[3]);
  work[3 * i + 2] = __ddiv_rn(r[2], r[3]);
}

// correspondences (radius search) and per-block partials: count, sum d2, sum src (3), sum dst (3)
__global__ void __launch_bounds__(kThreads) icp_correspond_kernel(const double* work, long long n, const NnParams* Pp,
                                                                  const unsigned* cell_start, const double* pts,
                                                                  const unsigned* ids, double r2, const IcpState* s,
                                                                  int* corr, double* part) {
  __shared__ double sh[8][kThreads];
  if (s->done) return;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (i < n) {
    const NnParams P = *Pp;
    const double x = work[3 * i], y = work[3 * i + 1], z = work[3 * i + 2];
    const Best b = nn_search(P, cell_start, pts, ids, x, y, z, r2);
    corr[i] = (int)b.pos;
    if (b.pos >= 0) {
      v[0] = 1.0; v[1] = b.d2;
      v[2] = x; v[3] = y; v[4] = z;
      v[5] = pts[3 * b.pos]; v[6] = pts[3 * b.pos + 1]; v[7] = pts[3 * b.pos + 2];
    }
  }
  gs_block_sum(v, sh);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 8; ++k) part[8 * (long long)blockIdx.x + k] = v[k];
  }
}

// one block: the correspondence set's fitness, rmse and means; the convergence test after an update (it > 0)
__global__ void __launch_bounds__(kThreads) icp_reduce_kernel(const double* part, int nb, long long n_src, int it,
                                                              double rel_fitness, double rel_rmse, IcpState* s) {
  __shared__ double sh[8][kThreads];
  if (s->done) return;
  double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int b = threadIdx.x; b < nb; b += kThreads) {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = dadd(v[k], part[8 * (long long)b + k]);
  }
  gs_block_sum(v, sh);
  if (threadIdx.x != 0) return;
  const double cnt = v[0];
  double fitness = 0.0, rmse = 0.0;
  if (cnt > 0.0) {
    fitness = __ddiv_rn(cnt, (double)n_src);
    rmse = __dsqrt_rn(__ddiv_rn(v[1], cnt));
    const double inv = __ddiv_rn(1.0, cnt);
    for (int j = 0; j < 3; ++j) { s->mean_s[j] = dmul(v[2 + j], inv); s->mean_d[j] = dmul(v[5 + j], inv); }
  }
  if (it > 0) {
    s->iterations = it;
    if (fabs(s->fitness - fitness) < rel_fitness && fabs(s->rmse - rmse) < rel_rmse) s->done = 1;
  }
  s->count = cnt;
  s->fitness = fitness;
  s->rmse = rmse;
}

// per-block partials of sum over correspondences of (d - mean_d)(s - mean_s)^T, row-major
__global__ void __launch_bounds__(kThreads) icp_cov_kernel(const double* work, long long n, const int* corr, const double* pts,
                                                           const IcpState* s, double* part) {
  __shared__ double sh[9][kThreads];
  if (s->done) return;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  double v[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (i < n && corr[i] >= 0) {
    const long long c = corr[i];
    double a[3], b[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) { b[j] = dsub(work[3 * i + j], s->mean_s[j]); a[j] = dsub(pts[3 * c + j], s->mean_d[j]); }
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = 0; q < 3; ++q) v[3 * r + q] = dmul(a[r], b[q]);
  }
  gs_block_sum(v, sh);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 9; ++k) part[9 * (long long)blockIdx.x + k] = v[k];
  }
}

// the rotation of Umeyama's method (no scaling) for the cross-covariance A: U diag(1, 1, det(U) det(V) < 0 ? -1 : 1) V^T.
// gs_umeyama_svd; u3 is taken as u1 x u2, for which the product reduces to u1 v1^T + u2 v2^T + det(V) (u1 x u2) v3^T,
// also for rank 2.  Rank < 2 (s2 <= 1e-14 s1): the rotation is not unique and the identity is returned.
__device__ void umeyama_rotation(const double A[9], double R[9]) {
  double B[9], V[9], sv[3];
  int ord[3];
  gs_umeyama_svd(A, B, V, sv, ord);
  for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.0 : 0.0;
  const double s1 = sv[ord[0]], s2 = sv[ord[1]];
  if (!(s1 > 0.0) || !(s2 > 1e-14 * s1)) return;
  double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3];
  for (int r = 0; r < 3; ++r) {
    u1[r] = B[3 * r + ord[0]] / s1;
    u2[r] = B[3 * r + ord[1]] / s2;
    v1[r] = V[3 * r + ord[0]]; v2[r] = V[3 * r + ord[1]]; v3[r] = V[3 * r + ord[2]];
  }
  u3[0] = u1[1] * u2[2] - u1[2] * u2[1];
  u3[1] = u1[2] * u2[0] - u1[0] * u2[2];
  u3[2] = u1[0] * u2[1] - u1[1] * u2[0];
  const double detv = v1[0] * (v2[1] * v3[2] - v2[2] * v3[1]) - v1[1] * (v2[0] * v3[2] - v2[2] * v3[0]) +
                      v1[2] * (v2[0] * v3[1] - v2[1] * v3[0]);
  const double sg = detv < 0.0 ? -1.0 : 1.0;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) R[3 * a + b] = u1[a] * v1[b] + u2[a] * v2[b] + sg * u3[a] * v3[b];
}

// one block: reduce the covariance partials, solve for the update (identity without correspondences), T <- update T
__global__ void __launch_bounds__(kThreads) icp_solve_kernel(const double* part, int nb, IcpState* s) {
  __shared__ double sh[9][kThreads];
  if (s->done) return;
  double v[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int b = threadIdx.x; b < nb; b += kThreads) {
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = dadd(v[k], part[9 * (long long)b + k]);
  }
  gs_block_sum(v, sh);
  if (threadIdx.x != 0) return;
  double U[16];
  for (int k = 0; k < 16; ++k) U[k] = (k % 5 == 0) ? 1.0 : 0.0;
  if (s->count > 0.0) {
    const double inv = __ddiv_rn(1.0, s->count);
    double A[9], R[9];
    for (int k = 0; k < 9; ++k) A[k] = dmul(inv, v[k]);
    umeyama_rotation(A, R);
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 3; ++b) U[4 * a + b] = R[3 * a + b];
      const double rm = dadd(dadd(dmul(R[3 * a], s->mean_s[0]), dmul(R[3 * a + 1], s->mean_s[1])), dmul(R[3 * a + 2], s->mean_s[2]));
      U[4 * a + 3] = dsub(s->mean_d[a], rm);
    }
  }
  double T[16];
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < 4; ++b) {
      double acc = dmul(U[4 * a], s->T[b]);
      for (int k = 1; k < 4; ++k) acc = dadd(acc, dmul(U[4 * a + k], s->T[4 * k + b]));
      T[4 * a + b] = acc;
    }
  for (int k = 0; k < 16; ++k) { s->upd[k] = U[k]; s->T[k] = T[k]; }
}

__global__ void icp_result_kernel(const IcpState* s, double* out) {
  const int t = threadIdx.x;
  if (t < 16) out[t] = s->T[t];
  if (t == 16) out[16] = s->fitness;
  if (t == 17) out[17] = s->rmse;
  if (t == 18) out[18] = (double)s->iterations;
}

}  // namespace

extern "C" {

size_t goslam_mesh_sample_workspace_bytes(int64_t n_faces) {
  if (n_faces < 1 || n_faces > kMaxFaces) return 0;
  size_t cb = 0;
  if (sample_cub_bytes(n_faces, &cb) != GOSLAM_OK) return 0;
  SampleWork w;
  return sample_layout(n_faces, cb, nullptr, &w);
}

int goslam_mesh_sample_surface(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                               const double* uniforms, int64_t count, double* samples, int64_t* face_index,
                               void* workspace, size_t workspace_bytes, void* stream) {
  if (n_verts < 1 || n_faces < 1 || n_faces > kMaxFaces || count < 0 || !verts || !faces ||
      (count > 0 && (!uniforms || !samples)))
    return GOSLAM_EINVAL;
  if (!workspace) return GOSLAM_EWORKSPACE;     // refused before the CUB size query, which needs a device
  size_t cb = 0;
  if (const int rc = sample_cub_bytes(n_faces, &cb)) return rc;
  SampleWork w;
  if (workspace_bytes < sample_layout(n_faces, cb, workspace, &w)) return GOSLAM_EWORKSPACE;
  if (count == 0) return GOSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  area_kernel<<<blocks_for(n_faces, kThreads), kThreads, 0, st>>>(verts, n_verts, (const long long*)faces, n_faces, w.area);
  GS_CHECK_LAUNCH();
  size_t tb = w.cub_bytes;
  GS_CUDA(cub::DeviceScan::InclusiveSum(w.cub_tmp, tb, w.area, w.cum, (int)n_faces, st));
  sample_kernel<<<blocks_for(count, kThreads), kThreads, 0, st>>>(verts, n_verts, (const long long*)faces, n_faces, w.cum,
                                                                  uniforms, count, samples, (long long*)face_index);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

size_t goslam_nn_index_workspace_bytes(int64_t n_points) {
  if (n_points < 1 || n_points > kMaxPoints) return 0;
  size_t cb = 0;
  if (nn_cub_bytes(n_points, &cb) != GOSLAM_OK) return 0;
  NnIndex x;
  return nn_layout(n_points, cb, nullptr, &x);
}

int goslam_nn_index_build(const double* points, int64_t n_points, double min_cell, void* index, size_t index_bytes,
                          void* stream) {
  if (n_points < 1 || n_points > kMaxPoints || !points || !(min_cell >= 0.0) || !(min_cell < INFINITY))
    return GOSLAM_EINVAL;
  if (!index) return GOSLAM_EWORKSPACE;     // refused before the CUB size query, which needs a device
  size_t cb = 0;
  if (const int rc = nn_cub_bytes(n_points, &cb)) return rc;
  NnIndex x;
  if (index_bytes < nn_layout(n_points, cb, index, &x)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = (int)std::min<long long>(blocks_for(n_points, kThreads), kBoxBlocks);
  box_kernel<<<nb, kThreads, 0, st>>>(points, n_points, x.box);
  GS_CHECK_LAUNCH();
  params_kernel<<<1, 32, 0, st>>>(x.box, nb, n_points, min_cell, x.params);
  GS_CHECK_LAUNCH();
  key_kernel<<<blocks_for(n_points, kThreads), kThreads, 0, st>>>(points, n_points, x.params, x.keys[0], x.vals[0]);
  GS_CHECK_LAUNCH();
  cub::DoubleBuffer<unsigned> kb(x.keys[0], x.keys[1]), vb(x.vals[0], x.vals[1]);
  size_t tb = x.cub_bytes;
  GS_CUDA(cub::DeviceRadixSort::SortPairs(x.cub_tmp, tb, kb, vb, (int)n_points, 0, key_bits(n_points), st));
  gather_kernel<<<blocks_for(n_points, kThreads), kThreads, 0, st>>>(points, n_points, vb.Current(), x.ids, x.pts);
  GS_CHECK_LAUNCH();
  const long long nc = max_cells(n_points);
  cell_start_kernel<<<blocks_for(nc + 1, kThreads), kThreads, 0, st>>>(kb.Current(), n_points, nc, x.cell_start);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_nn_query(const void* index, size_t index_bytes, int64_t n_points, const double* query, int64_t n_query,
                    double max_dist, double* dist, int64_t* idx, void* stream) {
  if (n_points < 1 || n_points > kMaxPoints || n_query < 0 || (n_query > 0 && (!query || (!dist && !idx))) ||
      !(max_dist > 0.0))
    return GOSLAM_EINVAL;
  if (!index) return GOSLAM_EWORKSPACE;     // refused before the CUB size query, which needs a device
  size_t cb = 0;
  if (const int rc = nn_cub_bytes(n_points, &cb)) return rc;
  NnIndex x;
  if (index_bytes < nn_layout(n_points, cb, index, &x)) return GOSLAM_EWORKSPACE;
  if (n_query == 0) return GOSLAM_OK;
  const double r2 = max_dist == INFINITY ? INFINITY : max_dist * max_dist;
  query_kernel<<<blocks_for(n_query, kThreads), kThreads, 0, (cudaStream_t)stream>>>(x.params, x.cell_start, x.pts, x.ids,
                                                                                     query, n_query, r2, dist,
                                                                                     (long long*)idx);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_nn_distance_stats(const double* dist, int64_t n, double threshold, double* out, void* stream) {
  if (n < 0 || (n > 0 && !dist) || !out || threshold != threshold) return GOSLAM_EINVAL;
  stats_kernel<<<1, kStatThreads, 0, (cudaStream_t)stream>>>(dist, n, threshold, out);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

size_t goslam_icp_workspace_bytes(int64_t n_source) {
  if (n_source < 1 || n_source > kMaxPoints) return 0;
  IcpWork w;
  return icp_layout(n_source, nullptr, &w);
}

int goslam_icp_point_to_point(const double* source, int64_t n_source, const void* index, size_t index_bytes,
                              int64_t n_target, double threshold, const double* init, int max_iteration,
                              double relative_fitness, double relative_rmse, double* result, void* workspace,
                              size_t workspace_bytes, void* stream) {
  if (n_source < 1 || n_source > kMaxPoints || n_target < 1 || n_target > kMaxPoints || !source || !init || !result ||
      !(threshold > 0.0) || !(threshold < INFINITY) || max_iteration < 0 || relative_fitness != relative_fitness ||
      relative_rmse != relative_rmse)
    return GOSLAM_EINVAL;
  if (!index || !workspace) return GOSLAM_EWORKSPACE;     // refused before the CUB size query, which needs a device
  size_t cb = 0;
  if (const int rc = nn_cub_bytes(n_target, &cb)) return rc;
  NnIndex x;
  if (index_bytes < nn_layout(n_target, cb, index, &x)) return GOSLAM_EWORKSPACE;
  IcpWork w;
  if (workspace_bytes < icp_layout(n_source, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned nb = blocks_for(n_source, kThreads);
  const double r2 = threshold * threshold;
  icp_init_kernel<<<1, 32, 0, st>>>(init, w.state);
  GS_CHECK_LAUNCH();
  icp_transform_kernel<<<nb, kThreads, 0, st>>>(source, n_source, w.state, 1, w.work);
  GS_CHECK_LAUNCH();
  for (int it = 0; it <= max_iteration; ++it) {
    if (it > 0) {
      icp_cov_kernel<<<nb, kThreads, 0, st>>>(w.work, n_source, w.corr, x.pts, w.state, w.part);
      GS_CHECK_LAUNCH();
      icp_solve_kernel<<<1, kThreads, 0, st>>>(w.part, (int)nb, w.state);
      GS_CHECK_LAUNCH();
      icp_transform_kernel<<<nb, kThreads, 0, st>>>(source, n_source, w.state, 0, w.work);
      GS_CHECK_LAUNCH();
    }
    icp_correspond_kernel<<<nb, kThreads, 0, st>>>(w.work, n_source, x.params, x.cell_start, x.pts, x.ids, r2, w.state,
                                                   w.corr, w.part);
    GS_CHECK_LAUNCH();
    icp_reduce_kernel<<<1, kThreads, 0, st>>>(w.part, (int)nb, n_source, it, relative_fitness, relative_rmse, w.state);
    GS_CHECK_LAUNCH();
  }
  icp_result_kernel<<<1, 32, 0, st>>>(w.state, result);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
