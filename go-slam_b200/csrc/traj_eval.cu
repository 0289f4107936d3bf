// traj_eval.cu — the trajectory error of SLAM.terminate (src/slam.py:341-370) on the device: evo's APE w.r.t. the
// translation part after a Sim(3) Umeyama alignment (main_ape.ape(..., align=True, correct_scale=True)).
//
//  * rows: row i is kept iff the fp64 sum of its 16 reference entries, in numpy's pairwise order, is finite; the kept
//    row ids in input order come from an ordered CUB select.  The kept count stays on the device: every later kernel
//    reads it there, so the host never waits.
//  * Umeyama with scale (evo geometry.umeyama_alignment): x = estimate positions, y = reference translations; means,
//    sigma_x^2 = (1/n) sum |x - mx|^2, C = (1/n) sum (y - my)(x - mx)^T, the SVD of C on the ICP's Jacobi SVD
//    (gs_umeyama_svd), degenerate unless two singular values exceed numpy's eps, R = U S V^T, c = (1 / sigma_x^2) trace(D S),
//    t = my - c (R mx).  With u3 = u1 x u2 (as the ICP), trace(D S) = s1 + s2 + det(V) <b3, u1 x u2>, b3 = A v3: neither
//    det(U) nor a division by a tiny s3 is needed.
//  * errors e_i = |(R (c x_i) + t) - y_i|; rmse, mean, std (two-pass), sse from fixed-order sums; min, median, max from
//    a CUB radix sort of the errors (padded with +inf up to n).
//  * every sum is per-thread partials in a grid of fixed size (a function of n only), a fixed tree per block and a
//    one-block finish in block order, every operation rounded on its own (no FMA): two runs are bit-identical.
#include <cub/cub.cuh>

#include "common.cuh"
#include "mesh_geom.cuh"

namespace {

constexpr int kThreads = 256;
constexpr long long kMaxRows = (1ll << 31) - 1;   // CUB item counts are int
constexpr int kMaxBlocks = 4 * kNumSms;
constexpr double kEps = 2.220446049250313e-16;    // np.finfo(np.float64).eps, evo's (absolute) rank threshold

__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }
int partial_blocks(long long n) { return (int)std::min<long long>(blocks_for(std::max<long long>(n, 1)), kMaxBlocks); }

struct ApeState {
  int m;            // kept rows (the select's count)
  int status;       // GOSLAM_APE_*
  double mx[3], my[3];
  double sx2;       // sigma_x^2
  double sv[3];     // singular values of C, descending
  double c, R[9], t[3];
  double mean, sse;
};

struct ApeWork {
  ApeState* state;
  unsigned char* flag;
  int* kept;
  double* xs;       // [m,3] kept estimate positions
  double* ys;       // [m,3] kept reference translations
  double* keys;     // [n] errors, +inf past m
  double* sorted;   // [n]
  double* part;     // [blocks, 10]
  void* cub_tmp;
  size_t cub_bytes;
};

// the CUB temporary bytes of the select and the sort; a failed size query (no device) is reported by the calls
size_t cub_bytes(long long n) {
  const int items = (int)std::max<long long>(n, 1);
  size_t a = 0, b = 0;
  cub::DeviceSelect::Flagged(nullptr, a, cub::CountingInputIterator<int>(0), (const unsigned char*)nullptr,
                             (int*)nullptr, (int*)nullptr, items);
  cub::DeviceRadixSort::SortKeys(nullptr, b, (const double*)nullptr, (double*)nullptr, items);
  return std::max<size_t>(std::max(a, b), 1);
}

size_t ape_layout(long long n, void* base, ApeWork* w) {
  GsArena ar(base);
  const size_t rows = (size_t)std::max<long long>(n, 1);
  w->state = ar.take<ApeState>(1);
  w->flag = ar.take<unsigned char>(rows);
  w->kept = ar.take<int>(rows);
  w->xs = ar.take<double>(3 * rows);
  w->ys = ar.take<double>(3 * rows);
  w->keys = ar.take<double>(rows);
  w->sorted = ar.take<double>(rows);
  w->part = ar.take<double>(10 * (size_t)partial_blocks(n));
  w->cub_bytes = cub_bytes(n);
  w->cub_tmp = ar.take<unsigned char>(w->cub_bytes);
  return ar.off;
}

// K partial sums per block into part[K * block]
template <int K>
__device__ __forceinline__ void write_partials(double (&v)[K], double (*sh)[kThreads], double* part) {
  gs_block_sum(v, sh);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) part[K * blockIdx.x + k] = v[k];
  }
}

// one block: the nb blocks' partials summed in block order; valid in thread 0
template <int K>
__device__ __forceinline__ void sum_partials(const double* part, int nb, double (&v)[K], double (*sh)[kThreads]) {
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = 0.0;
  for (int b = threadIdx.x; b < nb; b += kThreads) {
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = dadd(v[k], part[K * b + k]);
  }
  gs_block_sum(v, sh);
}

__global__ void ape_init_kernel(ApeState* s) {
  if (threadIdx.x != 0) return;
  s->m = 0;
  s->status = GOSLAM_APE_NO_ROWS;
  for (int k = 0; k < 3; ++k) s->sv[k] = nan("");
}

// row i is kept iff np.sum(ref[i]) is finite: numpy's pairwise sum of 16 contiguous doubles (eight running sums, then
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)))
__global__ void __launch_bounds__(kThreads) ape_keep_kernel(const double* ref, long long n, unsigned char* flag) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const double* p = ref + 16 * i;
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = dadd(p[j], p[8 + j]);
  const double sum = dadd(dadd(dadd(r[0], r[1]), dadd(r[2], r[3])), dadd(dadd(r[4], r[5]), dadd(r[6], r[7])));
  flag[i] = isfinite(sum) ? 1 : 0;
}

// the kept rows gathered (x = estimate, y = reference translation); partials of sum x, sum y, non-finite estimates
__global__ void __launch_bounds__(kThreads) ape_gather_kernel(const double* est, const double* ref, const int* kept,
                                                              const ApeState* s, double* xs, double* ys, double* part) {
  __shared__ double sh[7][kThreads];
  const long long m = s->m;
  double v[7] = {0, 0, 0, 0, 0, 0, 0};
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < m; i += (long long)gridDim.x * kThreads) {
    const long long r = kept[i];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double x = est[3 * r + j], y = ref[16 * r + 4 * j + 3];
      xs[3 * i + j] = x;
      ys[3 * i + j] = y;
      v[j] = dadd(v[j], x);
      v[3 + j] = dadd(v[3 + j], y);
      if (!isfinite(x)) v[6] = 1.0;
    }
  }
  write_partials(v, sh, part);
}

// one block: the status and the means (x.mean(axis=1): the sum divided by n)
__global__ void __launch_bounds__(kThreads) ape_mean_kernel(const double* part, int nb, ApeState* s) {
  __shared__ double sh[7][kThreads];
  double v[7];
  sum_partials(part, nb, v, sh);
  if (threadIdx.x != 0) return;
  const int m = s->m;
  s->status = m == 0 ? GOSLAM_APE_NO_ROWS : v[6] != 0.0 ? GOSLAM_APE_NONFINITE_ESTIMATE : GOSLAM_APE_OK;
  for (int j = 0; j < 3; ++j) {
    s->mx[j] = ddiv(v[j], (double)m);
    s->my[j] = ddiv(v[3 + j], (double)m);
  }
}

// partials of sum |x - mx|^2 and sum (y - my)(x - mx)^T (row-major)
__global__ void __launch_bounds__(kThreads) ape_cov_kernel(const double* xs, const double* ys, const ApeState* s,
                                                           double* part) {
  __shared__ double sh[10][kThreads];
  if (s->status != GOSLAM_APE_OK) return;
  const long long m = s->m;
  double v[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < m; i += (long long)gridDim.x * kThreads) {
    double a[3], b[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) { a[j] = dsub(xs[3 * i + j], s->mx[j]); b[j] = dsub(ys[3 * i + j], s->my[j]); }
    v[0] = dadd(v[0], dadd(dadd(dmul(a[0], a[0]), dmul(a[1], a[1])), dmul(a[2], a[2])));
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = 0; q < 3; ++q) v[1 + 3 * r + q] = dadd(v[1 + 3 * r + q], dmul(b[r], a[q]));
  }
  write_partials(v, sh, part);
}

// one block, one thread after the sums: Umeyama's Sim(3) (evo's rank rule and sign rule)
__global__ void __launch_bounds__(kThreads) ape_solve_kernel(const double* part, int nb, ApeState* s) {
  __shared__ double sh[10][kThreads];
  if (s->status != GOSLAM_APE_OK) return;
  double v[10];
  sum_partials(part, nb, v, sh);
  if (threadIdx.x != 0) return;
  const int m = s->m;
  const double inv = ddiv(1.0, (double)m);
  const double sx2 = dmul(inv, v[0]);
  double A[9], B[9], V[9], sv[3];
  int ord[3];
  for (int k = 0; k < 9; ++k) A[k] = dmul(inv, v[1 + k]);
  gs_umeyama_svd(A, B, V, sv, ord);
  const double s1 = sv[ord[0]], s2 = sv[ord[1]], s3 = sv[ord[2]];
  s->sv[0] = s1; s->sv[1] = s2; s->sv[2] = s3;
  s->sx2 = sx2;
  // fewer than three rows span at most a line: rank <= 1 whatever the rounding makes of the second singular value
  if (m < 3 || (s1 > kEps) + (s2 > kEps) + (s3 > kEps) < 2) { s->status = GOSLAM_APE_DEGENERATE; return; }
  double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3], b3[3];
  for (int r = 0; r < 3; ++r) {
    u1[r] = ddiv(B[3 * r + ord[0]], s1);
    u2[r] = ddiv(B[3 * r + ord[1]], s2);
    b3[r] = B[3 * r + ord[2]];
    v1[r] = V[3 * r + ord[0]]; v2[r] = V[3 * r + ord[1]]; v3[r] = V[3 * r + ord[2]];
  }
  u3[0] = dsub(dmul(u1[1], u2[2]), dmul(u1[2], u2[1]));
  u3[1] = dsub(dmul(u1[2], u2[0]), dmul(u1[0], u2[2]));
  u3[2] = dsub(dmul(u1[0], u2[1]), dmul(u1[1], u2[0]));
  const double detv = dadd(dsub(dmul(v1[0], dsub(dmul(v2[1], v3[2]), dmul(v2[2], v3[1]))),
                                dmul(v1[1], dsub(dmul(v2[0], v3[2]), dmul(v2[2], v3[0])))),
                           dmul(v1[2], dsub(dmul(v2[0], v3[1]), dmul(v2[1], v3[0]))));
  const double sg = detv < 0.0 ? -1.0 : 1.0;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b)
      s->R[3 * a + b] = dadd(dadd(dmul(u1[a], v1[b]), dmul(u2[a], v2[b])), dmul(dmul(sg, u3[a]), v3[b]));
  const double d3s = dmul(sg, dadd(dadd(dmul(b3[0], u3[0]), dmul(b3[1], u3[1])), dmul(b3[2], u3[2])));
  const double c = dmul(ddiv(1.0, sx2), dadd(dadd(s1, s2), d3s));   // evo: 1 / sigma_x * trace(D S)
  s->c = c;
  for (int a = 0; a < 3; ++a) {
    const double rm = dadd(dadd(dmul(s->R[3 * a], s->mx[0]), dmul(s->R[3 * a + 1], s->mx[1])), dmul(s->R[3 * a + 2], s->mx[2]));
    s->t[a] = dsub(s->my[a], dmul(c, rm));
  }
}

// e_i = |(R (c x_i) + t) - y_i| into errors and keys (keys padded with +inf to n); partials of sum e, sum e^2
__global__ void __launch_bounds__(kThreads) ape_error_kernel(const double* xs, const double* ys, long long n,
                                                             const ApeState* s, double* errors, double* keys,
                                                             double* part) {
  __shared__ double sh[2][kThreads];
  if (s->status != GOSLAM_APE_OK) return;
  const long long m = s->m;
  const double c = s->c;
  double R[9], t[3];
  for (int k = 0; k < 9; ++k) R[k] = s->R[k];
  for (int k = 0; k < 3; ++k) t[k] = s->t[k];
  double v[2] = {0, 0};
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
    if (i >= m) { keys[i] = INFINITY; continue; }
    double p[3], d[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) p[j] = dmul(c, xs[3 * i + j]);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double q = dadd(dadd(dadd(dmul(R[3 * a], p[0]), dmul(R[3 * a + 1], p[1])), dmul(R[3 * a + 2], p[2])), t[a]);
      d[a] = dsub(q, ys[3 * i + a]);
    }
    const double e2 = dadd(dadd(dmul(d[0], d[0]), dmul(d[1], d[1])), dmul(d[2], d[2]));
    const double e = __dsqrt_rn(e2);
    errors[i] = e;
    keys[i] = e;
    v[0] = dadd(v[0], e);
    v[1] = dadd(v[1], dmul(e, e));
  }
  write_partials(v, sh, part);
}

// one block: mean = sum e / n and sse = sum e^2
__global__ void __launch_bounds__(kThreads) ape_moment_kernel(const double* part, int nb, ApeState* s) {
  __shared__ double sh[2][kThreads];
  if (s->status != GOSLAM_APE_OK) return;
  double v[2];
  sum_partials(part, nb, v, sh);
  if (threadIdx.x != 0) return;
  s->mean = ddiv(v[0], (double)s->m);
  s->sse = v[1];
}

// partials of sum (e - mean)^2
__global__ void __launch_bounds__(kThreads) ape_spread_kernel(const double* errors, const ApeState* s, double* part) {
  __shared__ double sh[1][kThreads];
  if (s->status != GOSLAM_APE_OK) return;
  const long long m = s->m;
  const double mean = s->mean;
  double v[1] = {0};
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < m; i += (long long)gridDim.x * kThreads) {
    const double d = dsub(errors[i], mean);
    v[0] = dadd(v[0], dmul(d, d));
  }
  write_partials(v, sh, part);
}

// one block: std, the order statistics and the result record (NaN where the status leaves a value undefined)
__global__ void __launch_bounds__(kThreads) ape_result_kernel(const double* part, int nb, const double* sorted,
                                                              const ApeState* s, double* out) {
  __shared__ double sh[1][kThreads];
  const int status = s->status;
  double v[1] = {0};
  if (status == GOSLAM_APE_OK) sum_partials(part, nb, v, sh);
  if (threadIdx.x != 0) return;
  const int m = s->m;
  const double nan_ = nan("");
  out[GOSLAM_APE_STATUS] = (double)status;
  out[GOSLAM_APE_KEPT] = (double)m;
  for (int k = 0; k < 3; ++k) out[GOSLAM_APE_SINGULAR + k] = s->sv[k];
  if (status != GOSLAM_APE_OK) {
    for (int k = 0; k < 16; ++k) out[GOSLAM_APE_SIM3 + k] = nan_;
    for (int k = 0; k < 7; ++k) out[GOSLAM_APE_STATS + k] = nan_;
    return;
  }
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) out[GOSLAM_APE_SIM3 + 4 * a + b] = dmul(s->c, s->R[3 * a + b]);
    out[GOSLAM_APE_SIM3 + 4 * a + 3] = s->t[a];
  }
  for (int b = 0; b < 4; ++b) out[GOSLAM_APE_SIM3 + 12 + b] = b == 3 ? 1.0 : 0.0;
  const double lo = sorted[(m - 1) / 2], hi = sorted[m / 2];
  double* st = out + GOSLAM_APE_STATS;
  st[0] = __dsqrt_rn(ddiv(s->sse, (double)m));                      // rmse
  st[1] = s->mean;                                                  // mean
  st[2] = (m & 1) ? lo : ddiv(dadd(lo, hi), 2.0);                   // median (numpy's)
  st[3] = __dsqrt_rn(ddiv(v[0], (double)m));                        // std (population)
  st[4] = sorted[0];                                                // min
  st[5] = sorted[m - 1];                                            // max
  st[6] = s->sse;                                                   // sse
}

}  // namespace

extern "C" {

size_t goslam_ape_workspace_bytes(int64_t n) {
  if (n < 0 || n > kMaxRows) return 0;
  ApeWork w;
  return ape_layout(n, nullptr, &w);
}

int goslam_ape_sim3(const double* est, const double* ref, int64_t n, void* workspace, size_t workspace_bytes,
                    double* out, double* errors, void* stream) {
  if (n < 0 || n > kMaxRows || !out || (n > 0 && (!est || !ref || !errors))) return GOSLAM_EINVAL;
  ApeWork w;
  if (!workspace || workspace_bytes < ape_layout(n, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = partial_blocks(n);
  ape_init_kernel<<<1, 32, 0, st>>>(w.state);
  GS_CHECK_LAUNCH();
  if (n > 0) {
    ape_keep_kernel<<<blocks_for(n), kThreads, 0, st>>>(ref, n, w.flag);
    GS_CHECK_LAUNCH();
    size_t tb = w.cub_bytes;
    GS_CUDA(cub::DeviceSelect::Flagged(w.cub_tmp, tb, cub::CountingInputIterator<int>(0), w.flag, w.kept, &w.state->m,
                                       (int)n, st));
    ape_gather_kernel<<<nb, kThreads, 0, st>>>(est, ref, w.kept, w.state, w.xs, w.ys, w.part);
    GS_CHECK_LAUNCH();
    ape_mean_kernel<<<1, kThreads, 0, st>>>(w.part, nb, w.state);
    GS_CHECK_LAUNCH();
    ape_cov_kernel<<<nb, kThreads, 0, st>>>(w.xs, w.ys, w.state, w.part);
    GS_CHECK_LAUNCH();
    ape_solve_kernel<<<1, kThreads, 0, st>>>(w.part, nb, w.state);
    GS_CHECK_LAUNCH();
    ape_error_kernel<<<nb, kThreads, 0, st>>>(w.xs, w.ys, n, w.state, errors, w.keys, w.part);
    GS_CHECK_LAUNCH();
    ape_moment_kernel<<<1, kThreads, 0, st>>>(w.part, nb, w.state);
    GS_CHECK_LAUNCH();
    ape_spread_kernel<<<nb, kThreads, 0, st>>>(errors, w.state, w.part);
    GS_CHECK_LAUNCH();
    tb = w.cub_bytes;
    GS_CUDA(cub::DeviceRadixSort::SortKeys(w.cub_tmp, tb, w.keys, w.sorted, (int)n, 0, 64, st));
  }
  ape_result_kernel<<<1, kThreads, 0, st>>>(w.part, nb, w.sorted, w.state, out);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
