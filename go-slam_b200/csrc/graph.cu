// graph.cu — factor-graph edge selection on the device (SURVEY §8f-2).
//
// FactorGraph.add_proximity_factors (src/factor_graph.py:384-450) runs on every keyframe
// (src/frontend.py:58): after DepthVideo.distance it masks the distance matrix, suppresses around the
// edges the graph already has, lays down the local-window edges and then does a greedy non-maximum
// suppression over the remaining candidates in ascending distance — in Python, with one
// device->host sync (.item()) per candidate.  Here the whole selection is one launch of one block:
// parallel masking / suppression / local edges, a bitonic sort of the candidates by (distance, index),
// and a single warp walking the sorted list (the greedy order is inherently serial; the warp
// parallelises each suppression box).  Output = the reference's edge list, same order.
// Python index semantics the reference relies on are reproduced: a negative column index wraps,
// slice stops clamp.  Equal distances are ordered by index (a stable sort; the reference's
// torch.sort leaves that order unspecified).
#include "common.cuh"

namespace {

constexpr int kGT = 1024;

__device__ __forceinline__ unsigned g_f2ord(float f) {      // order-preserving, NaN above +inf
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

struct ProxArgs {
  const float* dist; const int64_t* ii_old; const int64_t* jj_old; int n_old;
  int t0, t1, t, rad, nms, max_factors, stereo, jfloor, loop;
  float thresh, dmax;
  float* dm;                    // [ilen*jlen] working copy
  unsigned long long* keys;     // [pow2 >= candidates]
  int* counters;                // [0] candidates, [1] edges written
  int64_t* es_i; int64_t* es_j; int cap;
  int nkeys_cap;
};

// d[max(0,di-nms):min(ilen,di+nms+1), max(0,dj-nms):min(jlen,dj+nms+1)] = inf with Python slice rules
__device__ __forceinline__ void box_bounds(int di, int dj, int nms, int ilen, int jlen, int& r0, int& r1,
                                           int& c0, int& c1) {
  r0 = max(0, di - nms); r1 = min(ilen, di + nms + 1);
  c0 = max(0, dj - nms); c1 = min(jlen, dj + nms + 1);
  if (r1 < 0) r1 = max(0, r1 + ilen);
  if (c1 < 0) c1 = max(0, c1 + jlen);
}

__global__ void __launch_bounds__(kGT) proximity_kernel(const ProxArgs a) {
  const int tid = threadIdx.x;
  const int ilen = a.t - a.t0, jlen = a.t - a.t1, n = ilen * jlen;
  const float inf = __int_as_float(0x7f800000);
  // ---- A: masked copy (:398-400) ----
  for (int k = tid; k < n; k += kGT) {
    float v = a.dist[k];
    const int i = a.t0 + k / jlen, j = a.t1 + k % jlen;
    if (i - a.rad < j) v = inf;
    if (v > a.dmax) v = inf;
    a.dm[k] = v;
  }
  if (tid == 0) { a.counters[0] = 0; a.counters[1] = 0; }
  __syncthreads();
  // ---- B: suppress around the edges the graph already has (:403-410); all writes are +inf: order-free ----
  for (int e = tid; e < a.n_old; e += kGT) {
    const int i = (int)a.ii_old[e], j = (int)a.jj_old[e];
    if (i >= a.t0 && i < a.t && j >= a.t1 && j < a.t) {
      const int di = i - a.t0, dj = j - a.t1;
      int r0, r1, c0, c1;
      box_bounds(di, dj, a.nms, ilen, jlen, r0, r1, c0, c1);
      a.dm[di * jlen + dj] = inf;
      for (int r = r0; r < r1; ++r)
        for (int c = c0; c < c1; ++c) a.dm[r * jlen + c] = inf;
    }
  }
  // ---- C: local-window edges (:412-425); their positions in `es` are known in closed form ----
  for (int i = a.t0 + tid; i < a.t; i += kGT) {
    int off = 0;
    for (int q = a.t0; q < i; ++q) off += (a.stereo ? 1 : 0) + 2 * (q - min(q, max(q - a.rad, a.jfloor)));
    const int di = i - a.t0;
    if (a.stereo) {
      if (off < a.cap) { a.es_i[off] = i; a.es_j[off] = i; }
      ++off;
      int dj = i - a.t1;
      if (dj < 0) dj += jlen;
      a.dm[di * jlen + dj] = inf;
    }
    for (int j = max(i - a.rad, a.jfloor); j < i; ++j) {
      if (off + 1 < a.cap) { a.es_i[off] = i; a.es_j[off] = j; a.es_i[off + 1] = j; a.es_j[off + 1] = i; }
      off += 2;
      const int dj = j - a.t1;
      a.dm[di * jlen + (dj < 0 ? dj + jlen : dj)] = inf;
      int r0, r1, c0, c1;
      box_bounds(di, dj, a.nms, ilen, jlen, r0, r1, c0, c1);
      for (int r = r0; r < r1; ++r)
        for (int c = c0; c < c1; ++c) a.dm[r * jlen + c] = inf;
    }
    if (i == a.t - 1) a.counters[1] = off;
  }
  __threadfence_block();
  __syncthreads();
  // ---- D: candidates d <= thresh -> (distance, index) keys (:428-430) ----
  for (int k = tid; k < n; k += kGT) {
    const float v = a.dm[k];
    if (v <= a.thresh) {
      const int slot = atomicAdd(&a.counters[0], 1);
      if (slot < a.nkeys_cap) a.keys[slot] = ((unsigned long long)g_f2ord(v) << 32) | (unsigned)k;
    }
  }
  __syncthreads();
  const int C = min(a.counters[0], a.nkeys_cap);
  int P2 = 1;
  while (P2 < C) P2 <<= 1;
  for (int k = C + tid; k < P2; k += kGT) a.keys[k] = ~0ull;
  __syncthreads();
  // ---- E: bitonic sort, ascending ----
  for (int size = 2; size <= P2; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = tid; t < (P2 >> 1); t += kGT) {
        const int lo = (t / stride) * (stride << 1) + (t % stride), hi = lo + stride;
        const bool asc = ((lo & size) == 0);
        const unsigned long long x = a.keys[lo], y = a.keys[hi];
        if ((x > y) == asc) { a.keys[lo] = y; a.keys[hi] = x; }
      }
      __syncthreads();
    }
  // ---- F: greedy non-maximum suppression in ascending distance (:432-447), one warp ----
  if (tid < 32) {
    int n_es = a.counters[1];
    volatile float* dmv = a.dm;
    for (int c = 0; c < C; ++c) {
      const int k = (int)(a.keys[c] & 0xffffffffull);
      const int di = k / jlen, dj = k % jlen;
      if (dmv[k] > a.thresh) continue;                  // suppressed meanwhile
      if (n_es > a.max_factors) break;
      if (a.loop) {
        // loop-closure candidates (src/backend.py:81-91): the 3x3 neighbourhood of (i, j) votes with the RAW
        // distances; if more than half of the 9 cells are below the threshold, every such cell off the
        // diagonal becomes an edge, in row-major (si, sj) order
        const int i = a.t0 + di, j = a.t1 + dj;
        const int si = i - 1 + tid / 3, sj = j - 1 + tid % 3;
        const bool in_rng = tid < 9 && si >= max(i - 1, a.t0) && si < min(i + 2, a.t) &&
                            sj >= max(j - 1, a.t1) && sj < min(j + 2, a.t);
        const bool vote = in_rng && a.dist[(si - a.t0) * jlen + (sj - a.t1)] <= a.thresh;
        const unsigned votes = __ballot_sync(0xffffffffu, vote);
        if (__popc(votes) > 4) {                       // int(9 * 0.5) = 4
          const bool take = vote && si != sj;
          const unsigned takes = __ballot_sync(0xffffffffu, take);
          const int pos = n_es + __popc(takes & ((1u << tid) - 1u));
          if (take && pos < a.cap) { a.es_i[pos] = si; a.es_j[pos] = sj; }
          n_es += __popc(takes);
        }
      } else {
        if (tid == 0 && n_es + 1 < a.cap) {
          const int i = a.t0 + di, j = a.t1 + dj;
          a.es_i[n_es] = i; a.es_j[n_es] = j; a.es_i[n_es + 1] = j; a.es_j[n_es + 1] = i;
        }
        n_es += 2;
      }
      int r0, r1, c0, c1;
      box_bounds(di, dj, a.nms, ilen, jlen, r0, r1, c0, c1);
      const int bw = c1 - c0, cells = (r1 - r0) * bw;
      for (int q = tid; q < cells; q += 32) dmv[(r0 + q / bw) * jlen + c0 + q % bw] = inf;
      __threadfence_block();
      __syncwarp();
    }
    if (tid == 0) a.counters[1] = n_es;
  }
}

// the distance matrix of the window, its candidate keys (a power of two of them, for the sort) and two counters
size_t prox_layout(int t0, int t1, int t, void* base, ProxArgs* a) {
  GsArena ar(base);
  const size_t n = (size_t)(t - t0) * (t - t1);
  size_t p2 = 1;
  while (p2 < n) p2 <<= 1;
  a->dm = ar.take<float>(n);
  a->keys = ar.take<unsigned long long>(p2);
  a->counters = ar.take<int>(2);
  a->nkeys_cap = (int)p2;
  return ar.off;
}

}  // namespace

extern "C" {

size_t goslam_proximity_workspace_bytes(int t0, int t1, int t) {
  if (t <= t0 || t <= t1 || t0 < 0 || t1 < 0) return 0;
  ProxArgs a;
  return prox_layout(t0, t1, t, nullptr, &a);
}

int goslam_proximity_edges(const float* dist, int t0, int t1, int t, int rad, int nms, float thresh,
                           float dmax, int jfloor, int loop, int max_factors, int stereo,
                           const int64_t* ii_old, const int64_t* jj_old,
                           int n_old, int64_t* es_i, int64_t* es_j, int cap, int* num_edges,
                           void* workspace, size_t workspace_bytes, void* stream) {
  if (t <= t0 || t <= t1 || t0 < 0 || t1 < 0 || rad < 0 || nms < 0 || n_old < 0 || cap < 0 || jfloor < 0)
    return GOSLAM_EINVAL;
  const int ilen = t - t0, jlen = t - t1;
  if ((long long)ilen * jlen > (1 << 24)) return GOSLAM_EINVAL;
  // the reference would raise IndexError for a column index below -jlen (src/factor_graph.py:423)
  const int jmin = (t0 - rad > jfloor ? t0 - rad : jfloor);
  if (rad > 0 && jmin - t1 < -jlen) return GOSLAM_EINVAL;
  if (stereo && t0 - t1 < -jlen) return GOSLAM_EINVAL;
  ProxArgs a{};
  if (!workspace || workspace_bytes < prox_layout(t0, t1, t, workspace, &a)) return GOSLAM_EWORKSPACE;
  a.dist = dist; a.ii_old = ii_old; a.jj_old = jj_old; a.n_old = n_old;
  a.t0 = t0; a.t1 = t1; a.t = t; a.rad = rad; a.nms = nms; a.max_factors = max_factors; a.stereo = stereo ? 1 : 0;
  a.thresh = thresh; a.dmax = dmax; a.jfloor = jfloor; a.loop = loop ? 1 : 0;
  a.es_i = es_i; a.es_j = es_j; a.cap = cap;
  proximity_kernel<<<1, kGT, 0, (cudaStream_t)stream>>>(a);
  GS_CHECK_LAUNCH();
  if (num_edges)
    GS_CUDA(cudaMemcpyAsync(num_edges, a.counters + 1, sizeof(int), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return GOSLAM_OK;
}

}  // extern "C"
