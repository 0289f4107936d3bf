// mesh.cu — marching cubes and the bound cull of InstantNeuS.extract_geometry (src/InstantNeuS.py:458-492).
//
// The reference hands the [res]^3 field to PyMCubes on one CPU core and culls with trimesh.  Here both run on the
// device in two calls each (count, then emit), so that the caller can size the outputs between them; the library
// allocates nothing and never synchronises.  The tables are generated (tools/gen_mc_tables.py -> mc_tables.cuh).
//
// Orders and scratch:
//   * one vertex per lattice edge whose ends are classified differently (inside iff u > iso, compared in fp64);
//     vertex order = ascending edge id 3 * linear(a) + axis (x-major).  The count pass stores the crossing bits as
//     a bitmask over edge ids plus an exclusive prefix count per 32-bit word (12 bytes per 32 edges, 1.125 bytes per
//     lattice point); a vertex's index is the word's prefix plus the popcount of the lower bits.
//   * faces are ordered by cell (x-major, z fastest), then by table order.  Cells go to blocks of kCellsPerBlock;
//     the count pass stores one triangle count per block, the emit pass recomputes every cell's case from u and
//     places its triangles by a block scan.  No per-cell state is stored.
//   * every order comes from scans (three-kernel tile scans below), never from atomics: outputs are deterministic.
//   * ids, counts and offsets are 64-bit: the edge ids of a 1024^3 lattice pass 2^31.
#include "common.cuh"
#include "mc_tables.cuh"

namespace {

typedef unsigned long long u64;

constexpr int kScanThreads = 256, kScanItems = 16, kScanTile = kScanThreads * kScanItems;
constexpr int kTopThreads = 1024;
constexpr int kCellThreads = 256, kCellItems = 4, kCellsPerBlock = kCellThreads * kCellItems;

long long cdiv64(long long a, long long b) { return (a + b - 1) / b; }

// exclusive scan of one value per thread over the block; *total = the block's sum.  Every thread must call it.
template <int NT>
__device__ __forceinline__ u64 block_exclusive_scan(u64 v, u64* total) {
  __shared__ u64 warp_tot[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u64 inc = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const u64 n = __shfl_up_sync(0xffffffffu, inc, off);
    if (lane >= off) inc += n;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    u64 w = lane < NT / 32 ? warp_tot[lane] : 0ull;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const u64 n = __shfl_up_sync(0xffffffffu, w, off);
      if (lane >= off) w += n;
    }
    warp_tot[lane] = w;
  }
  __syncthreads();
  const u64 excl = (warp ? warp_tot[warp - 1] : 0ull) + inc - v;
  *total = warp_tot[NT / 32 - 1];
  __syncthreads();                       // warp_tot is reused by the next call
  return excl;
}

struct PopcLoad {
  const unsigned* w;
  __device__ unsigned operator()(long long i) const { return __popc(w[i]); }
};
struct U32Load {
  const unsigned* p;
  __device__ unsigned operator()(long long i) const { return p[i]; }
};

// ---- exclusive scan of n loader values into u64 offsets: tile sums, one-block scan of the tile sums, apply ----
template <class L>
__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(L ld, long long n, u64* tile_sum) {
  const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
  u64 s = 0;
#pragma unroll
  for (int j = 0; j < kScanItems; ++j)
    if (base + j < n) s += ld(base + j);
  u64 tot;
  block_exclusive_scan<kScanThreads>(s, &tot);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kTopThreads) scan_top_kernel(u64* tile, long long ntiles, long long* total) {
  u64 carry = 0;
  for (long long b = 0; b < ntiles; b += kTopThreads) {
    const long long i = b + threadIdx.x;
    const u64 v = i < ntiles ? tile[i] : 0ull;
    u64 tot;
    const u64 ex = block_exclusive_scan<kTopThreads>(v, &tot);
    if (i < ntiles) tile[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0 && total) *total = (long long)carry;
}

template <class L>
__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(L ld, long long n, const u64* tile_off, u64* out) {
  const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
  unsigned v[kScanItems];
  u64 s = 0;
#pragma unroll
  for (int j = 0; j < kScanItems; ++j) {
    v[j] = base + j < n ? ld(base + j) : 0u;
    s += v[j];
  }
  u64 tot;
  u64 run = tile_off[blockIdx.x] + block_exclusive_scan<kScanThreads>(s, &tot);
#pragma unroll
  for (int j = 0; j < kScanItems; ++j)
    if (base + j < n) { out[base + j] = run; run += v[j]; }
}

template <class L>
int exclusive_scan(L ld, long long n, u64* out, u64* tiles, long long* total, cudaStream_t st) {
  const long long nt = cdiv64(n, kScanTile);
  if (nt > 0) {
    scan_reduce_kernel<L><<<(unsigned)nt, kScanThreads, 0, st>>>(ld, n, tiles);
    GS_CHECK_LAUNCH();
  }
  scan_top_kernel<<<1, kTopThreads, 0, st>>>(tiles, nt, total);
  GS_CHECK_LAUNCH();
  if (nt > 0) {
    scan_apply_kernel<L><<<(unsigned)nt, kScanThreads, 0, st>>>(ld, n, tiles, out);
    GS_CHECK_LAUNCH();
  }
  return GOSLAM_OK;
}

// ---- marching cubes -------------------------------------------------------------------------------------------
struct Lattice {
  const float* u;
  int nx, ny, nz;
  double iso;
  long long npts, ncell;
  long long nyz, cyz;                   // points per x plane, cells per x plane
  double inv_nyz, inv_nz, inv_cyz, inv_cz;  // reciprocals for gs_div_fast
};

Lattice make_lattice(const float* u, int nx, int ny, int nz, double iso) {
  Lattice g;
  g.u = u; g.nx = nx; g.ny = ny; g.nz = nz; g.iso = iso;
  g.npts = (long long)nx * ny * nz;
  g.ncell = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  g.nyz = (long long)ny * nz;
  g.cyz = (long long)(ny - 1) * (nz - 1);
  g.inv_nyz = 1.0 / (double)g.nyz;
  g.inv_nz = 1.0 / (double)nz;
  g.inv_cyz = 1.0 / (double)(g.cyz > 0 ? g.cyz : 1);
  g.inv_cz = 1.0 / (double)(nz > 1 ? nz - 1 : 1);
  return g;
}

struct McWork {
  unsigned* words;   // crossing bit of edge id e at words[e >> 5] bit (e & 31)
  u64* word_off;     // exclusive prefix popcount per word
  unsigned* cb_cnt;  // triangles per cell block
  u64* cb_off;       // their exclusive prefix
  u64* tiles;        // scan scratch
  long long nwords, ncb;
};

// one layout for the count and the emit pass; returns the bytes it needs
size_t mc_layout(const Lattice& g, const void* base, McWork* w) {
  GsArena ar(base);
  w->nwords = 3 * cdiv64(g.npts, 32);
  w->ncb = cdiv64(g.ncell, kCellsPerBlock);
  w->words = ar.take<unsigned>(w->nwords);
  w->word_off = ar.take<u64>(w->nwords);
  w->cb_cnt = ar.take<unsigned>(w->ncb);
  w->cb_off = ar.take<u64>(w->ncb);
  const long long nt = cdiv64(w->nwords > w->ncb ? w->nwords : w->ncb, kScanTile);
  w->tiles = ar.take<u64>(nt > 0 ? nt : 1);
  return ar.off;
}

__device__ __forceinline__ bool inside(const Lattice& g, long long i) { return (double)g.u[i] > g.iso; }

// lattice coordinates of point L
__device__ __forceinline__ void point_xyz(const Lattice& g, long long L, int* x, int* y, int* z) {
  const long long xi = gs_div_fast(L, g.nyz, g.inv_nyz);
  const long long r = L - xi * g.nyz;
  const long long yi = gs_div_fast(r, g.nz, g.inv_nz);
  *x = (int)xi; *y = (int)yi; *z = (int)(r - yi * g.nz);
}

// crossing bits of the three lattice edges that start at each point, packed by warp ballots: a warp owns 32 points
// = 96 edge ids = 3 whole words
__global__ void __launch_bounds__(256) mc_edge_kernel(const Lattice g, unsigned* words) {
  const long long L = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  if ((L & ~31ll) >= g.npts) return;                  // whole warps past the lattice own no word
  unsigned v = 0;
  if (L < g.npts) {
    int x, y, z;
    point_xyz(g, L, &x, &y, &z);
    const bool a = inside(g, L);
    if (x + 1 < g.nx && a != inside(g, L + g.nyz)) v |= 1u;
    if (y + 1 < g.ny && a != inside(g, L + g.nz)) v |= 2u;
    if (z + 1 < g.nz && a != inside(g, L + 1)) v |= 4u;
  }
  const long long w0 = (L >> 5) * 3;
#pragma unroll
  for (int w = 0; w < 3; ++w) {
    const int e = 32 * w + lane;
    const unsigned b = (__shfl_sync(0xffffffffu, v, e / 3) >> (e % 3)) & 1u;
    const unsigned word = __ballot_sync(0xffffffffu, b);
    if (lane == w) words[w0 + w] = word;
  }
}

// case index of cell c and the linear index of its corner 0
__device__ __forceinline__ int cell_case(const Lattice& g, long long c, long long* origin) {
  const long long cx = gs_div_fast(c, g.cyz, g.inv_cyz), r = c - cx * g.cyz;
  const long long cy = gs_div_fast(r, g.nz - 1, g.inv_cz), cz = r - cy * (g.nz - 1);
  const long long L = (cx * g.ny + cy) * g.nz + cz, nyz = g.nyz;
  int cs = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    cs |= inside(g, L + (k & 1) * nyz + ((k >> 1) & 1) * g.nz + ((k >> 2) & 1)) << k;
  *origin = L;
  return cs;
}

__global__ void __launch_bounds__(kCellThreads) mc_cell_count_kernel(const Lattice g, unsigned* cb_cnt) {
  unsigned s = 0;
#pragma unroll
  for (int k = 0; k < kCellItems; ++k) {
    const long long c = (long long)blockIdx.x * kCellsPerBlock + k * kCellThreads + threadIdx.x;
    if (c < g.ncell) {
      long long L;
      s += c_mc_ntri[cell_case(g, c, &L)];
    }
  }
  u64 tot;
  block_exclusive_scan<kCellThreads>(s, &tot);
  if (threadIdx.x == 0) cb_cnt[blockIdx.x] = (unsigned)tot;
}

__device__ __forceinline__ u64 vertex_index(const unsigned* words, const u64* word_off, long long id) {
  const unsigned w = words[id >> 5];
  return word_off[id >> 5] + __popc(w & ((1u << (id & 31)) - 1u));
}

__global__ void __launch_bounds__(kCellThreads) mc_face_kernel(const Lattice g, const unsigned* words, const u64* word_off,
                                                               const u64* cb_off, long long* faces, long long max_faces) {
  const long long nyz = (long long)g.ny * g.nz;
  u64 run = cb_off[blockIdx.x];
  for (int k = 0; k < kCellItems; ++k) {
    const long long c = (long long)blockIdx.x * kCellsPerBlock + k * kCellThreads + threadIdx.x;
    int cs = 0, nt = 0;
    long long L = 0;
    if (c < g.ncell) {
      cs = cell_case(g, c, &L);
      nt = c_mc_ntri[cs];
    }
    u64 tot;
    const u64 off = run + block_exclusive_scan<kCellThreads>((u64)nt, &tot);
    run += tot;
    for (int t = 0; t < nt; ++t) {
      if ((long long)(off + t) >= max_faces) break;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int e = c_mc_tris[cs][3 * t + j];
        // start corner of edge e: 0 along its axis a, bits (e & 1, e >> 1 & 1) along the other two axes
        const int a = e >> 2, b0 = e & 1, b1 = (e >> 1) & 1;
        const int dx = a == 0 ? 0 : b0;
        const int dy = a == 0 ? b0 : (a == 1 ? 0 : b1);
        const int dz = a == 2 ? 0 : b1;
        const long long id = 3 * (L + dx * nyz + dy * g.nz + dz) + a;
        faces[(off + t) * 3 + j] = (long long)vertex_index(words, word_off, id);
      }
    }
  }
}

struct WorldMap {
  double den[3];     // resolution - 1.0 per axis
  double range[3];   // (double)(float)(bmax - bmin)
  double bmin[3];
};

// vertex position: a with a_axis + t, t = (iso - ua) / (ub - ua) in fp64, then v / (res - 1.0) * range + bmin
// operation by operation (no contraction), as numpy evaluates it
__global__ void __launch_bounds__(256) mc_vertex_kernel(const Lattice g, const unsigned* words, const u64* word_off,
                                                        const WorldMap m, double* verts, long long max_verts) {
  const long long L = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (L >= g.npts) return;
  int x, y, z;
  point_xyz(g, L, &x, &y, &z);
  const long long stride[3] = {g.nyz, (long long)g.nz, 1};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const long long id = 3 * L + a;
    if (!((words[id >> 5] >> (id & 31)) & 1u)) continue;
    const u64 vi = vertex_index(words, word_off, id);
    if ((long long)vi >= max_verts) continue;
    const double ua = (double)g.u[L], ub = (double)g.u[L + stride[a]];
    const double t = __ddiv_rn(__dsub_rn(g.iso, ua), __dsub_rn(ub, ua));
    double p[3] = {(double)x, (double)y, (double)z};
    p[a] = __dadd_rn(p[a], t);
#pragma unroll
    for (int c = 0; c < 3; ++c)
      verts[vi * 3 + c] = __dadd_rn(__dmul_rn(__ddiv_rn(p[c], m.den[c]), m.range[c]), m.bmin[c]);
  }
}

// ---- bound cull -----------------------------------------------------------------------------------------------
struct CullWork {
  unsigned* vref;   // vertex referenced by a kept face
  u64* voff;        // new vertex index
  unsigned* fkeep;  // face kept
  u64* foff;        // new face index
  u64* tiles;
};

size_t cull_layout(long long nv, long long nf, const void* base, CullWork* w) {
  GsArena ar(base);
  w->vref = ar.take<unsigned>(nv > 0 ? nv : 1);
  w->voff = ar.take<u64>(nv > 0 ? nv : 1);
  w->fkeep = ar.take<unsigned>(nf > 0 ? nf : 1);
  w->foff = ar.take<u64>(nf > 0 ? nf : 1);
  const long long nt = cdiv64(nv > nf ? nv : nf, kScanTile);
  w->tiles = ar.take<u64>(nt > 0 ? nt : 1);
  return ar.off;
}

struct CullBox { double lo[3], hi[3]; };

__global__ void __launch_bounds__(256) cull_face_kernel(const double* verts, long long nv, const long long* faces, long long nf,
                                                        const CullBox b, unsigned* fkeep, unsigned* vref) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  long long v[3];
  bool keep = true;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    v[j] = faces[f * 3 + j];
    if (v[j] < 0 || v[j] >= nv) { keep = false; continue; }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double x = verts[v[j] * 3 + c];
      keep = keep && x >= b.lo[c] && x <= b.hi[c];
    }
  }
  fkeep[f] = keep ? 1u : 0u;
  if (keep) {
#pragma unroll
    for (int j = 0; j < 3; ++j) vref[v[j]] = 1u;     // every writer stores the same value
  }
}

// a face is kept iff face_mask[f] (when given) and vert_mask of its three vertices (when given): trimesh's
// update_faces(mask[faces].all(1)) of src/mesher.py:198,213,228
__global__ void __launch_bounds__(256) cull_mask_face_kernel(long long nv, const long long* faces, long long nf,
                                                             const unsigned char* face_mask, const unsigned char* vert_mask,
                                                             unsigned* fkeep, unsigned* vref) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  long long v[3];
  bool keep = !face_mask || face_mask[f];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    v[j] = faces[f * 3 + j];
    if (v[j] < 0 || v[j] >= nv) { keep = false; continue; }
    if (vert_mask && !vert_mask[v[j]]) keep = false;
  }
  fkeep[f] = keep ? 1u : 0u;
  if (keep) {
#pragma unroll
    for (int j = 0; j < 3; ++j) vref[v[j]] = 1u;
  }
}

__global__ void __launch_bounds__(256) cull_vertex_ids_kernel(long long nv, const unsigned* vref, const u64* voff, long long* ids,
                                                              long long max_ids) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv || !vref[i] || (long long)voff[i] >= max_ids) return;
  ids[voff[i]] = i;
}

__global__ void __launch_bounds__(256) cull_vertex_emit_kernel(const double* verts, long long nv, const unsigned* vref,
                                                               const u64* voff, double* out, long long max_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv || !vref[i] || (long long)voff[i] >= max_out) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) out[voff[i] * 3 + c] = verts[i * 3 + c];
}

__global__ void __launch_bounds__(256) cull_face_emit_kernel(const long long* faces, long long nf, const unsigned* fkeep,
                                                             const u64* foff, const u64* voff, long long* out, long long max_out) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf || !fkeep[f] || (long long)foff[f] >= max_out) return;
#pragma unroll
  for (int j = 0; j < 3; ++j) out[foff[f] * 3 + j] = (long long)voff[faces[f * 3 + j]];
}

bool lattice_ok(const void* u, int nx, int ny, int nz) {
  // 2^40 points: far beyond any device's memory, keeps every id and launch size in range
  return u && nx >= 2 && ny >= 2 && nz >= 2 && (long long)nx * ny * nz <= (1ll << 40);
}

unsigned blocks_for(long long n, int threads) { return (unsigned)cdiv64(n, threads); }

}  // namespace

extern "C" {

size_t goslam_mc_workspace_bytes(int nx, int ny, int nz) {
  if (nx < 2 || ny < 2 || nz < 2 || (long long)nx * ny * nz > (1ll << 40)) return 0;
  McWork w;
  return mc_layout(make_lattice(nullptr, nx, ny, nz, 0.0), nullptr, &w);
}

int goslam_mc_count(const float* u, int nx, int ny, int nz, double iso, void* workspace, size_t workspace_bytes,
                    int64_t* counts, void* stream) {
  if (!lattice_ok(u, nx, ny, nz) || !counts || iso != iso) return GOSLAM_EINVAL;
  const Lattice g = make_lattice(u, nx, ny, nz, iso);
  McWork w;
  if (!workspace || workspace_bytes < mc_layout(g, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  mc_edge_kernel<<<blocks_for(cdiv64(g.npts, 32) * 32, 256), 256, 0, st>>>(g, w.words);
  GS_CHECK_LAUNCH();
  int rc = exclusive_scan(PopcLoad{w.words}, w.nwords, w.word_off, w.tiles, (long long*)counts, st);
  if (rc != GOSLAM_OK) return rc;
  mc_cell_count_kernel<<<(unsigned)w.ncb, kCellThreads, 0, st>>>(g, w.cb_cnt);
  GS_CHECK_LAUNCH();
  return exclusive_scan(U32Load{w.cb_cnt}, w.ncb, w.cb_off, w.tiles, (long long*)counts + 1, st);
}

int goslam_mc_emit(const float* u, int nx, int ny, int nz, double iso, const float* bound_min, const float* bound_max,
                   const void* workspace, size_t workspace_bytes, double* verts, int64_t max_verts, int64_t* faces,
                   int64_t max_faces, void* stream) {
  if (!lattice_ok(u, nx, ny, nz) || !bound_min || !bound_max || iso != iso || max_verts < 0 || max_faces < 0 ||
      (max_verts > 0 && !verts) || (max_faces > 0 && !faces))
    return GOSLAM_EINVAL;
  const Lattice g = make_lattice(u, nx, ny, nz, iso);
  McWork w;
  if (!workspace || workspace_bytes < mc_layout(g, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  WorldMap m;
  const int n[3] = {nx, ny, nz};
  for (int c = 0; c < 3; ++c) {
    m.den[c] = (double)n[c] - 1.0;
    const float range = bound_max[c] - bound_min[c];      // numpy subtracts the float32 arrays first
    m.range[c] = (double)range;
    m.bmin[c] = (double)bound_min[c];
  }
  if (max_verts > 0) {
    mc_vertex_kernel<<<blocks_for(g.npts, 256), 256, 0, st>>>(g, w.words, w.word_off, m, verts, max_verts);
    GS_CHECK_LAUNCH();
  }
  if (max_faces > 0) {
    mc_face_kernel<<<(unsigned)w.ncb, kCellThreads, 0, st>>>(g, w.words, w.word_off, w.cb_off, (long long*)faces, max_faces);
    GS_CHECK_LAUNCH();
  }
  return GOSLAM_OK;
}

size_t goslam_mesh_cull_workspace_bytes(int64_t n_verts, int64_t n_faces) {
  if (n_verts < 0 || n_faces < 0) return 0;
  CullWork w;
  return cull_layout(n_verts, n_faces, nullptr, &w);
}

int goslam_mesh_cull_count(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const float* lo,
                           const float* hi, void* workspace, size_t workspace_bytes, int64_t* counts, void* stream) {
  if (n_verts < 0 || n_faces < 0 || (n_verts > 0 && !verts) || (n_faces > 0 && !faces) || !lo || !hi || !counts)
    return GOSLAM_EINVAL;
  CullWork w;
  if (!workspace || workspace_bytes < cull_layout(n_verts, n_faces, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  CullBox b;
  for (int c = 0; c < 3; ++c) { b.lo[c] = (double)lo[c]; b.hi[c] = (double)hi[c]; }
  if (n_verts > 0) GS_CUDA(cudaMemsetAsync(w.vref, 0, (size_t)n_verts * sizeof(unsigned), st));
  if (n_faces > 0) {
    cull_face_kernel<<<blocks_for(n_faces, 256), 256, 0, st>>>(verts, n_verts, (const long long*)faces, n_faces, b, w.fkeep, w.vref);
    GS_CHECK_LAUNCH();
  }
  int rc = exclusive_scan(U32Load{w.vref}, n_verts, w.voff, w.tiles, (long long*)counts, st);
  if (rc != GOSLAM_OK) return rc;
  return exclusive_scan(U32Load{w.fkeep}, n_faces, w.foff, w.tiles, (long long*)counts + 1, st);
}

int goslam_mesh_cull_emit(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const void* workspace,
                          size_t workspace_bytes, double* out_verts, int64_t max_out_verts, int64_t* out_faces,
                          int64_t max_out_faces, void* stream) {
  if (n_verts < 0 || n_faces < 0 || max_out_verts < 0 || max_out_faces < 0 || (n_verts > 0 && !verts) ||
      (n_faces > 0 && !faces) || (max_out_verts > 0 && !out_verts) || (max_out_faces > 0 && !out_faces))
    return GOSLAM_EINVAL;
  CullWork w;
  if (!workspace || workspace_bytes < cull_layout(n_verts, n_faces, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_verts > 0 && max_out_verts > 0) {
    cull_vertex_emit_kernel<<<blocks_for(n_verts, 256), 256, 0, st>>>(verts, n_verts, w.vref, w.voff, out_verts, max_out_verts);
    GS_CHECK_LAUNCH();
  }
  if (n_faces > 0 && max_out_faces > 0) {
    cull_face_emit_kernel<<<blocks_for(n_faces, 256), 256, 0, st>>>((const long long*)faces, n_faces, w.fkeep, w.foff, w.voff,
                                                                    (long long*)out_faces, max_out_faces);
    GS_CHECK_LAUNCH();
  }
  return GOSLAM_OK;
}

int goslam_mesh_cull_mask_count(int64_t n_verts, const int64_t* faces, int64_t n_faces, const unsigned char* face_mask,
                                const unsigned char* vert_mask, void* workspace, size_t workspace_bytes, int64_t* counts,
                                void* stream) {
  if (n_verts < 0 || n_faces < 0 || (n_faces > 0 && !faces) || !counts) return GOSLAM_EINVAL;
  CullWork w;
  if (!workspace || workspace_bytes < cull_layout(n_verts, n_faces, workspace, &w)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_verts > 0) GS_CUDA(cudaMemsetAsync(w.vref, 0, (size_t)n_verts * sizeof(unsigned), st));
  if (n_faces > 0) {
    cull_mask_face_kernel<<<blocks_for(n_faces, 256), 256, 0, st>>>(n_verts, (const long long*)faces, n_faces, face_mask,
                                                                     vert_mask, w.fkeep, w.vref);
    GS_CHECK_LAUNCH();
  }
  int rc = exclusive_scan(U32Load{w.vref}, n_verts, w.voff, w.tiles, (long long*)counts, st);
  if (rc != GOSLAM_OK) return rc;
  return exclusive_scan(U32Load{w.fkeep}, n_faces, w.foff, w.tiles, (long long*)counts + 1, st);
}

int goslam_mesh_cull_vertex_ids(int64_t n_verts, int64_t n_faces, const void* workspace, size_t workspace_bytes, int64_t* ids,
                                int64_t max_ids, void* stream) {
  if (n_verts < 0 || n_faces < 0 || max_ids < 0 || (max_ids > 0 && !ids)) return GOSLAM_EINVAL;
  CullWork w;
  if (!workspace || workspace_bytes < cull_layout(n_verts, n_faces, workspace, &w)) return GOSLAM_EWORKSPACE;
  if (n_verts > 0 && max_ids > 0) {
    cull_vertex_ids_kernel<<<blocks_for(n_verts, 256), 256, 0, (cudaStream_t)stream>>>(n_verts, w.vref, w.voff,
                                                                                       (long long*)ids, max_ids);
    GS_CHECK_LAUNCH();
  }
  return GOSLAM_OK;
}

}  // extern "C"
