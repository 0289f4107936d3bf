// corr_build_tc.cu — all-pairs correlation volume on Hopper tensor cores (wgmma + TMA)
// with the 4-level average-pool pyramid produced in the epilogue.
//
// Reference: CorrBlock.__init__ / CorrBlock.corr (src/modules/corr.py:25-41,67-76) —
// torch.matmul (cuBLAS) writes level 0, then three F.avg_pool2d passes re-read the volume.
//
// Design (one CTA per SM, persistent, warp-specialised, 384 threads = 3 warpgroups):
//   warpgroup 2 TMA producer (one thread; the warpgroup drops to 40 registers with setmaxnreg):
//               A tile = 128 source pixels x 128 channels (2 boxes of 64 ch, 128B-swizzled, K-major) once
//               per work item (edge, source tile, 8-row target band); B tile = an 8x16 patch of TARGET
//               pixels x 128 channels (4-D tensor map (ch, x, y, slot) -> rows ordered y*16+x), 2-stage
//               ring.  Out-of-image rows/cols are zero-filled by TMA.  Feature maps are indexed per edge on
//               the device (slot1 = rig*ii, slot2 = rig*jj + (ii==jj)), so no gathered copies exist.
//               A is released as soon as the item's last MMAs retire, so the next item's A and B tiles
//               load under the current epilogue and band write-out.
//               Warps 9-11 of this warpgroup are the store warps.  Per band they pool level 3 from the
//               staged level 2 and write both with one TMA tensor store each, out of a double-buffered band
//               pool handed over by mbarriers ("staged": the 8 consumer warps, "freed": the store thread
//               after cp.async.bulk.wait_group.read).  The consumer warpgroups never join.
//   warpgroups 0-1  consumers (232 registers each: the 128 fp32 accumulators and the epilogue stay in
//               registers, no local memory); warpgroup g takes the x-tiles of parity g (B stage g), so
//               one warpgroup's MMAs overlap the other's epilogue.  A warpgroup issues 32 wgmma m64n64k16
//               (fp16 in, fp32 accumulate) for the whole 128x128 tile, then per m64 half rounds to fp16.
//               Level 0 goes into swizzled staging with stmatrix, level 1 is pooled in registers from the
//               rounded fragment and staged beside it; lane 0 of each warp writes its own 16 source pixels
//               of both with TMA tensor stores, level 0 as soon as it is staged (tiled_half_epilogue), so
//               the warps of a warpgroup never wait for each other; the consumers issue no global stores.
//               Every level is pooled FROM THE ROUNDED finer level (the avg_pool2d numerics); level 2 is
//               staged per band and leaves with level 3 through the store warps.  The volume is never re-read.
// Output layout (GOSLAM_LAYOUT_TILED): levels 0 and 1 as 4x4-element (32-byte) tiles, levels 2 and 3 as one
// padded piece per 8-row band, so every store is whole sectors for any h x w.
// Why the band staging: partial 32-byte-sector writes cost an ECC read-modify-write in L2.
// The 1/4 feature scaling of the reference (`fmap / 4.0` in half) is applied by the K-major
// re-layout prepass, exactly as the reference does it, so the accumulator needs no scaling.
#include "common.cuh"
#include "tc_ptx.cuh"
#include <cstdio>
#include <cuda.h>
#include <cstdlib>
#include <cstring>

namespace {

constexpr int kD = 128;                 // channels (K)
constexpr int kBM = 128;                // source pixels per tile
constexpr int kPY = 8, kPX = 16;        // target patch
constexpr int kKBox = 64;               // channels per TMA box (128 B)
constexpr int kTileBytes = kBM * kD * 2;          // 32 KB (A or B tile)
constexpr int kBoxBytes = kBM * kKBox * 2;        // 16 KB
constexpr int kBStages = 2;                       // = the two consumer warpgroups: warpgroup g owns B stage g
constexpr int kGroupWarps = 4;                    // per consumer warpgroup: all 128 tile rows, as two m64 halves
constexpr int kEpiThreads = 2 * kGroupWarps * 32; // 256
constexpr int kThreadsTC = kEpiThreads + 128;     // + the TMA producer warpgroup
// register reallocation: 128 x 40 + 256 x 232 <= 65,536 (the producer needs few, the accumulators many)
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
constexpr int kMaxXB = 8;                                // x-tiles per band (w <= 128)
constexpr int kStoreWarps = 3;                           // producer-warpgroup warps 9-11 write levels 2, 3
// Shared memory, sized per launch from n_xb (the x-tiles of a band); offsets from a 1024-byte aligned base:
//   mbarriers                                   1 KB
//   A tile (128 source px x 128 ch)             32 KB
//   B stages (2 x 128 target px x 128 ch)       64 KB
//   level-0 staging (2 per warpgroup, m64)      4 x 16 KB
//   level-1 staging (2 per warpgroup, m64)      4 x 4 KB
//   level-2/3 band pool                         2 x 128 x (pitch2 + 32) B
//   reverse-edge pairing (partner, work order)  2 KB
//   + 1 KB of alignment slack.  w = 80 (n_xb = 5): 212 KB; w = 128 (n_xb = 8): 220 KB (<= 227 KB).
constexpr int kBarBytes = 1024;
constexpr int kL0HalfBytes = 64 * 2 * 128;        // m64 half of a tile's level 0: 64 source px x 2 tile rows x 128 B
constexpr int kL1HalfBytes = 64 * 64;             // ... of its level 1: 64 source px x one tile row of 2 tiles (64 B)
constexpr int kL0WarpBytes = kL0HalfBytes / kGroupWarps, kL1WarpBytes = kL1HalfBytes / kGroupWarps;  // 16 source px
constexpr int kL3BandBytes = kBM * 32;            // a band's level-3 pieces, 32 B per source pixel
constexpr int kFixedBytes = 1024 + kBarBytes + (1 + kBStages) * kTileBytes;
// Reverse-edge pairing (a build with an alias table): per edge of the call its partner if it is a reader
// (int16, -1 otherwise) and the work order of the edges (full edges first, then readers), for calls of up to
// kMaxPairEdges edges; larger calls are not paired.
constexpr int kMaxPairEdges = 512;
constexpr int kPairBytes = 2 * kMaxPairEdges * 2;
// the level-2 staging is dense: one piece of pitch2 bytes per source pixel, the box of the level-2 tensor map
__host__ __device__ constexpr int pitch2_of(int n_xb) { return (n_xb * 16 + 31) / 32 * 32; }
// one of the two band buffers, level 2 then level 3
__host__ __device__ constexpr int band_bytes(int n_xb) { return kBM * pitch2_of(n_xb) + kL3BandBytes; }
__host__ __device__ constexpr int smem_bytes(int n_xb) {
  return kFixedBytes + 2 * kBStages * (kL0HalfBytes + kL1HalfBytes) + 2 * band_bytes(n_xb) + kPairBytes;
}
static_assert(smem_bytes(kMaxXB) <= 227 * 1024, "corr_build_tc_kernel exceeds the 227 KB of shared memory of a block");

using namespace gs_tc;

struct TcParams {
  int num_levels, N, h, w, hw;
  int n_mt, n_yb, n_xb;       // m-tiles, y-blocks, x-blocks
  int n_items;                // N * n_mt * n_yb
  // optional edge -> feature-map-slot indirection (video-level K-major feature maps):
  // slot1 = rig*ii[e], slot2 = rig*jj[e] + (ii[e]==jj[e])   (src/factor_graph.py:108-113,290)
  const int64_t* ii; const int64_t* jj; int rig;
  const int* out_slot;        // optional edge -> output slot of the level buffers (CorrPool)
  // levels 0 and 1 are stored as 4x4-element (32-byte) tiles, tile-row-major inside each
  // source pixel's plane (plane = H4*W4 tiles; the padding is unspecified); levels 2, 3 stay row-major.
  int w4_0, h4_0, w4_1, h4_1;
  int pitch2, pitch3;         // bytes per (source pixel, band) of levels 2 / 3 (multiples of 32)
  // optional per-slot level-0 alias table (CorrPool), one 16-byte row per slot: alias[4s] = 2 * (slot holding s's
  // level 0) + (1 if that level 0 is stored transposed), words 1-3 zero.  With it the build pairs reverse edges of the call (pair_edges) and writes
  // the entry of every slot it builds; without it every edge writes its own level 0 and no table is touched.
  int* alias;
};

// Edge r of a call is the READER of edge e when (ii[r], jj[r]) == (jj[e], ii[e]), ii[e] != jj[e], both
// orientations occur exactly once in the call, and e < r.  corr(j,i)[q][p] = <f_j(q), f_i(p)> = corr(i,j)[p][q]
// and the wgmma sums the same products in the same k order for both, so a reader's level 0 is bit for bit the
// transpose of its partner's: the reader skips its level-0 stores and the lookup reads the partner's planes.
// Rig-2 self-edges (ii == jj) read the second camera and are never paired.  Fills part[n] (the partner of a
// reader, -1 otherwise) and order[] (the full edges, then the readers, each in call order) for n < N; every
// thread of the block takes part.
__device__ void pair_edges(const TcParams& p, int16_t* part, int16_t* order) {
  const int N = p.N;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const int64_t a = p.ii[n], b = p.jj[n];
    int fwd = 0, rev = 0, partner = -1;
    for (int m = 0; m < N; ++m) {
      const int64_t c = __ldg(p.ii + m), d = __ldg(p.jj + m);
      fwd += (c == a && d == b);
      if (c == b && d == a) { ++rev; partner = m; }
    }
    part[n] = (int16_t)((a != b && fwd == 1 && rev == 1 && partner < n) ? partner : -1);
  }
  __syncthreads();
  int n_full = 0;
  for (int m = 0; m < N; ++m) n_full += part[m] < 0;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const bool rd = part[n] >= 0;
    int rank = 0;
    for (int m = 0; m < n; ++m) rank += (part[m] >= 0) == rd;
    order[rd ? n_full + rank : rank] = (int16_t)n;
  }
  __syncthreads();
}

// Build-time switch for profiling builds only (tools/build_variant.py -DGOSLAM_TC_EXPERIMENT=N); the shipped
// library has it at 0.  1 = no output writes.  2 = stores only: no operand loads and no MMAs (the accumulators
// are zero), but the whole epilogue and every store, i.e. the floor of the kernel's write pattern.
#ifndef GOSLAM_TC_EXPERIMENT
#define GOSLAM_TC_EXPERIMENT 0
#endif
constexpr int kExperiment = GOSLAM_TC_EXPERIMENT;

// ---- packed fp16 rows live in registers as uint32 pairs (lo = even column) ----
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float lo_f(uint32_t u) {
  return __half2float(__ushort_as_half((unsigned short)(u & 0xffffu)));
}
__device__ __forceinline__ float hi_f(uint32_t u) {
  return __half2float(__ushort_as_half((unsigned short)(u >> 16)));
}
// 2x2 mean of ROUNDED halves, fp32 sum in row-major window order, one rounding (avg_pool2d)
__device__ __forceinline__ float pool_pair(uint32_t top, uint32_t bot) {
  float s = lo_f(top);
  s += hi_f(top);
  s += lo_f(bot);
  s += hi_f(bot);
  return s * 0.25f;
}

// Tiled epilogue of one m64 half of a 128x128 tile (this warp: 16 source rows x 128 target pixels, the
// wgmma fragment acc[ty][.], ty = tile row of level 0 = columns 64ty..64ty+63 = patch rows 4ty..4ty+3).
// Fragment: acc[ty][4j + 2rh + e] = source row 8rh + lane/4, patch row 4ty + j/2, x = 8(j%2) + 2(lane%4) + e.
//   level 0 -> st0, the box (64 halves, 2 tile rows, 64 source px) of the level-0 tensor map, 128B-swizzled:
//             smem row R = 2 src + ty holds tiles 0..3 of that tile row, 16-byte chunk 2t + r4/2 = rows
//             r4, r4+1 of tile t.  A lane owns x pair (2q, 2q+1), q = 4(j%2) + lane%4, i.e. half of a chunk
//             row; one shfl.xor(2) per two words completes the chunks, then stmatrix writes 8 rows x 16 B.
//   level 1 -> st1, the box (32 halves, 1 tile row, 64 source px) of the level-1 tensor map, 64B-swizzled:
//             the 2x2 pools of a lane's own x pair, rows 2k, 2k+1 (y1 = 2ty + k, x1 = q); one shfl.xor(1)
//             pairs x1 columns into words.
//   level 2 -> the band pool, from those level-1 words (y2 = lane parity).
// Every smem row a warp writes belongs to its own 16 source pixels.  between_levels() runs after the level-0
// stmatrix and before the first level-1 store (the warp issues its level-0 store there).
template <typename F>
__device__ __forceinline__ void tiled_half_epilogue(const float (&acc)[2][32], unsigned char* st0, unsigned char* st1,
                                                    unsigned char* pool2_row0, int p2src, int p2row, int xb,
                                                    int wrow, int lane, bool l0, F between_levels) {
  // packed rounded fp16 pairs: W[rh][ty][r4][jx] = x pair (8jx + 2(lane%4), +1) of patch row 4ty + r4
  uint32_t W[2][2][4][2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh)
#pragma unroll
    for (int ty = 0; ty < 2; ++ty)
#pragma unroll
      for (int r4 = 0; r4 < 4; ++r4)
#pragma unroll
        for (int jx = 0; jx < 2; ++jx) {
          const int j = 2 * r4 + jx;
          W[rh][ty][r4][jx] = pack2(acc[ty][4 * j + 2 * rh], acc[ty][4 * j + 2 * rh + 1]);
        }
  // ---- level 0: 8 x stmatrix.x4 (not for a reader edge, whose level 0 its partner holds) ----
  // Matrix row s (source row 8rh + s) takes tile row ty = a ^ (s >> 2): the 8 rows of a matrix then land on
  // 8 different swizzle phases (R & 7 = (2s + ty) & 7), so each matrix is one conflict-free wavefront.
  if (l0) {
    const bool lo = (lane & 3) < 2;                // lanes holding tile 2jx (the others: tile 2jx + 1)
    const bool dflip = (lane >> 4) & 1;            // data rows s = lane/4 >= 4
    const int s8 = lane & 7;                       // address: row s8 of matrix lane/8 = (rh, tile parity)
    const uint32_t st0_u = smem_u32(st0);
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int jx = 0; jx < 2; ++jx) {
          uint32_t m[4];
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) {
            const uint32_t ra = dflip ? W[rh][a ^ 1][2 * k][jx] : W[rh][a][2 * k][jx];
            const uint32_t rb = dflip ? W[rh][a ^ 1][2 * k + 1][jx] : W[rh][a][2 * k + 1][jx];
            const uint32_t recv = __shfl_xor_sync(0xffffffffu, lo ? rb : ra, 2);
            m[2 * rh] = lo ? ra : recv;            // tile 2jx:     (r4 = 2k | 2k+1) x (x 0-1 | 2-3)
            m[2 * rh + 1] = lo ? recv : rb;        // tile 2jx + 1
          }
          const int tya = a ^ (s8 >> 2);
          const int R = 2 * (wrow + 8 * (lane >> 4) + s8) + tya;
          const int chunk = 2 * (2 * jx + ((lane >> 3) & 1)) + k;
          stmatrix_x4(st0_u + R * 128 + ((chunk ^ (R & 7)) << 4), m);
        }
  }
  between_levels();
  // ---- levels 1 and 2 ----
  const bool ev = (lane & 1) == 0;                 // even lanes: level-1 rows 0, 1 and level-2 row 0
  const uint32_t st1_u = smem_u32(st1);
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int s = wrow + 8 * rh + (lane >> 2);     // source row within the m64 half
#pragma unroll
    for (int jx = 0; jx < 2; ++jx) {
      float v[4];                                  // level-1 rows y1 = 2ty + k at x1 = 4jx + lane%4
#pragma unroll
      for (int ty = 0; ty < 2; ++ty)
#pragma unroll
        for (int k = 0; k < 2; ++k) v[2 * ty + k] = pool_pair(W[rh][ty][2 * k][jx], W[rh][ty][2 * k + 1][jx]);
      const uint32_t own01 = pack2(v[0], v[1]), own23 = pack2(v[2], v[3]);
      const uint32_t recv = __shfl_xor_sync(0xffffffffu, ev ? own23 : own01, 1);
      const uint32_t mine = ev ? own01 : own23;
      const uint32_t lo_w = ev ? mine : recv, hi_w = ev ? recv : mine;   // even x1 column | odd x1 column
      const uint32_t w0 = __byte_perm(lo_w, hi_w, 0x5410);              // row 2 * (lane & 1)
      const uint32_t w1 = __byte_perm(lo_w, hi_w, 0x7632);              // row 2 * (lane & 1) + 1
      // tile jx, rows y1 (8 B each), column pair (lane & 3) / 2; 16-byte chunk 2jx + y1/2, 64B swizzle
      const int chunk = (2 * jx + (lane & 1)) ^ ((s >> 1) & 3);
      const uint32_t a1 = st1_u + s * 64 + (chunk << 4) + ((lane & 3) >> 1) * 4;
      // even lanes write row 0 first, odd lanes row 3 first: the two stores are conflict-free
      st_shared_u32(a1 + (ev ? 0 : 8), ev ? w0 : w1);
      st_shared_u32(a1 + (ev ? 8 : 0), ev ? w1 : w0);
      // level 2: row (lane & 1) of the band, column 4xb + 2jx + (lane & 3) / 2
      const uint32_t l2 = pack2(pool_pair(w0, w1), 0.f);
      st_shared_u16(smem_u32(pool2_row0 + s * p2src + (lane & 1) * p2row + xb * 8 + (2 * jx + ((lane & 3) >> 1)) * 2),
                    (uint16_t)(l2 & 0xffffu));
    }
  }
}

__global__ void __launch_bounds__(kThreadsTC, 1)
corr_build_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                     const __grid_constant__ CUtensorMap mapL0, const __grid_constant__ CUtensorMap mapL1,
                     const __grid_constant__ CUtensorMap mapL2, const __grid_constant__ CUtensorMap mapL3,
                     const TcParams p) {
  extern __shared__ unsigned char smem_raw[];
  // 1024-byte alignment for the 128B swizzle atoms (pointer arithmetic on smem_raw: stays in the shared window)
  unsigned char* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(base);
  unsigned char* smA = base + kBarBytes;                       // ONE A stage, reloaded once per band item
  unsigned char* smB = smA + kTileBytes;                       // [kBStages]
  uint64_t* full_a = bars;
  uint64_t* empty_a = bars + 1;
  uint64_t* full_b = bars + 2;                   // [kBStages]
  uint64_t* empty_b = full_b + kBStages;
  uint64_t* staged = empty_b + kBStages;         // [2] band buffers, written by all consumer warps
  uint64_t* freed = staged + 2;                  // [2] ... and read out by the store warps' TMA stores
  // level-0 / level-1 staging, two m64 halves per warpgroup, then the two band buffers (levels 2, 3)
  unsigned char* smL0 = smB + kBStages * kTileBytes;
  unsigned char* smL1 = smL0 + 2 * kBStages * kL0HalfBytes;
  int16_t* part = reinterpret_cast<int16_t*>(smL1 + 2 * kBStages * kL1HalfBytes + 2 * band_bytes(p.n_xb));
  int16_t* order = part + kMaxPairEdges;
  constexpr bool wr = kExperiment != 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    // A is released by every consumer warp once its last MMA of the item has retired
    mbar_init(full_a, 1); mbar_init(empty_a, kEpiThreads / 32);
    for (int i = 0; i < kBStages; ++i) { mbar_init(&full_b[i], 1); mbar_init(&empty_b[i], kGroupWarps); }
    for (int i = 0; i < 2; ++i) { mbar_init(&staged[i], kEpiThreads / 32); mbar_init(&freed[i], 1); }
    fence_barrier_init();
  }
  __syncthreads();
  const bool paired = p.alias != nullptr && p.ii != nullptr && p.N <= kMaxPairEdges;
  if (paired) pair_edges(p, part, order);
  if (p.alias != nullptr && blockIdx.x == 0) {
    // the level-0 alias entry (one 16-byte row) of every slot this call builds, staged in the level-0 staging
    // (not yet in use) and written with bulk copies, so that the kernel's global writes all leave through the
    // async proxy; stream order puts them before any lookup of these slots
    int4* rows = reinterpret_cast<int4*>(smL0);
    for (int n0 = 0; n0 < p.N; n0 += kMaxPairEdges) {
      const int cnt = min(kMaxPairEdges, p.N - n0);
      for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int n = n0 + i, s = p.out_slot ? __ldg(p.out_slot + n) : n;
        const int e = paired ? part[n] : -1;
        rows[i] = make_int4(e < 0 ? 2 * s : 2 * (p.out_slot ? __ldg(p.out_slot + e) : e) + 1, 0, 0, 0);
      }
      fence_async_smem();
      __syncthreads();
      if (threadIdx.x == 0) {
        for (int i = 0; i < cnt; ++i) {
          const int s = p.out_slot ? __ldg(p.out_slot + n0 + i) : n0 + i;
          bulk_store(p.alias + 4 * (size_t)s, rows + i, 16);
        }
        bulk_commit();
        bulk_wait_read<0>();                     // the staging is reused below; the writes finish by kernel exit
      }
      __syncthreads();
    }
  }
  // work item -> edge: the full edges' items first, then the readers', so that the round-robin deal gives
  // every CTA the same mix of both (to within one item each)
  const int per_edge = p.n_mt * p.n_yb;
  auto edge_of = [&](int item) { const int k = item / per_edge; return paired ? (int)order[k] : k; };

  if (warp >= kEpiThreads / 32) {
    // ===================== TMA producer (one thread of the producer warpgroup) =====================
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kEpiThreads / 32 && lane == 0) {
      // the feature maps are re-read by every band and edge; the 0.98 GB pyramid streams past them in L2
      const uint64_t keep = l2_evict_last();
      int aph = 0, bs = 0, bph = 0;
      for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
        const int yb = item % p.n_yb;
        const int mt = (item / p.n_yb) % p.n_mt;
        const int n = edge_of(item);
        int n1 = n, n2 = n;
        if (p.ii != nullptr) {
          const int fi = (int)p.ii[n], fj = (int)p.jj[n];
          n1 = p.rig * fi;
          n2 = p.rig * fj + ((fi == fj && p.rig > 1) ? 1 : 0);
        }
        mbar_wait(empty_a, aph ^ 1);
        if constexpr (kExperiment == 2) {
          mbar_arrive(full_a);
        } else {
          mbar_expect_tx(full_a, kTileBytes);
          tma_load_3d_hint(&mapA, full_a, smA, 0, mt * kBM, n1, keep);
          tma_load_3d_hint(&mapA, full_a, smA + kBoxBytes, kKBox, mt * kBM, n1, keep);
        }
        aph ^= 1;
        for (int xb = 0; xb < p.n_xb; ++xb) {
          mbar_wait(&empty_b[bs], bph ^ 1);
          if constexpr (kExperiment == 2) {
            mbar_arrive(&full_b[bs]);
          } else {
            mbar_expect_tx(&full_b[bs], kTileBytes);
            tma_load_4d_hint(&mapB, &full_b[bs], smB + bs * kTileBytes, 0, xb * kPX, yb * kPY, n2, keep);
            tma_load_4d_hint(&mapB, &full_b[bs], smB + bs * kTileBytes + kBoxBytes, kKBox, xb * kPX,
                             yb * kPY, n2, keep);
          }
          if (++bs == kBStages) { bs = 0; bph ^= 1; }
        }
      }
    } else if (warp > kEpiThreads / 32) {
      // ===================== store warps: levels 2 and 3 of each band =====================
      const int sid = threadIdx.x - (kEpiThreads + 32);          // 0 .. 95
      const int p2src = p.pitch2, p2row = p.n_xb * 8;
      unsigned char* pool2 = smL1 + 2 * kBStages * kL1HalfBytes;
      const int h2 = p.h >> 2, h3 = p.h >> 3;
      int it = 0;                                                // items of this CTA so far
      for (int item = blockIdx.x; item < p.n_items; item += gridDim.x, ++it) {
        const int yb = item % p.n_yb;
        const int mt = (item / p.n_yb) % p.n_mt;
        const int n = edge_of(item);
        const bool out2 = wr && p.num_levels > 2 && 2 * yb < h2, out3 = wr && p.num_levels > 3 && yb < h3;
        unsigned char* s2 = pool2 + (it & 1) * band_bytes(p.n_xb);
        const uint32_t s2_u = smem_u32(s2), s3_u = s2_u + kBM * p2src;
        mbar_wait(&staged[it & 1], (it >> 1) & 1);
        if (out3) {
          // word k of a source pixel's level-3 piece = columns 2k, 2k + 1, pooled from x-tile k of level 2
          for (int i = sid; i < kBM * 8; i += kStoreWarps * 32) {
            const int k = i & 7;
            uint32_t v = 0u;
            if (k < p.n_xb) {
              const uint32_t a = s2_u + (i >> 3) * p2src + 8 * k;
              v = pack2(pool_pair(ld_shared_u32(a), ld_shared_u32(a + p2row)),
                        pool_pair(ld_shared_u32(a + 4), ld_shared_u32(a + p2row + 4)));
            }
            st_shared_u32(s3_u + 4 * i, v);
          }
          fence_async_smem();
        }
        named_bar_sync(4, kStoreWarps * 32);
        if (sid == 0) {
          // source pixels >= hw of the ragged last m-tile are clipped by the maps' per-slot bound
          const int n_out = p.out_slot ? __ldg(p.out_slot + n) : n;
          if (out2) tma_store_4d_hint(&mapL2, s2, 0, yb, mt * kBM, n_out, l2_evict_first());
          if (out3) tma_store_4d_hint(&mapL3, s2 + kBM * p2src, 0, yb, mt * kBM, n_out, l2_evict_first());
          bulk_commit();
          bulk_wait_read<0>();
          mbar_arrive(&freed[it & 1]);
        }
      }
      if (sid == 0) bulk_wait_all();
    }
  } else {
    // ===================== consumers (warps 0..7): wgmma + epilogue, two warpgroups =====================
    setmaxnreg_inc<kConsumerRegs>();
    const int group = warp >> 2;                  // takes the tiles of parity `group`, held in B stage `group`
    const int etid = threadIdx.x;                 // 0..255
    const int ts = group;
    // band staging strides (bytes)
    const int p2row = p.n_xb * 8;
    const int p2src = pitch2_of(p.n_xb);
    unsigned char* pool2 = smL1 + 2 * kBStages * kL1HalfBytes;
    if (etid < 2 * kBM) {
      // the level-2 piece's padding to pitch2 is written out with it: zeros, once per band buffer
      unsigned char* piece = pool2 + (etid >> 7) * band_bytes(p.n_xb) + (etid & (kBM - 1)) * p2src;
      for (int b = 2 * p2row; b < p2src; b += 4) st_shared_u32(smem_u32(piece + b), 0u);
    }
    const uint64_t stream = l2_evict_first();     // the pyramid is written once and not read back here
    int aph = 0, bph = 0, tile = 0, it = 0;
    for (int item = blockIdx.x; item < p.n_items; item += gridDim.x, ++it) {
      const int yb = item % p.n_yb;
      const int mt = (item / p.n_yb) % p.n_mt;
      const int n = edge_of(item);
      const int n_out = p.out_slot ? __ldg(p.out_slot + n) : n;
      const bool own0 = !paired || part[n] < 0;   // a reader's level 0 is its partner's, transposed
      mbar_wait(full_a, aph);
      aph ^= 1;
      bool a_held = true;
      // band buffer it % 2, free once the store warps' TMA has read out the band staged there before
      unsigned char* band = pool2 + (it & 1) * band_bytes(p.n_xb);
      mbar_wait(&freed[it & 1], ((it >> 1) & 1) ^ 1);
      for (int xb = 0; xb < p.n_xb; ++xb, ++tile) {
        if ((tile & (kBStages - 1)) != ts) continue;
        mbar_wait(&full_b[ts], bph);
        bph ^= 1;
        // 128 x 128 x 128 tile: two m64 row halves, N = 128 as two m64n64 halves (columns 0-63 | 64-127)
        float acc[2][2][32];
        if constexpr (kExperiment == 2) {
          // one opaque zero per accumulator, so the compiler keeps the whole epilogue
#pragma unroll
          for (int i = 0; i < 128; ++i) {
            uint32_t z;
            asm volatile("mov.b32 %0, 0;" : "=r"(z));
            acc[i >> 6][(i >> 5) & 1][i & 31] = __uint_as_float(z);
          }
        } else {
          const uint32_t a_addr = smem_u32(smA);
          const uint32_t b_addr = smem_u32(smB + ts * kTileBytes);
          wgmma_fence();
#pragma unroll
          for (int kb = 0; kb < kD / kKBox; ++kb) {
#pragma unroll
            for (int k = 0; k < kKBox / 16; ++k) {
              const uint64_t db = make_desc_sw128(b_addr + kb * kBoxBytes + k * 32);
              const uint32_t on = (kb | k) != 0 ? 1u : 0u;
#pragma unroll
              for (int mh = 0; mh < 2; ++mh) {
                const uint64_t da = make_desc_sw128(a_addr + mh * 64 * 128 + kb * kBoxBytes + k * 32);
                wgmma_m64n64(acc[mh][0], da, db, on);
                wgmma_m64n64(acc[mh][1], da, db + ((64 * 128) >> 4), on);
              }
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
        }
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&empty_b[ts]);                // this warp's MMAs are done reading the B stage
          if (xb + kBStages >= p.n_xb) mbar_arrive(empty_a);  // ... and its last MMA of the item has retired
        }
        if (xb + kBStages >= p.n_xb) a_held = false;
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
          unsigned char* st0 = smL0 + (group * 2 + mh) * kL0HalfBytes;
          unsigned char* st1 = smL1 + (group * 2 + mh) * kL1HalfBytes;
          // Each warp writes its own 16 source pixels: one bulk group for level 0, issued as soon as its stmatrix
          // is done, and one for level 1.  A buffer is written again two halves later, once wait_group.read has
          // retired its group there; the three newer groups may still be in flight.
          const int wq = warp & 3;
          const int s0 = mt * kBM + mh * 64 + wq * 16;
          const bool out0 = wr && s0 < p.hw;         // rows >= hw of the ragged last m-tile: clipped by the maps
          if (lane == 0) bulk_wait_read<3>();
          __syncwarp();
          tiled_half_epilogue(acc[mh], st0, st1, band + mh * 64 * p2src, p2src, p2row, xb, wq * 16, lane, own0, [&] {
            fence_async_smem();                      // the staged box becomes visible to the TMA engine
            __syncwarp();
            if (lane == 0) {
              if (out0 && own0) tma_store_4d_hint(&mapL0, st0 + wq * kL0WarpBytes, xb * 64, 2 * yb, s0, n_out, stream);
              bulk_commit();
              bulk_wait_read<3>();
            }
            __syncwarp();
          });
          fence_async_smem();
          __syncwarp();
          if (lane == 0) {
            if (out0 && p.num_levels > 1 && yb < p.h4_1)
              tma_store_4d_hint(&mapL1, st1 + wq * kL1WarpBytes, xb * 32, yb, s0, n_out, stream);
            bulk_commit();
          }
        }
      }
      // a warp that had no tile in this item releases A here
      if (a_held && lane == 0) mbar_arrive(empty_a);
      // hand the band to the store warps; the two consumer warpgroups go on without joining
      fence_async_smem();                        // staged rows become visible to the async (TMA) proxy
      __syncwarp();
      if (lane == 0) mbar_arrive(&staged[it & 1]);
    }
    bulk_wait_all();
  }
}

// [F, D, hw] (channel-major) -> [F, hw, D] (K-major), D = 128, times 1/4 in half — the reference's
// `fmap / 4.0` on the half tensor (src/modules/corr.py:71-72): exact for normal values.
__global__ void __launch_bounds__(256)
to_kmajor_kernel(const __half* __restrict__ in, __half* __restrict__ out, int hw) {
  __shared__ __align__(16) __half tile[kD][64 + 2];
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * 64;
  const __half* src = in + (size_t)n * kD * hw;
  const __half q = __float2half_rn(0.25f);
  if ((hw & 7) == 0 && p0 + 64 <= hw) {
    // 16-byte loads (8 pixels of one channel), scaled as half2, stored as 4 words
    const __half2 q2 = __half2half2(q);
    for (int idx = threadIdx.x; idx < kD * 8; idx += 256) {
      const int k = idx >> 3, pp = (idx & 7) * 8;
      uint4 v = __ldg(reinterpret_cast<const uint4*>(src + (size_t)k * hw + p0 + pp));
      __half2* h = reinterpret_cast<__half2*>(&v);
      uint32_t* dstw = reinterpret_cast<uint32_t*>(&tile[k][pp]);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const __half2 r = __hmul2(h[u], q2);
        dstw[u] = *reinterpret_cast<const uint32_t*>(&r);
      }
    }
  } else {
    for (int idx = threadIdx.x; idx < kD * 64; idx += 256) {
      const int k = idx / 64, pp = idx % 64;
      tile[k][pp] = (p0 + pp < hw) ? __hmul(src[(size_t)k * hw + p0 + pp], q) : __half(0.f);
    }
  }
  __syncthreads();
  __half* dst = out + ((size_t)n * hw + p0) * kD;
  for (int idx = threadIdx.x; idx < 64 * (kD / 2); idx += 256) {
    const int pp = idx / (kD / 2), k2 = idx % (kD / 2);
    if (p0 + pp < hw) {
      __half2 v = __halves2half2(tile[2 * k2][pp], tile[2 * k2 + 1][pp]);
      reinterpret_cast<__half2*>(dst + (size_t)pp * kD)[k2] = v;
    }
  }
}

// Tensor maps depend only on (base pointer, frame count, h, w, kind): a factor graph builds from the same
// video-level K-major buffer into the same slot pool for its whole life, so the cuTensorMapEncodeTiled driver
// calls of a launch (~2 us of host time each) are paid once.  Small most-recently-used table, shared by all
// threads.  kind: 0 = A operand, 1 = B operand, 2 .. 5 = tiled level 0 .. 3 output (F unused).  A tiled launch
// needs six maps, so the table holds those of a few pools at once.
struct MapKey {
  const void* base; int F, h, w, kind;
  bool operator==(const MapKey& o) const {
    return base == o.base && F == o.F && h == o.h && w == o.w && kind == o.kind;
  }
};

bool encode_map(GsEncodeTiled enc, const MapKey& k, CUtensorMap* out) {
  const cuuint64_t hw = (cuuint64_t)k.h * k.w;
  if (k.kind == 0) {           // A: [F, hw, 128] as (ch, pixel, frame), box 64 ch x 128 pixels
    cuuint64_t dims[3] = {(cuuint64_t)kD, hw, (cuuint64_t)k.F};
    cuuint64_t strides[2] = {(cuuint64_t)kD * 2, hw * kD * 2};
    cuuint32_t box[3] = {(cuuint32_t)kKBox, (cuuint32_t)kBM, 1};
    cuuint32_t es[3] = {1, 1, 1};
    return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(k.base), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  }
  if (k.kind >= 4) {
    // tiled level 2 / 3 output: per (slot, source pixel) one piece of pitch2 / 32 bytes per band, as the 4-D tensor
    // (halves within a piece, band, source pixel, slot).  Box = one band of a 128-source-pixel tile, the dense
    // staging of the store warps.  The source pixel is bounded per slot as for levels 0 / 1.
    const int n_yb = gs_cdiv(k.h, kPY);
    const cuuint64_t piece = k.kind == 4 ? (cuuint64_t)pitch2_of(gs_cdiv(k.w, kPX)) : 32;
    const cuuint64_t slot_bytes = hw * n_yb * piece;
    cuuint64_t slots = ((cuuint64_t)1 << 40) / slot_bytes;
    if (slots > 0x7fffffffull) slots = 0x7fffffffull;
    cuuint64_t dims[4] = {piece / 2, (cuuint64_t)n_yb, hw, slots};
    cuuint64_t strides[3] = {piece, n_yb * piece, slot_bytes};
    cuuint32_t box[4] = {(cuuint32_t)(piece / 2), 1u, (cuuint32_t)kBM, 1u};
    cuuint32_t es[4] = {1, 1, 1, 1};
    return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(k.base), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  }
  if (k.kind >= 2) {
    // tiled level 0 / 1 output, one plane of H4 x W4 tiles (32 B) per (slot, source pixel), as the 4-D tensor
    // (halves within a tile row, tile row, source pixel, slot).  Box = one warp's 16 source px of a 128x128 tile:
    //   level 0: 64 halves (4 tiles) x 2 tile rows x 16 source px, 128B-swizzled;
    //   level 1: 32 halves (2 tiles) x 1 tile row x 16 source px, 64B-swizzled.
    // A warp's rows are a 1024-byte aligned quarter of its m64 half's staging, so the swizzle phases are those
    // of the whole half.
    // The source-pixel bound is per slot, so the ragged last m-tile of a slot is clipped, and so are tile
    // rows / columns past H4 / W4.  The slot count is left open (CorrPool slot ids come from the device):
    // as many slots as 2^40 bytes hold.
    const int lv = k.kind - 2;
    const cuuint64_t w4 = (cuuint64_t)gs_cdiv(k.w >> lv, 4), h4 = (cuuint64_t)gs_cdiv(k.h >> lv, 4);
    const cuuint64_t slot_bytes = hw * h4 * w4 * 32;
    cuuint64_t slots = ((cuuint64_t)1 << 40) / slot_bytes;
    if (slots > 0x7fffffffull) slots = 0x7fffffffull;
    cuuint64_t dims[4] = {w4 * 16, h4, hw, slots};
    cuuint64_t strides[3] = {w4 * 32, h4 * w4 * 32, slot_bytes};
    cuuint32_t box[4] = {lv == 0 ? 64u : 32u, lv == 0 ? 2u : 1u, 16u, 1u};
    cuuint32_t es[4] = {1, 1, 1, 1};
    return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(k.base), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, lv == 0 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
               CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  }
  // B: (ch, x, y, frame), box 64 ch x 16 x 8: an image patch; rows / columns outside the image read as zero
  cuuint64_t dims[4] = {(cuuint64_t)kD, (cuuint64_t)k.w, (cuuint64_t)k.h, (cuuint64_t)k.F};
  cuuint64_t strides[3] = {(cuuint64_t)kD * 2, (cuuint64_t)k.w * kD * 2, hw * kD * 2};
  cuuint32_t box[4] = {(cuuint32_t)kKBox, (cuuint32_t)kPX, (cuuint32_t)kPY, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(k.base), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

GsTensorMapCache<MapKey, 32, encode_map> g_maps;

// opt-in dynamic shared memory is a per-device function attribute (gs_device_setup)
int corr_build_setup(int) {
  GS_CUDA(cudaFuncSetAttribute(corr_build_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(kMaxXB)));
  return GOSLAM_OK;
}

// launch the tensor-core kernel on the video-level K-major (pre-scaled) feature maps f = [F, hw, 128]
int launch_tc(const __half* f, int F, const int64_t* ii, const int64_t* jj, int rig, const int* out_slot,
              int* alias, __half* const* levels, int num_levels, int N, int h, int w, cudaStream_t st) {
  const int hw = h * w;
  // the tensor stores need 16-byte aligned level buffers
  for (int i = 0; i < num_levels; ++i)
    if (reinterpret_cast<uintptr_t>(levels[i]) & 15) return GOSLAM_EINVAL;
  CUtensorMap mapA, mapB, mapL0, mapL1, mapL2, mapL3;
  if (!g_maps.get(MapKey{f, F, h, w, 0}, &mapA) || !g_maps.get(MapKey{f, F, h, w, 1}, &mapB))
    return GOSLAM_ELAUNCH;
  mapL0 = mapL1 = mapL2 = mapL3 = mapA;      // the maps of levels >= num_levels are unused
  CUtensorMap* maps[4] = {&mapL0, &mapL1, &mapL2, &mapL3};
  for (int i = 0; i < num_levels; ++i)
    if (!g_maps.get(MapKey{levels[i], 0, h, w, 2 + i}, maps[i])) return GOSLAM_ELAUNCH;
  TcParams p{};
  p.num_levels = num_levels; p.N = N; p.h = h; p.w = w; p.hw = hw;
  p.n_mt = gs_cdiv(hw, kBM); p.n_yb = gs_cdiv(h, kPY); p.n_xb = gs_cdiv(w, kPX);
  p.n_items = N * p.n_mt * p.n_yb;
  p.ii = ii; p.jj = jj; p.rig = rig; p.out_slot = out_slot; p.alias = alias;
  p.w4_0 = gs_cdiv(w, 4); p.h4_0 = gs_cdiv(h, 4);
  p.w4_1 = gs_cdiv(w >> 1, 4); p.h4_1 = gs_cdiv(h >> 1, 4);
  p.pitch2 = pitch2_of(p.n_xb); p.pitch3 = 32;
  int sms = 0;
  int rc = gs_device_setup<corr_build_setup>();
  if (rc == GOSLAM_OK) rc = gs_sm_count(&sms);
  if (rc) return rc;
  const int grid = p.n_items < sms ? p.n_items : sms;
  corr_build_tc_kernel<<<grid, kThreadsTC, smem_bytes(p.n_xb), st>>>(mapA, mapB, mapL0, mapL1, mapL2, mapL3, p);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // namespace

extern "C" {

int goslam_fmaps_to_kmajor(const void* fmaps, void* out, int F, int D, int h, int w, void* stream) {
  if (F < 0 || D != kD || h <= 0 || w <= 0) return GOSLAM_EINVAL;
  if (F == 0) return GOSLAM_OK;
  dim3 tg(gs_cdiv(h * w, 64), F);
  to_kmajor_kernel<<<tg, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(fmaps),
                                                         reinterpret_cast<__half*>(out), h * w);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

size_t goslam_corr_level_plane_elems(int level, int layout, int h, int w) {
  if (level < 0 || level > 3 || h <= 0 || w <= 0) return 0;
  const int hl = h >> level, wl = w >> level;
  if (hl <= 0 || wl <= 0) return 0;
  if (layout == GOSLAM_LAYOUT_TILED) {
    if (level < 2) return (size_t)gs_cdiv(hl, 4) * gs_cdiv(wl, 4) * 16;
    // levels 2 / 3: one padded piece per 8-row band of level 0 (2 rows / 1 row of the level)
    const int n_yb = gs_cdiv(h, kPY), n_xb = gs_cdiv(w, kPX);
    return level == 2 ? (size_t)n_yb * ((n_xb * 8 + 15) / 16 * 16) : (size_t)n_yb * 16;
  }
  return (size_t)hl * wl;
}

int goslam_corr_pool_build(const void* fmaps_kmajor, int F, int rig, const int64_t* ii,
                           const int64_t* jj, const int* slots, void* const* levels,
                           int num_levels, int N, int D, int h, int w, void* stream) {
  return goslam_corr_pool_build_paired(fmaps_kmajor, F, rig, ii, jj, slots, nullptr, levels, num_levels, N, D, h,
                                       w, stream);
}

int goslam_corr_pool_build_paired(const void* fmaps_kmajor, int F, int rig, const int64_t* ii,
                                  const int64_t* jj, const int* slots, int* alias, void* const* levels,
                                  int num_levels, int N, int D, int h, int w, void* stream) {
  if (N < 0 || F <= 0 || rig < 1 || D != kD || h <= 0 || w <= 0 || num_levels < 1 || num_levels > 4)
    return GOSLAM_EINVAL;
  if ((h >> (num_levels - 1)) <= 0 || (w >> (num_levels - 1)) <= 0) return GOSLAM_EINVAL;
  if (w > kMaxXB * kPX) return GOSLAM_EINVAL;
  if (N == 0) return GOSLAM_OK;
  return launch_tc(reinterpret_cast<const __half*>(fmaps_kmajor), F, ii, jj, rig, slots, alias,
                   reinterpret_cast<__half* const*>(levels), num_levels, N, h, w, (cudaStream_t)stream);
}

}  // extern "C"

namespace {

// Materialize aliased level-0 planes: slot slots[i] gets its own level 0, the transpose of holders[i]'s, and its
// alias entry is reset to itself.  Element (q, p) of the slot is element (p, q) of the holder; the padding of a
// plane is written as zeros, as the build leaves it.
__global__ void __launch_bounds__(256)
corr_unalias_kernel(__half* __restrict__ l0, int* __restrict__ alias, const int* __restrict__ slots,
                    const int* __restrict__ holders, int h, int w) {
  const int hw = h * w, w4 = gs_cdiv(w, 4);
  const long long plane = (long long)gs_cdiv(h, 4) * w4 * 16;
  const int s = __ldg(slots + blockIdx.y), t = __ldg(holders + blockIdx.y);
  __half* dst = l0 + (long long)s * hw * plane;
  const __half* src = l0 + (long long)t * hw * plane;
  const long long total = (long long)hw * plane;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i / plane), off = (int)(i % plane);
    const int tile = off >> 4, py = (tile / w4) * 4 + ((off >> 2) & 3), px = (tile % w4) * 4 + (off & 3);
    __half v = __float2half(0.f);
    if (py < h && px < w) {
      const int qy = q / w, qx = q % w;
      const int qoff = ((qy >> 2) * w4 + (qx >> 2)) * 16 + (qy & 3) * 4 + (qx & 3);
      v = src[(long long)(py * w + px) * plane + qoff];
    }
    dst[i] = v;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) alias[4 * (size_t)s] = 2 * s;
}

}  // namespace

extern "C" {

int goslam_corr_pool_unalias(void* level0, int* alias, const int* slots, const int* holders, int n, int h, int w,
                             void* stream) {
  if (n < 0 || h <= 0 || w <= 0) return GOSLAM_EINVAL;
  if (n == 0) return GOSLAM_OK;
  corr_unalias_kernel<<<dim3(264, n), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<__half*>(level0), alias,
                                                                       slots, holders, h, w);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

}  // extern "C"
