// conv_tc.cu — the update operator's ConvGRU (SURVEY §8f-4) on Hopper wgmma: 3x3 / 1x1 convolutions as an
// implicit GEMM with the GRU gates fused into the epilogues.
//
// Replaces ConvGRU.forward (src/modules/gru.py:21-39) as called by UpdateModule.forward
// (src/droid_net.py:125, `self.gru(net, inp, corr, flow)`):
//     glo = mean_hw(sigmoid(w(net)) * net)                                   1x1 conv + pooling
//     z = sigmoid(convz([net|inp|corr|flow]) + convz_glo(glo))               3x3, 448 -> 128
//     r = sigmoid(convr([net|inp|corr|flow]) + convr_glo(glo))               3x3, 448 -> 128
//     q = tanh(convq([r*net|inp|corr|flow]) + convq_glo(glo))                3x3, 448 -> 128
//     net' = (1 - z) * net + z * q
// The reference runs 7 cuDNN convolutions, 2 torch.cat of the 448-channel input and ~12 elementwise kernels.
// Here: three launches of ONE kernel (conv_tc_kernel) with different epilogues, plus two tiny ones:
//   pass G  1x1 conv of net, epilogue: sigmoid(.)*net, per-image channel sums       -> glo_sum [B,128]
//   (gru_glo_fc_kernel: the three 128x128 matvecs on the pooled vector              -> glo     [B,384])
//   pass ZR 3x3 conv with z and r stacked to N = 256 (the activation tile is loaded once for both
//           gates), epilogue: bias + glo, sigmoid, z and r*net written                -> z, rnet
//   pass Q  3x3 conv over [rnet|inp|corr|flow], epilogue: tanh, (1-z)*net + z*q       -> net'
//
// Implicit GEMM: M = 128 output pixels (an 8x16 image patch), N = output channels (128 or 256),
// K = taps x input channels in chunks of 64.  Activations are NHWC fp16, so the patch shifted by a tap is ONE
// TMA box (64 ch, 16, 8, 1) of a 4-D tensor map (ch, x, y, image) — image borders are the TMA's zero fill, the
// concatenated input never exists (one tensor map per source tensor) — and lands K-major / SWIZZLE_128B, exactly
// the A operand.  Weights are [tap][cout][cin] fp16: box (64, N, 1) = the B operand.  Two consumer warpgroups
// (tile rows 0-63 | 64-127) issue wgmma m64nNk16 with fp32 register accumulators and run the epilogue on the
// fragment; warp 8 = TMA producer, which keeps a 4-stage ring of (A, B) chunks ahead of the MMAs.
// fp16 operands, fp32 accumulation, fp32 gate arithmetic, fp16 state — what the reference's autocast region
// computes (src/factor_graph.py:198, torch.cuda.amp.autocast) with one rounding less per gate.
// The whole operator (goslam_update_op) rounds to fp16 exactly where it stores: operands (weights except the fp32 w_glo,
// net, inp, corr, flow in the 7x7 im2col), the encoder outputs c1, c2, f1, f2, the GRU's z, r*net and net' (glo, r and q
// stay fp32), the hidden layer, a1, the scatter-mean, a2 and upmask; delta, weight and eta are written as fp32.
// oracle/update_oracle.py (round16=True) restates this in float64.
#include "common.cuh"
#include "tc_ptx.cuh"

using namespace gs_tc;

namespace {

constexpr int kPY = 8, kPX = 16, kBM = kPY * kPX;   // output patch = MMA M
constexpr int kKC = 64;                             // channels per K chunk (128-byte rows)
constexpr int kABytes = kBM * kKC * 2;              // 16 KB
constexpr int kMaxN = 256;
constexpr int kBBytes = kMaxN * kKC * 2;            // 32 KB (a 128-channel pass uses half)
constexpr int kStages = 4;
constexpr int kConsumerWarps = 8;                   // two warpgroups: tile rows 0-63 | 64-127
constexpr int kThreadsC = (kConsumerWarps + 1) * 32; // + the TMA producer warp
constexpr int kVecMax = 1024;                       // per-channel epilogue vector (bias, or bias + glo of the tile's image)
constexpr int kSmemC = 1024 + kStages * (kABytes + kBBytes) + 256 + kVecMax * 4;
constexpr int kMaxIn = 4;

enum { EPI_ACT = 0, EPI_GLO = 1, EPI_ZR = 2, EPI_Q = 3 };
enum { ACT_NONE = 0, ACT_RELU = 1, ACT_SIGMOID = 2, ACT_SOFTPLUS = 3 };

struct ConvMaps {
  CUtensorMap in[kMaxIn];
  CUtensorMap w;
};

struct ConvParams {
  int B, h, w, n_yb, n_xb, n_tiles;
  int taps;                 // 1 or 9
  int n_in;
  int chunks[kMaxIn];       // K chunks (64 channels) of each input tensor
  int coff[kMaxIn];         // first channel of each input inside its tensor (a channel slice of a wider NHWC tensor)
  int N;                    // output channels per tile (16..256, multiple of 16)
  int n_nt;                 // output-channel tiles (cout_pad / N)
  // EPI_ACT: out = act(conv + bias) * out_scale, NHWC [.., out_stride] at channel out_offset, first `cout` channels
  int act, cout, out_stride, out_offset, out_f32;
  float out_scale;
  void* out;
  // f32 outputs only: channels >= split go to out2 (same stride) and get act2 instead of act (fused 2-channel heads)
  int split, act2;
  void* out2;
  int epi;
  const float* bias;        // [N]
  const float* glo;         // [B, 384] (z | r | q) or nullptr
  const __half* net;        // [B, h, w, 128] NHWC
  const __half* z_in;       // EPI_Q
  __half* z_out;            // EPI_ZR
  __half* rnet_out;         // EPI_ZR
  __half* net_out;          // EPI_Q
  float* glo_sum;           // EPI_GLO: [B * patches * 8, 128] partial sums over 16 pixels of sigmoid(.) * net
};

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

// 16 halves = one whole 32-byte sector per store (16-byte pieces are partial-sector writes: read-modify-write in L2)
__device__ __forceinline__ void st_sector(void* dst, const uint32_t (&o)[8]) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4}; st.global.v4.b32 [%0+16], {%5,%6,%7,%8};" ::"l"(dst), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]),
               "r"(o[4]), "r"(o[5]), "r"(o[6]), "r"(o[7]) : "memory");
}
// Fragment of one consumer thread after the m64nN MMAs: acc[4J + e] = tile row wrow + lane/4 + 8*(e>>1), output
// channel (of the tile) 8J + 2*(lane%4) + (e&1), J = 0 .. N/8-1 (N/64 m64n64 MMAs, then m64n16 for the rest).
template <int N>
__device__ __forceinline__ void conv_mma_k16(float (&acc)[N / 2], uint32_t a_addr, uint32_t b_addr, uint32_t on) {
  const uint64_t da = make_desc_sw128(a_addr);
#pragma unroll
  for (int s = 0; s < N / 64; ++s)
    wgmma_m64n64(*reinterpret_cast<float(*)[32]>(acc + 32 * s), da, make_desc_sw128(b_addr + s * 64 * 128), on);
#pragma unroll
  for (int s = (N / 64) * 4; s < N / 16; ++s)
    wgmma_m64n16(*reinterpret_cast<float(*)[8]>(acc + 8 * s), da, make_desc_sw128(b_addr + s * 16 * 128), on);
}

template <int N>
__global__ void __launch_bounds__(kThreadsC, 1)
conv_tc_kernel(const __grid_constant__ ConvMaps maps, const ConvParams p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base =
      reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* smA = base;
  unsigned char* smB = base + kStages * kABytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + kStages * (kABytes + kBBytes));
  uint64_t* full = bars;                    // [kStages]
  uint64_t* empty = full + kStages;         // [kStages]
  float* svec = reinterpret_cast<float*>(base + kStages * (kABytes + kBBytes) + 256);   // [kVecMax]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // EPI_ACT / EPI_GLO: the bias vector is the same for every tile: stage it once
  if (p.epi == EPI_ACT || p.epi == EPI_GLO)
    for (int i = threadIdx.x; i < p.n_nt * N && i < kVecMax; i += kThreadsC) svec[i] = p.bias[i];
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();
  int kiters = 0;
  for (int i = 0; i < p.n_in; ++i) kiters += p.chunks[i];
  kiters *= p.taps;
  const uint32_t stage_tx = kABytes + (uint32_t)N * kKC * 2;

  if (warp == kConsumerWarps) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const int nt = tile % p.n_nt, pt = tile / p.n_nt;
        const int xb = pt % p.n_xb, yb = (pt / p.n_xb) % p.n_yb, b = pt / (p.n_xb * p.n_yb);
        for (int tap = 0; tap < p.taps; ++tap) {
          const int dy = p.taps == 9 ? tap / 3 - 1 : 0, dx = p.taps == 9 ? tap % 3 - 1 : 0;
          int gchunk = 0;
          for (int ci = 0; ci < p.n_in; ++ci)
            for (int kc = 0; kc < p.chunks[ci]; ++kc, ++gchunk) {
              mbar_wait(&empty[s], ph ^ 1);
              mbar_expect_tx(&full[s], stage_tx);
              tma_load_4d(&maps.in[ci], &full[s], smA + s * kABytes, p.coff[ci] + kc * kKC, xb * kPX + dx, yb * kPY + dy, b);
              tma_load_3d(&maps.w, &full[s], smB + s * kBBytes, gchunk * kKC, nt * N, tap);
              if (++s == kStages) { s = 0; ph ^= 1; }
            }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup g = tile rows 64g..64g+63 =====================
    const int wrow = (warp >> 2) * 64 + (warp & 3) * 16;
    const int q = lane & 3;
    int r_[2], pyx[2];
    r_[0] = wrow + (lane >> 2); r_[1] = r_[0] + 8;
    pyx[0] = r_[0]; pyx[1] = r_[1];
    int s = 0, ph = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
      const int nt = tile % p.n_nt, pt = tile / p.n_nt;
      const int xb = pt % p.n_xb, yb = (pt / p.n_xb) % p.n_yb, b = pt / (p.n_xb * p.n_yb);
      float acc[N / 2];
      for (int it = 0; it < kiters; ++it) {
        mbar_wait(&full[s], ph);
        const uint32_t a_addr = smem_u32(smA + s * kABytes) + (warp >> 2) * 64 * 128;
        const uint32_t b_addr = smem_u32(smB + s * kBBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kKC / 16; ++k) conv_mma_k16<N>(acc, a_addr + k * 32, b_addr + k * 32, (it | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        if (++s == kStages) { s = 0; ph ^= 1; }
      }
      bool ok[2];
      size_t pix[2];
#pragma unroll
      for (int e2 = 0; e2 < 2; ++e2) {
        const int y = yb * kPY + pyx[e2] / kPX, x = xb * kPX + pyx[e2] % kPX;
        ok[e2] = y < p.h && x < p.w;
        pix[e2] = ((size_t)b * p.h + (ok[e2] ? y : 0)) * p.w + (ok[e2] ? x : 0);
      }
      if (p.epi == EPI_ZR || p.epi == EPI_Q) {
        // per-tile channel vector = bias + the image's global term, staged by the 256 consumer threads
        asm volatile("bar.sync 2, 256;" ::: "memory");          // previous tile's vector no longer in use
        const float* glo = p.glo + (size_t)b * 384 + (p.epi == EPI_Q ? 256 : 0);
        for (int i = threadIdx.x; i < N; i += 256) svec[i] = p.bias[i] + glo[i];
        asm volatile("bar.sync 2, 256;" ::: "memory");
      }
      if (p.epi == EPI_ACT) {
#pragma unroll
        for (int J = 0; J < N / 8; ++J) {
          const int ch = nt * N + 8 * J + 2 * q;       // output channel of acc[4J + 2*e2 + {0,1}]
#pragma unroll
          for (int e2 = 0; e2 < 2; ++e2) {
            float r[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              float v = acc[4 * J + 2 * e2 + u] + svec[ch + u];
              // small fused heads: channels >= split take act2 instead of act.  A split layer has cout <= 8, so only
              // J = 0 holds stored channels; testing J (a compile-time constant) keeps every other column's act uniform
              const int act = (J == 0 && p.split > 0 && ch + u >= p.split) ? p.act2 : p.act;
              if (act == ACT_RELU) v = fmaxf(v, 0.f);
              else if (act == ACT_SIGMOID) v = sigmoidf_(v);
              else if (act == ACT_SOFTPLUS) v = (v > 20.f) ? v : log1pf(__expf(v));
              r[u] = v * p.out_scale;
            }
            if (!ok[e2]) continue;
            if (p.out_f32) {
              float* dst = reinterpret_cast<float*>(p.out) + pix[e2] * p.out_stride + p.out_offset;
              float* dst2 = reinterpret_cast<float*>(p.out2) + pix[e2] * p.out_stride - p.split;
#pragma unroll
              for (int u = 0; u < 2; ++u)
                if (ch + u < p.cout) {
                  if (p.split > 0 && ch + u >= p.split) dst2[ch + u] = r[u];
                  else dst[ch + u] = r[u];
                }
            } else {
              __half* dst = reinterpret_cast<__half*>(p.out) + pix[e2] * p.out_stride + p.out_offset + ch;
              if (ch + 1 < p.cout) *reinterpret_cast<__half2*>(dst) = __floats2half2_rn(r[0], r[1]);
              else if (ch < p.cout) dst[0] = __float2half_rn(r[0]);
            }
          }
        }
      } else if (p.epi == EPI_GLO) {
        // g = sigmoid(conv + b) * net; per-image channel sums (the mean's divisor is applied by the fc kernel):
        // one partial per (patch, warp) = 16 pixels, summed in a fixed order: deterministic
        float* part = p.glo_sum + ((size_t)pt * kConsumerWarps + (wrow >> 4)) * 128;
#pragma unroll
        for (int J = 0; J < N / 8; ++J) {
          const int ch = 8 * J + 2 * q;
          float t[2] = {0.f, 0.f};
#pragma unroll
          for (int e2 = 0; e2 < 2; ++e2) {
            if (!ok[e2]) continue;
            const float2 nv = __half22float2(__ldg(reinterpret_cast<const __half2*>(p.net + pix[e2] * 128 + ch)));
            t[0] += sigmoidf_(acc[4 * J + 2 * e2] + svec[ch]) * nv.x;
            t[1] += sigmoidf_(acc[4 * J + 2 * e2 + 1] + svec[ch + 1]) * nv.y;
          }
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            t[0] += __shfl_xor_sync(0xffffffffu, t[0], o);
            t[1] += __shfl_xor_sync(0xffffffffu, t[1], o);
          }
          if (lane < 4) *reinterpret_cast<float2*>(part + ch) = make_float2(t[0], t[1]);
        }
      } else if (p.epi == EPI_ZR) {
#pragma unroll
        for (int J = 0; J < N / 8; ++J) {
          const int ch = 8 * J + 2 * q, c = ch & 127;
          const bool is_r = ch >= 128;
#pragma unroll
          for (int e2 = 0; e2 < 2; ++e2) {
            if (!ok[e2]) continue;
            const float g0 = sigmoidf_(acc[4 * J + 2 * e2] + svec[ch]), g1 = sigmoidf_(acc[4 * J + 2 * e2 + 1] + svec[ch + 1]);
            __half2 h;
            if (is_r) {
              const float2 nv = __half22float2(__ldg(reinterpret_cast<const __half2*>(p.net + pix[e2] * 128 + c)));
              h = __floats2half2_rn(g0 * nv.x, g1 * nv.y);
            } else {
              h = __floats2half2_rn(g0, g1);
            }
            *reinterpret_cast<__half2*>((is_r ? p.rnet_out : p.z_out) + pix[e2] * 128 + c) = h;
          }
        }
      } else {   // EPI_Q
#pragma unroll
        for (int J = 0; J < N / 8; ++J) {
          const int ch = 8 * J + 2 * q;
#pragma unroll
          for (int e2 = 0; e2 < 2; ++e2) {
            if (!ok[e2]) continue;
            const float q0 = tanhf(acc[4 * J + 2 * e2] + svec[ch]), q1 = tanhf(acc[4 * J + 2 * e2 + 1] + svec[ch + 1]);
            const float2 nv = __half22float2(__ldg(reinterpret_cast<const __half2*>(p.net + pix[e2] * 128 + ch)));
            const float2 zz = __half22float2(__ldg(reinterpret_cast<const __half2*>(p.z_in + pix[e2] * 128 + ch)));
            *reinterpret_cast<__half2*>(p.net_out + pix[e2] * 128 + ch) =
                __floats2half2_rn((1.0f - zz.x) * nv.x + zz.x * q0, (1.0f - zz.y) * nv.y + zz.y * q1);
          }
        }
      }
    }
  }
}

// glo[b] = W_glo mean_px(sigmoid(w(net)) * net) + b_glo : sums the per-(patch, warp) partials of pass G in a fixed order,
// then the three 1x1 "global" convolutions on the pooled vector, one warp per output (coalesced weight rows)
__global__ void __launch_bounds__(256)
gru_glo_fc_kernel(const float* __restrict__ part, int parts_per_image, const float* __restrict__ w_glo,
                  const float* __restrict__ b_glo, float* __restrict__ glo, float inv_hw) {
  __shared__ float v[128];
  const int b = blockIdx.x;
  if (threadIdx.x < 128) {
    const float* pp = part + (size_t)b * parts_per_image * 128 + threadIdx.x;
    float acc = 0.f;
    for (int i = 0; i < parts_per_image; ++i) acc += pp[(size_t)i * 128];
    v[threadIdx.x] = acc * inv_hw;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = warp; o < 384; o += 8) {
    const float4 wv = *reinterpret_cast<const float4*>(w_glo + (size_t)o * 128 + lane * 4);
    float acc = wv.x * v[lane * 4] + wv.y * v[lane * 4 + 1] + wv.z * v[lane * 4 + 2] + wv.w * v[lane * 4 + 3];
    acc = gs_warp_sum(acc);
    if (lane == 0) glo[(size_t)b * 384 + o] = acc + b_glo[o];
  }
}

// [B, rows, cols] -> [B, cols, rows] fp16 through a 32x32 shared-memory tile (generic shapes)
__global__ void transpose_f16_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int rows, int cols) {
  __shared__ __half t[32][34];
  const size_t boff = (size_t)blockIdx.z * rows * cols;
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    if (r < rows && c < cols) t[i][threadIdx.x] = src[boff + (size_t)r * cols + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < rows && c < cols) dst[boff + (size_t)c * rows + r] = t[threadIdx.x][i];
  }
}

// Fast path of the two layout conversions, 64 x 64 tiles: 16-byte loads along the source's contiguous dimension, whole
// 32-byte sectors (16 halves) on the way out, both shared-memory phases conflict-free (row stride 33 words).
//   NCHW -> NHWC: src [B][C][hw] (rows = channels, zero beyond C), dst [B][hw][Cpad]
__global__ void __launch_bounds__(256)
nchw_to_nhwc64_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int C, int Cpad, int hw) {
  __shared__ uint32_t t[64][33];
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;          // r: channel, c: pixel
  const __half* s = src + (size_t)blockIdx.z * C * hw;
  __half* d = dst + (size_t)blockIdx.z * hw * Cpad;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = threadIdx.x + 256 * i, r = idx >> 3, c8 = idx & 7;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r0 + r < C && c0 + c8 * 8 < hw) v = __ldg(reinterpret_cast<const uint4*>(s + (size_t)(r0 + r) * hw + c0 + c8 * 8));
    t[r][c8 * 4 + 0] = v.x; t[r][c8 * 4 + 1] = v.y; t[r][c8 * 4 + 2] = v.z; t[r][c8 * 4 + 3] = v.w;
  }
  __syncthreads();
  const int px = threadIdx.x & 63, r16 = threadIdx.x >> 6;
  if (c0 + px < hw && r0 + r16 * 16 < Cpad) {
    uint32_t o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t a = t[r16 * 16 + 2 * j][px >> 1], b = t[r16 * 16 + 2 * j + 1][px >> 1];
      const uint32_t lo = (px & 1) ? (a >> 16) : (a & 0xffffu), hi = (px & 1) ? (b >> 16) : (b & 0xffffu);
      o[j] = lo | (hi << 16);
    }
    st_sector(d + (size_t)(c0 + px) * Cpad + r0 + r16 * 16, o);
  }
}
//   NHWC -> NCHW: src [B][hw][C] (C % 64 == 0), dst [B][C][hw]; rows = pixels here
__global__ void __launch_bounds__(256)
nhwc_to_nchw64_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int C, int hw) {
  __shared__ uint32_t t[64][33];
  const int p0 = blockIdx.y * 64, c0 = blockIdx.x * 64;          // rows: pixel, cols: channel
  const __half* s = src + (size_t)blockIdx.z * hw * C;
  __half* d = dst + (size_t)blockIdx.z * C * hw;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = threadIdx.x + 256 * i, r = idx >> 3, c8 = idx & 7;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (p0 + r < hw) v = __ldg(reinterpret_cast<const uint4*>(s + (size_t)(p0 + r) * C + c0 + c8 * 8));
    t[r][c8 * 4 + 0] = v.x; t[r][c8 * 4 + 1] = v.y; t[r][c8 * 4 + 2] = v.z; t[r][c8 * 4 + 3] = v.w;
  }
  __syncthreads();
  const int ch = threadIdx.x & 63, q16 = threadIdx.x >> 6;        // 16 consecutive pixels of one channel
  if (p0 + q16 * 16 < hw) {
    uint32_t o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t a = t[q16 * 16 + 2 * j][ch >> 1], b = t[q16 * 16 + 2 * j + 1][ch >> 1];
      const uint32_t lo = (ch & 1) ? (a >> 16) : (a & 0xffffu), hi = (ch & 1) ? (b >> 16) : (b & 0xffffu);
      o[j] = lo | (hi << 16);
    }
    __half* dp = d + (size_t)(c0 + ch) * hw + p0 + q16 * 16;
    if (p0 + q16 * 16 + 16 <= hw) st_sector(dp, o);
    else
      for (int j = 0; j < 16 && p0 + q16 * 16 + j < hw; ++j)
        dp[j] = __ushort_as_half((unsigned short)((o[j >> 1] >> ((j & 1) * 16)) & 0xffffu));
  }
}

// [B, C, hw] -> [B, hw, Cpad] with zero channels C..Cpad-1
__global__ void transpose_pad_f16_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int C, int Cpad, int hw) {
  __shared__ __half t[32][34];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;          // r: channel, c: pixel
  const __half* s = src + (size_t)blockIdx.z * C * hw;
  __half* d = dst + (size_t)blockIdx.z * hw * Cpad;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    t[i][threadIdx.x] = (r < C && c < hw) ? s[(size_t)r * hw + c] : __half(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < Cpad && c < hw) d[(size_t)c * Cpad + r] = t[threadIdx.x][i];
  }
}

// flow_encoder.0 (src/droid_net.py:84): 7x7 convolution of the 4 motion channels to 128 + ReLU on tensor cores.
//   in  [B,4,h,w] f32 (the motion features as FactorGraph hands them over), out [B,h,w,128] f16 NHWC
constexpr int kF7Halo = (kPY + 6) * (kPX + 6) * 4;   // 14x22x4 input halo of an 8x16 output patch
// im2col in shared memory.  K = 49 taps x 4 channels = 196, zero-padded to 256 = four 64-wide
// chunks.  The 128 builder threads (one per output pixel of the 8x16 patch) write their im2col row straight into the
// K-major SWIZZLE_128B operand layout the TMA would have produced (row r of a chunk at r*128 B inside 8-row / 1024-byte
// atoms, its 16-byte pieces XOR-ed with r % 8); the weights [128][256] come in once per CTA by TMA; two warpgroups
// (tile rows 0-63 | 64-127) issue 16 k-steps of two wgmma m64n64k16 each; bias + ReLU epilogue to NHWC f16.
constexpr int kF7K = 256, kF7ABytes = kBM * kF7K * 2, kF7BBytes = 128 * kF7K * 2;
constexpr int kF7Threads = 256;
constexpr int kF7Smem = 1024 + kF7ABytes + kF7BBytes + kF7Halo * 4 + 128 * 4 + 256;
__global__ void __launch_bounds__(kF7Threads, 1)
flow7x7_tc_kernel(const __grid_constant__ CUtensorMap wmap, const float* __restrict__ in, const float* __restrict__ bias,
                  __half* __restrict__ out, int B, int h, int w) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base =
      reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* smA = base;
  unsigned char* smB = base + kF7ABytes;
  float* si = reinterpret_cast<float*>(smB + kF7BBytes);          // [14][22][4]
  float* sb = si + kF7Halo;                                       // [128]
  uint64_t* w_full = reinterpret_cast<uint64_t*>(sb + 128);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) { mbar_init(w_full, 1); fence_barrier_init(); }
  for (int i = threadIdx.x; i < 128; i += kF7Threads) sb[i] = bias[i];
  __syncthreads();
  if (threadIdx.x == 0) {                            // weights: four (64 K, 128 cout) boxes, once
    mbar_expect_tx(w_full, kF7BBytes);
    for (int kc = 0; kc < 4; ++kc) tma_load_3d(&wmap, w_full, smB + kc * (128 * 128), kc * 64, 0, 0);
  }
  const int n_xb = gs_cdiv_dev(w, kPX), n_yb = gs_cdiv_dev(h, kPY), n_tiles = B * n_xb * n_yb;
  const int wg_row = (warp >> 2) * 64;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int xb = tile % n_xb, yb = (tile / n_xb) % n_yb, b = tile / (n_xb * n_yb);
    // ---- input halo (fp32), all threads
    for (int i = threadIdx.x; i < kF7Halo; i += kF7Threads) {
      const int ci = i & 3, xx = (i >> 2) % (kPX + 6), yy = (i >> 2) / (kPX + 6);
      const int gx = xb * kPX + xx - 3, gy = yb * kPY + yy - 3;
      si[i] = (gx >= 0 && gx < w && gy >= 0 && gy < h) ? in[(((size_t)b * 4 + ci) * h + gy) * w + gx] : 0.f;
    }
    __syncthreads();
    // ---- im2col rows into the swizzled A tile
    if (threadIdx.x < 128) {
      const int r = threadIdx.x, py = r / kPX, px = r % kPX;
      unsigned char* rowp = smA + (r >> 3) * 1024 + (r & 7) * 128;
      for (int t2 = 0; t2 < 32; ++t2) {              // pairs of taps = one 16-byte piece (8 halves)
        uint32_t o[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int t = 2 * t2 + u;
          if (t < 49) {
            const float4 v = *reinterpret_cast<const float4*>(si + ((py + t / 7) * (kPX + 6) + px + t % 7) * 4);
            const __half2 a = __floats2half2_rn(v.x, v.y), c = __floats2half2_rn(v.z, v.w);
            o[2 * u] = *reinterpret_cast<const uint32_t*>(&a);
            o[2 * u + 1] = *reinterpret_cast<const uint32_t*>(&c);
          }
        }
        const int kc = t2 >> 3, c16 = t2 & 7;
        *reinterpret_cast<uint4*>(rowp + kc * (kBM * 128) + ((c16 ^ (r & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
    fence_async_smem();                              // generic-proxy writes -> visible to the tensor core (async proxy)
    __syncthreads();
    if (tile == (int)blockIdx.x) mbar_wait(w_full, 0);
    float acc[2][32];
    {
      const uint32_t a_addr = smem_u32(smA) + wg_row * 128, b_addr = smem_u32(smB);
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < 4; ++kc)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t da = make_desc_sw128(a_addr + kc * (kBM * 128) + k * 32);
          const uint32_t bb = b_addr + kc * (128 * 128) + k * 32;
          const uint32_t on = (kc | k) != 0 ? 1u : 0u;
          wgmma_m64n64(acc[0], da, make_desc_sw128(bb), on);
          wgmma_m64n64(acc[1], da, make_desc_sw128(bb + 64 * 128), on);
        }
      wgmma_commit();
      wgmma_wait<0>();
    }
    // ---- epilogue on the fragment: acc[s][4j + e] = row + 8*(e>>1), channel 64s + 8j + 2*(lane%4) + (e&1)
#pragma unroll
    for (int e2 = 0; e2 < 2; ++e2) {
      const int r = wg_row + (warp & 3) * 16 + (lane >> 2) + 8 * e2, py = r / kPX, px = r % kPX;
      const int y = yb * kPY + py, x = xb * kPX + px;
      if (y < h && x < w) {
        __half* dst = out + (((size_t)b * h + y) * w + x) * 128;
#pragma unroll
        for (int sub = 0; sub < 2; ++sub)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = 64 * sub + 8 * j + 2 * (lane & 3);
            *reinterpret_cast<__half2*>(dst + c) = __floats2half2_rn(fmaxf(acc[sub][4 * j + 2 * e2] + sb[c], 0.f),
                                                                     fmaxf(acc[sub][4 * j + 2 * e2 + 1] + sb[c + 1], 0.f));
          }
      }
    }
    __syncthreads();                                 // A tile and halo free for the next tile
  }
}

// GraphAgg's scatter_mean (src/droid_net.py:59): mean over the edges of each source frame, NHWC f16, fp32 sums in edge
// order (deterministic).  thread = (frame slot m, pixel, 8-channel chunk)
__global__ void __launch_bounds__(256)
scatter_mean_kernel(const __half* __restrict__ a1, const int* __restrict__ slot, __half* __restrict__ mean, int N, int M,
                    int hw) {
  const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
  const size_t total = (size_t)M * hw * 16;
  if (t >= total) return;
  const int c8 = (int)(t & 15);
  const size_t px = (t >> 4) % hw;
  const int m = (int)((t >> 4) / hw);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int cnt = 0;
  for (int e = 0; e < N; ++e) {
    if (__ldg(slot + e) != m) continue;
    ++cnt;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(a1 + ((size_t)e * hw + px) * 128 + c8 * 8));
    const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(hv[j]); acc[2 * j] += f.x; acc[2 * j + 1] += f.y; }
  }
  const float inv = cnt > 0 ? 1.0f / (float)cnt : 0.f;
  __half2 o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = __floats2half2_rn(acc[2 * j] * inv, acc[2 * j + 1] * inv);
  *reinterpret_cast<uint4*>(mean + ((size_t)m * hw + px) * 128 + c8 * 8) = *reinterpret_cast<const uint4*>(o);
}

// Tensor maps depend only on (base pointer, shape): the update operator runs the same layers on the same workspace
// buffers call after call, so the driver's encode (~1.5 us of host time each, ~50 per operator call) is cached.
struct CMapKey {
  const void* base; int a, b, c, d, kind;
  bool operator==(const CMapKey& o) const {
    return base == o.base && a == o.a && b == o.b && c == o.c && d == o.d && kind == o.kind;
  }
};
bool act_map_raw(GsEncodeTiled enc, const void* base, int B, int h, int w, int C, CUtensorMap* out);
bool weight_map_raw(GsEncodeTiled enc, const void* base, int taps, int N, int Cin, CUtensorMap* out, int n_tile);
bool encode_cmap(GsEncodeTiled enc, const CMapKey& k, CUtensorMap* out) {
  return k.kind == 0 ? act_map_raw(enc, k.base, k.a, k.b, k.c, k.d, out)
                     : weight_map_raw(enc, k.base, k.a, k.b, k.c, out, k.d);
}
GsTensorMapCache<CMapKey, 128, encode_cmap> g_cmaps;
bool act_map(const void* base, int B, int h, int w, int C, CUtensorMap* out) {
  return g_cmaps.get(CMapKey{base, B, h, w, C, 0}, out);
}
bool weight_map(const void* base, int taps, int N, int Cin, CUtensorMap* out, int n_tile = 0) {
  return g_cmaps.get(CMapKey{base, taps, N, Cin, n_tile, 1}, out);
}

// activation map: NHWC [B, h, w, C] as (ch, x, y, image), box 64 ch x 16 x 8
bool act_map_raw(GsEncodeTiled enc, const void* base, int B, int h, int w, int C, CUtensorMap* out) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)w * C * 2, (cuuint64_t)h * w * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)kKC, (cuuint32_t)kPX, (cuuint32_t)kPY, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// weight map: [taps, N, Cin] as (cin, cout, tap), box 64 x N
bool weight_map_raw(GsEncodeTiled enc, const void* base, int taps, int N, int Cin, CUtensorMap* out, int n_tile) {
  cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)N, (cuuint64_t)taps};
  cuuint64_t strides[2] = {(cuuint64_t)Cin * 2, (cuuint64_t)N * Cin * 2};
  cuuint32_t box[3] = {(cuuint32_t)kKC, (cuuint32_t)(n_tile > 0 ? n_tile : N), 1};
  cuuint32_t es[3] = {1, 1, 1};
  return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// one instantiation per output-channel tile width N = 16, 32, .., 256
template <int N>
int conv_setup(int) {
  GS_CUDA(cudaFuncSetAttribute(conv_tc_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemC));
  return GOSLAM_OK;
}
template <int N>
int conv_launch_n(const ConvMaps& maps, const ConvParams& p, int grid, cudaStream_t st) {
  const int rc = gs_device_setup<conv_setup<N>>();
  if (rc) return rc;
  conv_tc_kernel<N><<<grid, kThreadsC, kSmemC, st>>>(maps, p);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int conv_launch(const ConvMaps& maps, ConvParams p, cudaStream_t st) {
  int sms = 0;
  const int rc = gs_sm_count(&sms);
  if (rc) return rc;
  p.n_yb = gs_cdiv(p.h, kPY); p.n_xb = gs_cdiv(p.w, kPX);
  if (p.n_nt < 1) p.n_nt = 1;
  p.n_tiles = p.B * p.n_yb * p.n_xb * p.n_nt;
  const int grid = p.n_tiles < sms ? p.n_tiles : sms;
  switch (p.N) {
    case 16: return conv_launch_n<16>(maps, p, grid, st);
    case 32: return conv_launch_n<32>(maps, p, grid, st);
    case 48: return conv_launch_n<48>(maps, p, grid, st);
    case 64: return conv_launch_n<64>(maps, p, grid, st);
    case 80: return conv_launch_n<80>(maps, p, grid, st);
    case 96: return conv_launch_n<96>(maps, p, grid, st);
    case 112: return conv_launch_n<112>(maps, p, grid, st);
    case 128: return conv_launch_n<128>(maps, p, grid, st);
    case 144: return conv_launch_n<144>(maps, p, grid, st);
    case 160: return conv_launch_n<160>(maps, p, grid, st);
    case 176: return conv_launch_n<176>(maps, p, grid, st);
    case 192: return conv_launch_n<192>(maps, p, grid, st);
    case 208: return conv_launch_n<208>(maps, p, grid, st);
    case 224: return conv_launch_n<224>(maps, p, grid, st);
    case 240: return conv_launch_n<240>(maps, p, grid, st);
    case 256: return conv_launch_n<256>(maps, p, grid, st);
    default: return GOSLAM_EINVAL;
  }
}

int flow7x7_setup(int) {
  GS_CUDA(cudaFuncSetAttribute(flow7x7_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kF7Smem));
  return GOSLAM_OK;
}

struct GruWs {
  float* glo_sum;   // [B,128]
  float* glo;       // [B,384]
  __half* z;        // [B,h,w,128]
  __half* rnet;     // [B,h,w,128]
};
size_t gru_layout(int B, int h, int w, void* base, GruWs* ws) {
  if (B <= 0 || h <= 0 || w <= 0) return 256;   // what the size function has always reported for an invalid shape
  GsArena a(base);
  GruWs& g = *ws;
  g.glo_sum = a.take<float>((size_t)B * gs_cdiv(h, kPY) * gs_cdiv(w, kPX) * kConsumerWarps * 128);
  g.glo = a.take<float>((size_t)B * 384);
  g.z = a.take<__half>((size_t)B * h * w * 128);
  g.rnet = a.take<__half>((size_t)B * h * w * 128);
  // the reported size keeps 256 bytes of slack past the carve, which the entry point does not require
  return base ? a.off : a.off + 256;
}

}  // namespace

extern "C" {

int goslam_nchw_to_nhwc_f16(const void* src, void* dst, int B, int C, int hw, void* stream) {
  if (B < 0 || C <= 0 || hw <= 0) return GOSLAM_EINVAL;
  if (B == 0) return GOSLAM_OK;
  if (hw % 16 == 0 && C % 16 == 0) {
    nchw_to_nhwc64_kernel<<<dim3(gs_cdiv(hw, 64), gs_cdiv(C, 64), B), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __half*>(src), reinterpret_cast<__half*>(dst), C, C, hw);
    GS_CHECK_LAUNCH();
    return GOSLAM_OK;
  }
  dim3 grid(gs_cdiv(hw, 32), gs_cdiv(C, 32), B), block(32, 8);
  transpose_f16_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(src),
                                                                  reinterpret_cast<__half*>(dst), C, hw);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_nhwc_to_nchw_f16(const void* src, void* dst, int B, int C, int hw, void* stream) {
  if (B < 0 || C <= 0 || hw <= 0) return GOSLAM_EINVAL;
  if (B == 0) return GOSLAM_OK;
  if (hw % 16 == 0 && C % 64 == 0) {
    nhwc_to_nchw64_kernel<<<dim3(C / 64, gs_cdiv(hw, 64), B), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __half*>(src), reinterpret_cast<__half*>(dst), C, hw);
    GS_CHECK_LAUNCH();
    return GOSLAM_OK;
  }
  dim3 grid(gs_cdiv(C, 32), gs_cdiv(hw, 32), B), block(32, 8);
  transpose_f16_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(src),
                                                                  reinterpret_cast<__half*>(dst), hw, C);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

int goslam_conv2d_nhwc(const goslam_conv_desc* d, int B, int h, int w, void* stream) {
  if (!d || B < 0 || h <= 0 || w <= 0 || d->n_in < 1 || d->n_in > kMaxIn) return GOSLAM_EINVAL;
  if ((d->taps != 1 && d->taps != 9) || d->cout < 1 || d->cout_pad < d->cout || d->cout_pad % 16) return GOSLAM_EINVAL;
  const int N = d->cout_pad <= kMaxN ? d->cout_pad : (d->cout_pad % 192 == 0 ? 192 : (d->cout_pad % 256 == 0 ? 256 : 128));
  // the epilogue stages the whole bias vector in shared memory
  if (d->cout_pad % N || d->cout_pad > kVecMax) return GOSLAM_EINVAL;
  if (B == 0) return GOSLAM_OK;
  ConvMaps m{};
  ConvParams p{};
  p.B = B; p.h = h; p.w = w; p.taps = d->taps; p.n_in = d->n_in; p.N = N; p.n_nt = d->cout_pad / N;
  int cin_total = 0;
  for (int i = 0; i < d->n_in; ++i) {
    if (d->cin[i] <= 0 || d->cin[i] % kKC || d->cin_off[i] % kKC || d->cin_stride[i] < d->cin_off[i] + d->cin[i]) return GOSLAM_EINVAL;
    p.chunks[i] = d->cin[i] / kKC; p.coff[i] = d->cin_off[i];
    cin_total += d->cin[i];
    if (!act_map(d->in[i], B, h, w, d->cin_stride[i], &m.in[i])) return GOSLAM_ELAUNCH;
  }
  if (!weight_map(d->weight, d->taps, d->cout_pad, cin_total, &m.w, N)) return GOSLAM_ELAUNCH;
  p.epi = EPI_ACT; p.bias = d->bias; p.act = d->act; p.cout = d->cout; p.out = d->out; p.out_f32 = d->out_f32;
  p.out_stride = d->out_stride; p.out_offset = d->out_offset; p.out_scale = d->out_scale;
  p.split = d->split; p.act2 = d->act2; p.out2 = d->out2;
  if (d->split > 0 && (!d->out_f32 || !d->out2 || d->cout > 8)) return GOSLAM_EINVAL;
  if (!d->out_f32 && ((d->out_stride % 8) || (d->out_offset % 8))) return GOSLAM_EINVAL;
  return conv_launch(m, p, (cudaStream_t)stream);
}

int goslam_nchw_to_nhwc_f16_pad(const void* src, void* dst, int B, int C, int Cpad, int hw, void* stream) {
  if (B < 0 || C <= 0 || Cpad < C || hw <= 0) return GOSLAM_EINVAL;
  if (B == 0) return GOSLAM_OK;
  if (hw % 16 == 0 && Cpad % 16 == 0 && hw % 8 == 0) {
    nchw_to_nhwc64_kernel<<<dim3(gs_cdiv(hw, 64), gs_cdiv(Cpad, 64), B), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __half*>(src), reinterpret_cast<__half*>(dst), C, Cpad, hw);
    GS_CHECK_LAUNCH();
    return GOSLAM_OK;
  }
  dim3 grid(gs_cdiv(hw, 32), gs_cdiv(Cpad, 32), B), block(32, 8);
  transpose_pad_f16_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(src),
                                                                      reinterpret_cast<__half*>(dst), C, Cpad, hw);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}

size_t goslam_conv_gru_workspace_bytes(int B, int h, int w) {
  GruWs ws;
  return gru_layout(B, h, w, nullptr, &ws);
}

// ------------------------------------------------------------------------------------------------------
// The whole update operator in one call (UpdateModule.forward, src/droid_net.py:107-140): layout conversion of the
// reference-shaped inputs, encoders, ConvGRU, heads, GraphAgg — ~20 launches issued from here, tensor maps cached.
// ------------------------------------------------------------------------------------------------------
struct OpWs {
  __half *corr256, *c1, *c2, *f1, *f2, *net, *inp, *state, *hid, *a1, *mean, *a2, *up;
  void* gru;
  size_t gru_bytes;
};
static size_t op_layout(int N, int M, int h, int w, void* base, OpWs* out) {
  if (N <= 0 || h <= 0 || w <= 0) return 256;   // what the size function has always reported for an invalid shape
  GsArena a(base);
  OpWs& o = *out;
  const size_t px = (size_t)N * h * w, pm = (size_t)(M > 0 ? M : 1) * h * w;
  o.corr256 = a.take<__half>(px * 256); o.c1 = a.take<__half>(px * 128); o.c2 = a.take<__half>(px * 128);
  o.f1 = a.take<__half>(px * 128); o.f2 = a.take<__half>(px * 64);
  o.net = a.take<__half>(px * 128); o.inp = a.take<__half>(px * 128); o.state = a.take<__half>(px * 128);
  o.hid = a.take<__half>(px * 256); o.a1 = a.take<__half>(px * 128);
  o.mean = a.take<__half>(pm * 128); o.a2 = a.take<__half>(pm * 128); o.up = a.take<__half>(pm * 576);
  GruWs gru;
  o.gru_bytes = gru_layout(N, h, w, nullptr, &gru);   // the GRU's reported size, slack included
  o.gru = a.take<char>(o.gru_bytes);
  // the reported size keeps 256 bytes of slack past the carve, which the entry point does not require
  return base ? a.off : a.off + 256;
}

static int layer(const void* in, int cin, int cin_off, int cin_stride, const void* wgt, const float* bias, int taps, int cout,
          int cout_pad, int act, float scale, void* out, int out_f32, int out_stride, int B, int h, int w, void* stream) {
  goslam_conv_desc d{};
  d.in[0] = in; d.cin[0] = cin; d.cin_off[0] = cin_off; d.cin_stride[0] = cin_stride; d.n_in = 1;
  d.weight = wgt; d.bias = bias; d.taps = taps; d.cout = cout; d.cout_pad = cout_pad; d.act = act; d.out_scale = scale;
  d.out = out; d.out_f32 = out_f32; d.out_stride = out_stride; d.out_offset = 0;
  return goslam_conv2d_nhwc(&d, B, h, w, stream);
}

size_t goslam_update_op_workspace_bytes(int N, int M, int h, int w) {
  OpWs ws;
  return op_layout(N, M, h, w, nullptr, &ws);
}

int goslam_update_op(const goslam_update_weights* W, const void* net, const void* inp, const void* corr,
                     const float* flow, const int* frame_slot, int N, int M, int h, int w, void* net_out,
                     float* delta, float* weight, float* eta, void* upmask, void* workspace,
                     size_t workspace_bytes, void* stream) {
  if (!W || N < 0 || h <= 0 || w <= 0 || (frame_slot && M <= 0)) return GOSLAM_EINVAL;
  if (N == 0) return GOSLAM_OK;
  OpWs ws;
  if (!workspace || workspace_bytes < op_layout(N, frame_slot ? M : 0, h, w, workspace, &ws)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int hw = h * w;
  int rc;
#define GS_TRY(x) do { rc = (x); if (rc) return rc; } while (0)
  // ---- reference-shaped inputs ([N,C,h,w]) -> NHWC f16
  GS_TRY(goslam_nchw_to_nhwc_f16_pad(corr, ws.corr256, N, 196, 256, hw, stream));
  GS_TRY(goslam_nchw_to_nhwc_f16(net, ws.net, N, 128, hw, stream));
  GS_TRY(goslam_nchw_to_nhwc_f16(inp, ws.inp, N, 128, hw, stream));
  // ---- encoders (src/droid_net.py:76-88)
  GS_TRY(layer(ws.corr256, 256, 0, 256, W->corr0_w, W->corr0_b, 1, 128, 128, ACT_RELU, 1.f, ws.c1, 0, 128, N, h, w, stream));
  GS_TRY(layer(ws.c1, 128, 0, 128, W->corr2_w, W->corr2_b, 9, 128, 128, ACT_RELU, 1.f, ws.c2, 0, 128, N, h, w, stream));
  {
    // 7x7 motion encoder: im2col + wgmma (flow0_w f16 [128][256], K = (ky*7+kx)*4 + ci, zero beyond 196)
    CUtensorMap wm;
    if (!weight_map(W->flow0_w, 1, 128, kF7K, &wm, 128)) return GOSLAM_ELAUNCH;
    int sms = 0;
    rc = gs_device_setup<flow7x7_setup>();
    if (rc == GOSLAM_OK) rc = gs_sm_count(&sms);
    if (rc) return rc;
    const int n_tiles = N * gs_cdiv(h, kPY) * gs_cdiv(w, kPX);
    flow7x7_tc_kernel<<<n_tiles < sms ? n_tiles : sms, kF7Threads, kF7Smem, st>>>(wm, flow, W->flow0_b, ws.f1, N, h, w);
    GS_CHECK_LAUNCH();
  }
  GS_TRY(layer(ws.f1, 128, 0, 128, W->flow2_w, W->flow2_b, 9, 64, 64, ACT_RELU, 1.f, ws.f2, 0, 64, N, h, w, stream));
  // ---- ConvGRU
  GS_TRY(goslam_conv_gru(&W->gru, ws.net, ws.inp, ws.c2, ws.f2, ws.state, N, h, w, ws.gru, ws.gru_bytes, stream));
  // ---- heads: delta.0 | weight.0 stacked (shared input), then the two 2-channel heads on their halves, fp32 out
  GS_TRY(layer(ws.state, 128, 0, 128, W->hid_w, W->hid_b, 9, 256, 256, ACT_RELU, 1.f, ws.hid, 0, 256, N, h, w, stream));
  {
    // delta.2 and weight.2 in ONE pass over the 256 hidden channels with block-diagonal weights
    // (heads_w [9][16][256]: row 0-1 = delta.2 on channels 0..127, rows 2-3 = weight.2 on channels 128..255)
    goslam_conv_desc d{};
    d.in[0] = ws.hid; d.cin[0] = 256; d.cin_off[0] = 0; d.cin_stride[0] = 256; d.n_in = 1;
    d.weight = W->delta_w; d.bias = W->delta_b; d.taps = 9; d.cout = 4; d.cout_pad = 16; d.act = ACT_NONE; d.out_scale = 1.f;
    d.out = delta; d.out_f32 = 1; d.out_stride = 2; d.out_offset = 0; d.split = 2; d.act2 = ACT_SIGMOID; d.out2 = weight;
    GS_TRY(goslam_conv2d_nhwc(&d, N, h, w, stream));
  }
  GS_TRY(goslam_nhwc_to_nchw_f16(ws.state, net_out, N, 128, hw, stream));
  if (!frame_slot) return GOSLAM_OK;
  // ---- GraphAgg (src/droid_net.py:51-67)
  GS_TRY(layer(ws.state, 128, 0, 128, W->agg1_w, W->agg1_b, 9, 128, 128, ACT_RELU, 1.f, ws.a1, 0, 128, N, h, w, stream));
  {
    const size_t total = (size_t)M * hw * 16;
    scatter_mean_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ws.a1, frame_slot, ws.mean, N, M, hw);
    GS_CHECK_LAUNCH();
  }
  GS_TRY(layer(ws.mean, 128, 0, 128, W->agg2_w, W->agg2_b, 9, 128, 128, ACT_RELU, 1.f, ws.a2, 0, 128, M, h, w, stream));
  GS_TRY(layer(ws.a2, 128, 0, 128, W->eta_w, W->eta_b, 9, 1, 16, ACT_SOFTPLUS, 0.01f, eta, 1, 1, M, h, w, stream));
  GS_TRY(layer(ws.a2, 128, 0, 128, W->upmask_w, W->upmask_b, 1, 576, 576, ACT_NONE, 1.f, ws.up, 0, 576, M, h, w, stream));
  GS_TRY(goslam_nhwc_to_nchw_f16(ws.up, upmask, M, 576, hw, stream));
#undef GS_TRY
  return GOSLAM_OK;
}

int goslam_conv_gru(const goslam_gru_weights* wts, const void* net, const void* inp, const void* corr,
                    const void* flow, void* net_out, int B, int h, int w, void* workspace,
                    size_t workspace_bytes, void* stream) {
  if (!wts || B < 0 || h <= 0 || w <= 0) return GOSLAM_EINVAL;
  if (B == 0) return GOSLAM_OK;
  GruWs ws;
  if (!workspace || workspace_bytes < gru_layout(B, h, w, workspace, &ws)) return GOSLAM_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  ConvMaps m{};
  ConvParams p{};
  p.B = B; p.h = h; p.w = w;
  p.net = reinterpret_cast<const __half*>(net);
  // ---- pass G: glo_sum = sum_px sigmoid(w(net)) * net
  if (!act_map(net, B, h, w, 128, &m.in[0]) || !weight_map(wts->w_w, 1, 128, 128, &m.w)) return GOSLAM_ELAUNCH;
  p.n_nt = 1;
  p.taps = 1; p.n_in = 1; p.chunks[0] = 2; p.N = 128; p.epi = EPI_GLO; p.bias = wts->b_w; p.glo = nullptr;
  p.glo_sum = ws.glo_sum;
  int rc = conv_launch(m, p, st);
  if (rc) return rc;
  gru_glo_fc_kernel<<<B, 256, 0, st>>>(ws.glo_sum, gs_cdiv(h, kPY) * gs_cdiv(w, kPX) * kConsumerWarps, wts->w_glo, wts->b_glo, ws.glo,
                                       1.0f / (float)(h * w));
  GS_CHECK_LAUNCH();
  // ---- pass ZR: z, r*net
  if (!act_map(inp, B, h, w, 128, &m.in[1]) || !act_map(corr, B, h, w, 128, &m.in[2]) ||
      !act_map(flow, B, h, w, 64, &m.in[3]) || !weight_map(wts->w_zr, 9, 256, 448, &m.w))
    return GOSLAM_ELAUNCH;
  p.taps = 9; p.n_in = 4; p.chunks[0] = 2; p.chunks[1] = 2; p.chunks[2] = 2; p.chunks[3] = 1;
  p.N = 256; p.epi = EPI_ZR; p.bias = wts->b_zr; p.glo = ws.glo; p.z_out = ws.z; p.rnet_out = ws.rnet;
  rc = conv_launch(m, p, st);
  if (rc) return rc;
  // ---- pass Q: net' = (1 - z) net + z tanh(convq([r*net | inp | corr | flow]) + glo_q)
  if (!act_map(ws.rnet, B, h, w, 128, &m.in[0]) || !weight_map(wts->w_q, 9, 128, 448, &m.w)) return GOSLAM_ELAUNCH;
  p.N = 128; p.epi = EPI_Q; p.bias = wts->b_q; p.z_in = ws.z; p.net_out = reinterpret_cast<__half*>(net_out);
  return conv_launch(m, p, st);
}

}  // extern "C"
