// encoder.cu — DroidNet's BasicEncoder forward (src/modules/extractor.py) for norm_fn 'instance' (fnet) and 'none'
// (cnet), sm_90a.
//
// Activations live in the workspace as NHWC f16; every convolution is one tensor-core implicit GEMM (mma.sync
// m16n8k16, f32 accumulation) over 64-pixel x BN-channel tiles of one image:
//   stem     7x7 s2, 3 -> 32, reads the NCHW image (f32 or f16), optional (x - mean[c]) / std[c] in f32 then f16
//   blocks   3x3 (s1 or s2) conv1 / conv2 and the 1x1 s2 downsample
//   out      1x1 128 -> out_dim with bias, written NCHW f16; optionally tanh of channels 0-127 / relu of 128-255
// Instance norm (biased variance, eps 1e-5): a conv's epilogue writes its f16 output and, per tile, the mean and M2 of
// each channel over the tile's pixels (computed from the f16 values).  A merge kernel folds the tiles in a fixed order
// (Chan's update, no atomics) into (mean, rstd) per (image, channel).  The next conv applies (x - mean) * rstd and the
// ReLU while it loads its operands; a residual block's tail is one elementwise pass relu(relu(n2(y)) + n3(x)).
// With norm 'none' the tail folds into conv2's epilogue: bias, relu, residual add, relu.
#include "common.cuh"

namespace {

constexpr int kBM = 64;               // output pixels per tile
constexpr int kBK = 32;               // K per stage
constexpr int kLds = kBK + 8;         // smem row stride in halfs (80 bytes: ldmatrix rows hit distinct banks)
constexpr int kThreads = 128;         // 4 warps, 2 (M) x 2 (N)
constexpr int kStemK = 147;           // 7 * 7 * 3
constexpr int kStemKpad = 160;
constexpr int kDims[6] = {32, 32, 64, 64, 128, 128};   // output channels of layer1.0 .. layer3.1
constexpr int kMaxC = 128;

struct ConvArgs {
  const __half* in;        // NHWC [B][Hi][Wi][Cin]
  const void* image;       // stem only: NCHW [B][3][Hi][Wi]
  int image_f16;
  const float* mean;       // stem only: [3] or null
  const float* stdv;
  const float* in_stats;   // [B][Cin][2] (mean, rstd) applied to `in` on load, or null
  int in_relu;             // ReLU after the input normalisation
  const __half* w;         // [Cout][Kpad]
  const float* bias;       // [Cout]
  int Hi, Wi, Cin, Ho, Wo, Cout, ksize, stride, pad, Kpad;
  int relu;                // epilogue ReLU (norm 'none')
  const __half* res;       // norm 'none' conv2: out = relu(relu(v) + res), res NHWC [B][Ho][Wo][Cout]
  __half* out;             // NHWC [B][Ho][Wo][Cout], or null when writing NCHW
  float* part;             // [B][tiles][Cout][2] per-tile (mean, M2), or null
  __half* out_nchw;        // final conv: NCHW [B][Cout][Ho][Wo] (split: channels 0-127)
  __half* out2_nchw;       // split: channels 128-255 as [B][128][Ho][Wo]
  int split;
};

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// one 16-byte operand vector (8 channels) of the input, normalised on load
__device__ __forceinline__ uint4 xform8(uint4 v, const float* s_stats, int c0, bool relu) {
  __half* h = reinterpret_cast<__half*>(&v);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float x = (__half2float(h[j]) - s_stats[2 * (c0 + j)]) * s_stats[2 * (c0 + j) + 1];
    if (relu) x = fmaxf(x, 0.0f);
    h[j] = __float2half_rn(x);
  }
  return v;
}

template <int BN>
struct Smem {
  static constexpr int kStage = (kBM + BN) * kLds;                 // halfs per stage
  static constexpr int kOut = kBM * (BN + 8);                       // epilogue tile, halfs
  static constexpr int kHalfs = (2 * kStage > kOut) ? 2 * kStage : kOut;
};

template <int BN, bool STEM>
__global__ void __launch_bounds__(kThreads) encoder_conv_kernel(const ConvArgs a) {
  __shared__ __align__(16) __half smem[Smem<BN>::kHalfs];
  __shared__ float s_stats[2 * kMaxC];
  __shared__ float s_bias[BN];
  constexpr int kStage = Smem<BN>::kStage;
  constexpr int NT = BN / 16;                 // n8 tiles per warp (warp covers BN / 2 channels)
  const int tile = blockIdx.x, b = blockIdx.y, n0 = blockIdx.z * BN;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int HWo = a.Ho * a.Wo, m0 = tile * kBM;
  const bool xf = !STEM && a.in_stats != nullptr;

  if (xf)
    for (int i = tid; i < 2 * a.Cin; i += kThreads) s_stats[i] = a.in_stats[(size_t)b * 2 * a.Cin + i];
  for (int i = tid; i < BN; i += kThreads) s_bias[i] = a.bias[n0 + i];

  // ---- operand staging -------------------------------------------------------------------------------------------
  // non-stem A: 256 vectors of 8 channels per stage, thread t loads rows (t >> 2) and (t >> 2) + 32, segment t & 3
  int row_oy[2], row_ox[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = m0 + (tid >> 2) + 32 * i;
    row_oy[i] = m < HWo ? m / a.Wo : -(1 << 20);
    row_ox[i] = m < HWo ? m - (m / a.Wo) * a.Wo : 0;
  }
  const int cpt = STEM ? 1 : a.Cin / kBK;     // stages per tap
  const int nk = a.Kpad / kBK;
  constexpr int kBVec = BN * 4 / kThreads;    // weight vectors per thread per stage
  uint4 ra[STEM ? 1 : 2], rb[kBVec];
  __half rs[STEM ? 16 : 1];

  auto load_stage = [&](int q) {
    if constexpr (STEM) {
      // each thread owns k column (lane) of rows warp + 4 i
      const int k = q * kBK + lane;
      const bool kval = k < kStemK;
      const int tap = kval ? k / 3 : 0, c = kval ? k - 3 * (k / 3) : 0;
      const int ky = tap / 7, kx = tap - 7 * (tap / 7);
      const float mu = a.mean ? a.mean[c] : 0.0f, sd = a.mean ? a.stdv[c] : 1.0f;
      const size_t plane = (size_t)a.Hi * a.Wi;
      const size_t base = ((size_t)b * 3 + c) * plane;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int m = m0 + warp + 4 * i;
        float v = 0.0f;
        if (kval && m < HWo) {
          const int oy = m / a.Wo, ox = m - oy * a.Wo;
          const int iy = oy * 2 - 3 + ky, ix = ox * 2 - 3 + kx;
          if (iy >= 0 && iy < a.Hi && ix >= 0 && ix < a.Wi) {
            const size_t off = base + (size_t)iy * a.Wi + ix;
            if (a.image_f16) {
              v = __half2float(reinterpret_cast<const __half*>(a.image)[off]);
              // the in-place sub_ / div_ on an f16 tensor rounds after each op
              if (a.mean) v = __half2float(__float2half_rn(__fdiv_rn(__half2float(__float2half_rn(__fsub_rn(v, mu))), sd)));
            } else {
              v = reinterpret_cast<const float*>(a.image)[off];
              if (a.mean) v = __fdiv_rn(__fsub_rn(v, mu), sd);
            }
          }
        }
        rs[i] = __float2half_rn(v);
      }
    } else {
      const int tap = q / cpt, c0 = (q - tap * cpt) * kBK + (tid & 3) * 8;
      const int ky = tap / a.ksize, kx = tap - ky * a.ksize;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int iy = row_oy[i] * a.stride - a.pad + ky, ix = row_ox[i] * a.stride - a.pad + kx;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (iy >= 0 && iy < a.Hi && ix >= 0 && ix < a.Wi) {
          v = __ldg(reinterpret_cast<const uint4*>(a.in + (((size_t)b * a.Hi + iy) * a.Wi + ix) * a.Cin + c0));
          if (xf) v = xform8(v, s_stats, c0, a.in_relu);
        }
        ra[i] = v;
      }
    }
#pragma unroll
    for (int i = 0; i < kBVec; ++i) {
      const int v = tid + i * kThreads, r = v >> 2, s = v & 3;
      rb[i] = __ldg(reinterpret_cast<const uint4*>(a.w + (size_t)(n0 + r) * a.Kpad + q * kBK + s * 8));
    }
  };
  auto store_stage = [&](int buf) {
    __half* sA = smem + buf * kStage;
    __half* sB = sA + kBM * kLds;
    if constexpr (STEM) {
#pragma unroll
      for (int i = 0; i < 16; ++i) sA[(warp + 4 * i) * kLds + lane] = rs[i];
    } else {
#pragma unroll
      for (int i = 0; i < 2; ++i)
        *reinterpret_cast<uint4*>(sA + ((tid >> 2) + 32 * i) * kLds + (tid & 3) * 8) = ra[i];
    }
#pragma unroll
    for (int i = 0; i < kBVec; ++i) {
      const int v = tid + i * kThreads;
      *reinterpret_cast<uint4*>(sB + (v >> 2) * kLds + (v & 3) * 8) = rb[i];
    }
  };

  float acc[2][NT][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0f;

  const int wm = warp >> 1, wn = warp & 1;
  __syncthreads();                               // s_stats before the first transformed load
  load_stage(0);
  store_stage(0);
  __syncthreads();
  for (int q = 0; q < nk; ++q) {
    const int buf = q & 1;
    if (q + 1 < nk) load_stage(q + 1);
    const __half* sA = smem + buf * kStage;
    const __half* sB = sA + kBM * kLds;
#pragma unroll
    for (int kk = 0; kk < kBK; kk += 16) {
      uint32_t af[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i)
        ldmatrix_x4(af[i], smem_addr(sA + (wm * 32 + i * 16 + (lane & 15)) * kLds + kk + (lane >> 4) * 8));
#pragma unroll
      for (int j = 0; j < NT; j += 2) {
        uint32_t bf[4];
        const int n = wn * (BN / 2) + j * 8 + (lane & 7) + ((lane >> 4) << 3);
        ldmatrix_x4(bf, smem_addr(sB + n * kLds + kk + ((lane >> 3) & 1) * 8));
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          mma_16816(acc[i][j], af[i], bf[0], bf[1]);
          mma_16816(acc[i][j + 1], af[i], bf[2], bf[3]);
        }
      }
    }
    if (q + 1 < nk) store_stage(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue: bias (+ relu / residual), f16 tile in shared memory -----------------------------------------------
  constexpr int kOs = BN + 8;
  __half* sC = smem;                             // the stages are dead after the last barrier
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = wm * 32 + i * 16 + (lane >> 2) + 8 * h;
        const int c = wn * (BN / 2) + j * 8 + (lane & 3) * 2;
        __half v0 = __float2half_rn(acc[i][j][2 * h] + s_bias[c]);
        __half v1 = __float2half_rn(acc[i][j][2 * h + 1] + s_bias[c + 1]);
        if (a.relu) {
          v0 = __hmax(v0, __float2half(0.0f));
          v1 = __hmax(v1, __float2half(0.0f));
        }
        if (a.res != nullptr && m0 + r < HWo) {
          const __half2 x = *reinterpret_cast<const __half2*>(a.res + ((size_t)b * HWo + m0 + r) * a.Cout + n0 + c);
          v0 = __float2half_rn(fmaxf(__half2float(v0) + __half2float(x.x), 0.0f));
          v1 = __float2half_rn(fmaxf(__half2float(v1) + __half2float(x.y), 0.0f));
        }
        *reinterpret_cast<__half2*>(sC + r * kOs + c) = __halves2half2(v0, v1);
      }
  __syncthreads();
  const int rows = min(kBM, HWo - m0);
  if (a.part != nullptr && tid < BN) {
    // per-channel tile statistics of the f16 values, two passes over the tile
    float s = 0.0f;
    for (int r = 0; r < rows; ++r) s += __half2float(sC[r * kOs + tid]);
    const float mean = s / (float)rows;
    float m2 = 0.0f;
    for (int r = 0; r < rows; ++r) {
      const float d = __half2float(sC[r * kOs + tid]) - mean;
      m2 = fmaf(d, d, m2);
    }
    float* p = a.part + (((size_t)b * gridDim.x + tile) * a.Cout + n0 + tid) * 2;
    p[0] = mean;
    p[1] = m2;
  }
  if (a.out != nullptr) {
    constexpr int kVec = BN / 8;
    for (int v = tid; v < rows * kVec; v += kThreads) {
      const int r = v / kVec, s = v - r * kVec;
      *reinterpret_cast<uint4*>(a.out + ((size_t)b * HWo + m0 + r) * a.Cout + n0 + s * 8) =
          *reinterpret_cast<const uint4*>(sC + r * kOs + s * 8);
    }
  } else {
    for (int v = tid; v < kBM * BN; v += kThreads) {
      const int c = v / kBM, r = v - c * kBM, n = n0 + c;
      if (r >= rows) continue;
      const __half x = sC[r * kOs + c];
      if (!a.split) {
        a.out_nchw[((size_t)b * a.Cout + n) * HWo + m0 + r] = x;
      } else if (n < 128) {
        a.out_nchw[((size_t)b * 128 + n) * HWo + m0 + r] = __float2half_rn(tanhf(__half2float(x)));
      } else {
        a.out2_nchw[((size_t)b * 128 + n - 128) * HWo + m0 + r] = __float2half_rn(fmaxf(__half2float(x), 0.0f));
      }
    }
  }
}

// Chan's update: fold (nb, mb, Mb) into (n, mean, m2)
__device__ __forceinline__ void chan_merge(float& n, float& mean, float& m2, float nb, float mb, float Mb) {
  const float tot = n + nb;
  if (nb == 0.0f || tot == 0.0f) return;
  const float d = mb - mean;
  mean += d * (nb / tot);
  m2 += Mb + d * d * (n * nb / tot);
  n = tot;
}

// one warp per (image, channel): lane l folds tiles l, l + 32, ... in order, then a fixed shuffle tree -> (mean, rstd)
__global__ void encoder_stats_kernel(const float* __restrict__ part, int B, int C, int HW, int tiles,
                                     float* __restrict__ stats) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  float n = 0.0f, mean = 0.0f, m2 = 0.0f;
  for (int t = lane; t < tiles; t += 32) {
    const float2 p = __ldg(reinterpret_cast<const float2*>(part + (((size_t)b * tiles + t) * C + c) * 2));
    chan_merge(n, mean, m2, (float)min(kBM, HW - t * kBM), p.x, p.y);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float nb = __shfl_down_sync(0xffffffffu, n, o), mb = __shfl_down_sync(0xffffffffu, mean, o),
                Mb = __shfl_down_sync(0xffffffffu, m2, o);
    chan_merge(n, mean, m2, nb, mb, Mb);
  }
  if (lane == 0) {
    stats[2 * i] = mean;
    stats[2 * i + 1] = 1.0f / sqrtf(m2 / (float)HW + 1e-5f);
  }
}

// residual block tail (instance norm): out = relu(relu((y - m2) r2) + x'), x' = (x - m3) r3 [relu] or x
__global__ void encoder_tail_kernel(const __half* __restrict__ y, const float* __restrict__ s2, const __half* __restrict__ x,
                                    const float* __restrict__ s3, int x_relu, int B, int HW, int C,
                                    __half* __restrict__ out) {
  const size_t nvec = (size_t)B * HW * C / 8;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  const int cv = C / 8;
  const int c0 = (int)(i % cv) * 8;
  const int b = (int)(i / ((size_t)HW * cv));
  uint4 yv = __ldg(reinterpret_cast<const uint4*>(y) + i), xv = __ldg(reinterpret_cast<const uint4*>(x) + i), ov;
  const __half *yh = reinterpret_cast<const __half*>(&yv), *xh = reinterpret_cast<const __half*>(&xv);
  __half* oh = reinterpret_cast<__half*>(&ov);
  const float* t2 = s2 + ((size_t)b * C + c0) * 2;
  const float* t3 = s3 ? s3 + ((size_t)b * C + c0) * 2 : nullptr;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float yn = fmaxf((__half2float(yh[j]) - t2[2 * j]) * t2[2 * j + 1], 0.0f);
    float xn = __half2float(xh[j]);
    if (t3) xn = (xn - t3[2 * j]) * t3[2 * j + 1];
    if (x_relu) xn = fmaxf(xn, 0.0f);
    oh[j] = __float2half_rn(fmaxf(yn + xn, 0.0f));
  }
  reinterpret_cast<uint4*>(out)[i] = ov;
}

// ---- host side --------------------------------------------------------------------------------------------------

struct Layout {
  __half* act[4];
  float* part[3];
  float* stats[4];
};

int tiles_of(int hw) { return gs_cdiv(hw, kBM); }

bool shape_ok(int B, int H, int W) {
  return B >= 1 && B <= 65535 && H >= 8 && W >= 8 && H % 8 == 0 && W % 8 == 0 && (long long)H * W <= (1LL << 24) &&
         (long long)B * H * W * 8 < (1LL << 40);
}

size_t encoder_layout(int B, int H, int W, int norm, void* base, Layout* L) {
  const size_t act = (size_t)B * (H / 2) * (W / 2) * 32;     // the largest activation (stem / layer1)
  size_t part = 0;
  const int hw[3] = {(H / 2) * (W / 2), (H / 4) * (W / 4), (H / 8) * (W / 8)};
  for (int l = 0; l < 3; ++l) part = part > (size_t)tiles_of(hw[l]) * (32 << l) ? part : (size_t)tiles_of(hw[l]) * (32 << l);
  part *= (size_t)B * 2;
  GsArena ar(base);
  for (int i = 0; i < 4; ++i) L->act[i] = ar.take<__half>(act);
  for (int i = 0; i < 3; ++i) L->part[i] = norm ? ar.take<float>(part) : nullptr;
  for (int i = 0; i < 4; ++i) L->stats[i] = norm ? ar.take<float>((size_t)B * kMaxC * 2) : nullptr;
  return ar.off;
}

ConvArgs conv_args(const goslam_encoder_conv& cw, const __half* in, int Hi, int Wi, int Cin, int Cout, int ksize,
                   int stride) {
  ConvArgs a = {};
  a.in = in;
  a.w = (const __half*)cw.w;
  a.bias = cw.b;
  a.Hi = Hi; a.Wi = Wi; a.Cin = Cin; a.Cout = Cout; a.ksize = ksize; a.stride = stride;
  a.pad = ksize / 2;
  a.Ho = (Hi + 2 * a.pad - ksize) / stride + 1;
  a.Wo = (Wi + 2 * a.pad - ksize) / stride + 1;
  a.Kpad = ksize * ksize * Cin;
  return a;
}

template <int BN, bool STEM>
void launch_bn(const ConvArgs& a, int B, cudaStream_t s) {
  dim3 grid(tiles_of(a.Ho * a.Wo), B, a.Cout / BN);
  encoder_conv_kernel<BN, STEM><<<grid, kThreads, 0, s>>>(a);
}

void launch_conv(const ConvArgs& a, int B, cudaStream_t s) {
  if (a.Cout % 128 == 0) launch_bn<128, false>(a, B, s);
  else if (a.Cout % 64 == 0) launch_bn<64, false>(a, B, s);
  else launch_bn<32, false>(a, B, s);
}

void launch_stats(const ConvArgs& a, int B, float* stats, cudaStream_t s) {
  const int n = B * a.Cout;   // one warp each, 4 per block
  encoder_stats_kernel<<<gs_cdiv(n, 4), 128, 0, s>>>(a.part, B, a.Cout, a.Ho * a.Wo, tiles_of(a.Ho * a.Wo), stats);
}

bool conv_ok(const goslam_encoder_conv& c) { return c.w != nullptr && c.b != nullptr; }

}  // namespace

extern "C" size_t goslam_encoder_workspace_bytes(int B, int H, int W, int norm) {
  if (!shape_ok(B, H, W) || (norm != GOSLAM_NORM_NONE && norm != GOSLAM_NORM_INSTANCE)) return 0;
  Layout L;
  return encoder_layout(B, H, W, norm, nullptr, &L);
}

extern "C" int goslam_basic_encoder(const goslam_encoder_weights* wt, int norm, int out_dim, const void* image,
                                    int image_is_f16, const float* mean, const float* stdv, int B, int H, int W, void* out,
                                    void* out2, int split, void* workspace, size_t workspace_bytes, void* stream) {
  if (wt == nullptr || !shape_ok(B, H, W) || (norm != GOSLAM_NORM_NONE && norm != GOSLAM_NORM_INSTANCE))
    return GOSLAM_EINVAL;
  if (out_dim <= 0 || out_dim % 32 != 0 || (split && (out_dim != 256 || out2 == nullptr)) || image == nullptr ||
      out == nullptr || (mean == nullptr) != (stdv == nullptr))
    return GOSLAM_EINVAL;
  if (!conv_ok(wt->stem) || !conv_ok(wt->out)) return GOSLAM_EINVAL;
  for (int i = 0; i < 6; ++i) {
    if (!conv_ok(wt->block[i][0]) || !conv_ok(wt->block[i][1])) return GOSLAM_EINVAL;
    if ((i == 2 || i == 4) && !conv_ok(wt->block[i][2])) return GOSLAM_EINVAL;
  }
  Layout L;
  if (!workspace || workspace_bytes < encoder_layout(B, H, W, norm, workspace, &L)) return GOSLAM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  const bool inst = norm == GOSLAM_NORM_INSTANCE;

  // stem
  ConvArgs st = conv_args(wt->stem, nullptr, H, W, 3, 32, 7, 2);
  st.image = image; st.image_f16 = image_is_f16; st.mean = mean; st.stdv = stdv;
  st.Kpad = kStemKpad;
  st.out = L.act[0];
  st.relu = !inst;
  st.part = inst ? L.part[0] : nullptr;
  launch_bn<32, true>(st, B, s);
  GS_CHECK_LAUNCH();
  if (inst) { launch_stats(st, B, L.stats[0], s); GS_CHECK_LAUNCH(); }

  int x = 0, Hi = st.Ho, Wi = st.Wo, Cin = 32;
  const float* xs = inst ? L.stats[0] : nullptr;   // the block input's pending normalisation (stem: norm1 + relu1)
  int xrelu = inst;
  for (int blk = 0; blk < 6; ++blk) {
    const int C = kDims[blk], stride = (blk == 2 || blk == 4) ? 2 : 1;
    int o[3], k = 0;
    for (int i = 0; i < 4; ++i) if (i != x) o[k++] = i;
    const int t1 = o[0], t2 = o[1], d = o[2];
    ConvArgs c1 = conv_args(wt->block[blk][0], L.act[x], Hi, Wi, Cin, C, 3, stride);
    c1.in_stats = xs; c1.in_relu = xrelu;
    c1.out = L.act[t1];
    c1.relu = !inst;
    c1.part = inst ? L.part[0] : nullptr;
    launch_conv(c1, B, s);
    GS_CHECK_LAUNCH();
    if (inst) { launch_stats(c1, B, L.stats[1], s); GS_CHECK_LAUNCH(); }
    if (stride == 2) {
      ConvArgs dn = conv_args(wt->block[blk][2], L.act[x], Hi, Wi, Cin, C, 1, 2);
      dn.in_stats = xs; dn.in_relu = xrelu;
      dn.out = L.act[d];
      dn.part = inst ? L.part[2] : nullptr;
      launch_conv(dn, B, s);
      GS_CHECK_LAUNCH();
      if (inst) { launch_stats(dn, B, L.stats[3], s); GS_CHECK_LAUNCH(); }
    }
    const int r = stride == 2 ? d : x;
    ConvArgs c2 = conv_args(wt->block[blk][1], L.act[t1], c1.Ho, c1.Wo, C, C, 3, 1);
    c2.in_stats = inst ? L.stats[1] : nullptr; c2.in_relu = inst;
    c2.out = L.act[t2];
    if (inst) {
      c2.part = L.part[1];
    } else {
      c2.relu = 1;
      c2.res = L.act[r];
    }
    launch_conv(c2, B, s);
    GS_CHECK_LAUNCH();
    if (inst) {
      launch_stats(c2, B, L.stats[2], s);
      GS_CHECK_LAUNCH();
      const size_t nvec = (size_t)B * c2.Ho * c2.Wo * C / 8;
      encoder_tail_kernel<<<(unsigned)((nvec + 255) / 256), 256, 0, s>>>(
          L.act[t2], L.stats[2], L.act[r], stride == 2 ? L.stats[3] : xs, stride == 2 ? 0 : xrelu, B, c2.Ho * c2.Wo, C,
          L.act[t1]);
      GS_CHECK_LAUNCH();
      x = t1;
    } else {
      x = t2;
    }
    xs = nullptr; xrelu = 0;
    Hi = c2.Ho; Wi = c2.Wo; Cin = C;
  }

  ConvArgs f = conv_args(wt->out, L.act[x], Hi, Wi, 128, out_dim, 1, 1);
  f.out_nchw = (__half*)out;
  f.out2_nchw = (__half*)out2;
  f.split = split;
  launch_conv(f, B, s);
  GS_CHECK_LAUNCH();
  return GOSLAM_OK;
}
