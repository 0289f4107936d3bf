// corr_build_simt.cu — all-pairs correlation build, CUDA-core version + pyramid pooling.
//
// Reference: CorrBlock.corr / CorrBlock.__init__ (src/modules/corr.py:25-41,67-76):
//   corr[n] = (fmap1[n]/4)^T (fmap2[n]/4); level i+1 = F.avg_pool2d(level i, 2, 2).
// goslam_corr_build: the row-major build for f32 feature maps and for f16 ones outside the tensor-core
// kernel's envelope (D != 128 or w > 128), and the validation twin of that kernel (corr_build_tc.cu):
// same numerics contract — fp32 accumulate over the channels, x 1/16, one rounding to the volume
// dtype; each pooled level is the mean of the *rounded* finer level (fp32 sum of 4 in
// row-major window order, x 0.25, one rounding), exactly what avg_pool2d does.
#include "common.cuh"

namespace {

constexpr int TM = 64, TN = 64, TK = 16;

template <typename TIn, typename TOut>
__global__ void __launch_bounds__(256)
corr_gemm_simt(const TIn* __restrict__ f1, const TIn* __restrict__ f2, TOut* __restrict__ out,
               int D, int hw) {
  // A[k][m] = f1[n][k][m], B[k][p] = f2[n][k][p]; out[n][m][p]
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  const int n = blockIdx.z;
  const int m0 = blockIdx.y * TM, p0 = blockIdx.x * TN;
  const TIn* A = f1 + (size_t)n * D * hw;
  const TIn* B = f2 + (size_t)n * D * hw;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < D; k0 += TK) {
    for (int idx = threadIdx.x; idx < TK * TM; idx += 256) {
      const int kk = idx / TM, mm = idx % TM;
      const int m = m0 + mm, p = p0 + mm;
      As[kk][mm] = (m < hw && k0 + kk < D) ? (float)A[(size_t)(k0 + kk) * hw + m] : 0.f;
      Bs[kk][mm] = (p < hw && k0 + kk < D) ? (float)B[(size_t)(k0 + kk) * hw + p] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  TOut* O = out + (size_t)n * hw * hw;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= hw) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int p = p0 + tx * 4 + j;
      if (p < hw) O[(size_t)m * hw + p] = (TOut)(acc[i][j] * 0.0625f);
    }
  }
}

// level i -> level i+1 over [planes, h2, w2] -> [planes, h2/2, w2/2]
template <typename T>
__global__ void __launch_bounds__(256)
pool2x2_kernel(const T* __restrict__ in, T* __restrict__ out, long long planes, int h2, int w2) {
  const int ho = h2 >> 1, wo = w2 >> 1;
  const long long total = planes * ho * wo;
  for (long long idx = (long long)blockIdx.x * 256 + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * 256) {
    const int x = (int)(idx % wo);
    const int y = (int)((idx / wo) % ho);
    const long long pl = idx / ((long long)wo * ho);
    const T* p = in + (pl * h2 + 2 * y) * w2 + 2 * x;
    float s = (float)p[0];
    s += (float)p[1];
    s += (float)p[w2];
    s += (float)p[w2 + 1];
    out[idx] = (T)(s * 0.25f);
  }
}

template <typename TIn, typename TOut>
int build_simt(const TIn* f1, const TIn* f2, TOut* const* levels, int num_levels, int N, int D,
               int h, int w, cudaStream_t st) {
  const int hw = h * w;
  dim3 grid(gs_cdiv(hw, TN), gs_cdiv(hw, TM), N);
  corr_gemm_simt<TIn, TOut><<<grid, 256, 0, st>>>(f1, f2, levels[0], D, hw);
  GS_CHECK_LAUNCH();
  for (int i = 0; i + 1 < num_levels; ++i) {
    const int h2 = h >> i, w2 = w >> i;
    if ((h2 >> 1) <= 0 || (w2 >> 1) <= 0) return GOSLAM_EINVAL;
    const long long planes = (long long)N * hw;
    const long long total = planes * (h2 >> 1) * (w2 >> 1);
    const int blocks = (int)((total + 255) / 256 > kNumSms * 32 ? kNumSms * 32 : (total + 255) / 256);
    pool2x2_kernel<TOut><<<blocks, 256, 0, st>>>(levels[i], levels[i + 1], planes, h2, w2);
    GS_CHECK_LAUNCH();
  }
  return GOSLAM_OK;
}

}  // namespace

extern "C" int goslam_corr_build(const void* fmap1, const void* fmap2, int dtype, void* const* levels,
                                 int num_levels, int N, int D, int h, int w, void* stream) {
  if (N < 0 || D <= 0 || h <= 0 || w <= 0 || num_levels < 1 || num_levels > 4) return GOSLAM_EINVAL;
  if ((h >> (num_levels - 1)) <= 0 || (w >> (num_levels - 1)) <= 0) return GOSLAM_EINVAL;
  if (dtype != GOSLAM_F16 && dtype != GOSLAM_F32) return GOSLAM_EINVAL;
  if (N == 0) return GOSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == GOSLAM_F16)
    return build_simt<__half, __half>(static_cast<const __half*>(fmap1), static_cast<const __half*>(fmap2),
                                      reinterpret_cast<__half* const*>(levels), num_levels, N, D, h, w, st);
  return build_simt<float, float>(static_cast<const float*>(fmap1), static_cast<const float*>(fmap2),
                                  reinterpret_cast<float* const*>(levels), num_levels, N, D, h, w, st);
}
