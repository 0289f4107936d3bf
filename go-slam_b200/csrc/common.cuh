// common.cuh — shared device/host helpers for libgoslam_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "goslam_b200.h"

// Streaming-multiprocessor count of the H100 SXM: grid size of the persistent kernels and of the fixed-grid
// reductions (their per-block partials are summed in block order, so the grid also fixes the rounding order).
constexpr int kNumSms = 132;

#define GS_MIN_DEPTH 0.25f   // src/lib/droid_kernels.cu:26 (CUDA side; the Python side uses 0.2)

// the CUDA error behind the most recent GOSLAM_ELAUNCH of this thread (goslam_last_cuda_error)
void gs_note_cuda_error(cudaError_t e);

#define GS_CHECK_LAUNCH()                                        \
  do {                                                           \
    cudaError_t e__ = cudaGetLastError();                        \
    if (e__ != cudaSuccess) { gs_note_cuda_error(e__); return GOSLAM_ELAUNCH; } \
  } while (0)

__host__ __device__ static inline int gs_cdiv(int a, int b) { return (a + b - 1) / b; }
#define gs_cdiv_dev gs_cdiv
static inline size_t gs_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Bump allocator over a caller-provided workspace.
struct GsArena {
  char* base; size_t cap; size_t off;
  GsArena(void* p, size_t c) : base((char*)p), cap(c), off(0) {}
  template <typename T> T* take(size_t n) {
    size_t bytes = gs_align(n * sizeof(T));
    T* r = (T*)(base + off);
    off += bytes;
    return r;
  }
  bool ok() const { return off <= cap && (base != nullptr || off == 0); }
};

// a / b for 0 <= a < 2^51 and b >= 1 through the double reciprocal inv_b = 1.0 / b: the product is within one of the
// quotient, one correction step makes it exact.  A few instructions where the 64-bit integer division is a long
// emulated sequence.
__device__ __forceinline__ long long gs_div_fast(long long a, long long b, double inv_b) {
  long long q = (long long)((double)a * inv_b);
  const long long r = a - q * b;
  if (r < 0) --q;
  else if (r >= b) ++q;
  return q;
}

__device__ __forceinline__ float gs_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double gs_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
