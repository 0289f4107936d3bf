// common.cuh — shared device/host helpers for libgoslam_b200 (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <mutex>
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

// Evaluates a CUDA runtime or CUB call; if it fails, notes its error and returns GOSLAM_ELAUNCH.  The runtime's copy
// of the error is cleared, so a later GS_CHECK_LAUNCH (maybe in another entry point) does not report it again.
#define GS_CUDA(expr)                                            \
  do {                                                           \
    const cudaError_t e__ = (expr);                              \
    if (e__ != cudaSuccess) { (void)cudaGetLastError(); gs_note_cuda_error(e__); return GOSLAM_ELAUNCH; } \
  } while (0)

// host helpers shared by the .cu files (api.cu); hidden, so that the library exports only its C-ABI
#define GS_HIDDEN __attribute__((visibility("hidden")))

// Function attributes, occupancy and constant memory are per device.  gs_device_setup<Setup>() runs Setup(dev) on the
// current device unless it has already succeeded there, and returns its GOSLAM_* code; thread-safe.  A failed setup
// is not remembered, so the next call tries again.  No current device, or an ordinal of kGsMaxDevices or more, gives
// GOSLAM_ELAUNCH with the CUDA error noted.  dev_out, if given, receives the ordinal.
constexpr int kGsMaxDevices = 64;
GS_HIDDEN int gs_device_setup_once(int (*setup)(int dev), bool* done, int* dev_out);
template <int (*Setup)(int dev)>
int gs_device_setup(int* dev_out = nullptr) {
  static bool done[kGsMaxDevices];
  return gs_device_setup_once(Setup, done, dev_out);
}

// multiprocessor count of the current device, read once per device; fails as gs_device_setup
GS_HIDDEN int gs_sm_count(int* sms);

// cuTensorMapEncodeTiled, looked up from the driver once per process (thread-safe); GOSLAM_ELAUNCH, error noted, if
// the driver lacks it
typedef CUresult (*GsEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
GS_HIDDEN int gs_encode_tiled(GsEncodeTiled* fn);

// Tensor maps depend only on what the caller's Key holds (a base pointer, a shape, a kind), and launches use the same
// buffers call after call, so each map is encoded once (~2 us of host time) and kept in a most-recently-used table of
// Slots entries shared by all threads.  Encode makes the map of a key; Key needs ==.
template <typename Key, int Slots, bool (*Encode)(GsEncodeTiled, const Key&, CUtensorMap*)>
class GsTensorMapCache {
 public:
  // false, with the CUDA error noted, when the map cannot be made
  bool get(const Key& k, CUtensorMap* out) {
    std::lock_guard<std::mutex> lock(mu_);
    int victim = -1;
    for (int i = 0; i < Slots; ++i) {
      Slot& s = table_[i];
      if (s.used && s.key == k) {
        s.stamp = ++clock_;
        *out = s.map;
        return true;
      }
      // victim: a free slot if there is one, else the least recently used
      if (victim < 0 || (table_[victim].used && (!s.used || s.stamp < table_[victim].stamp))) victim = i;
    }
    Slot& v = table_[victim];
    v.used = false;
    GsEncodeTiled enc;
    if (gs_encode_tiled(&enc) != GOSLAM_OK) return false;
    // the encoder returns a driver CUresult, not a runtime error: report a rejected encode as an invalid argument
    if (!Encode(enc, k, &v.map)) { gs_note_cuda_error(cudaErrorInvalidValue); return false; }
    v.key = k; v.used = true; v.stamp = ++clock_;
    *out = v.map;
    return true;
  }

 private:
  struct Slot { Key key; CUtensorMap map; unsigned long long stamp; bool used; };
  Slot table_[Slots] = {};
  unsigned long long clock_ = 0;
  std::mutex mu_;
};

__host__ __device__ static inline int gs_cdiv(int a, int b) { return (a + b - 1) / b; }
#define gs_cdiv_dev gs_cdiv
static inline size_t gs_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Bump allocator over a caller-provided workspace: take<T>(n) hands out the next 256-byte aligned block of n Ts, and
// off is the bytes taken so far.  Each workspace has one layout function, xxx_layout(shape..., base, &carve), that
// takes its blocks in order and returns off: with a null base the arena only counts (every pointer is null), which
// is how the matching goslam_*_workspace_bytes sizes the workspace; with the caller's base it carves it.
struct GsArena {
  char* base; size_t off = 0;
  explicit GsArena(const void* p) : base((char*)p) {}
  template <typename T> T* take(size_t n) {
    T* r = base ? (T*)(base + off) : nullptr;
    off += gs_align(n * sizeof(T));
    return r;
  }
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

// K sums of a block of Threads threads in a fixed tree, every addition rounded on its own (no FMA), so the result does
// not depend on scheduling or on the compiler; valid in thread 0.  The fp64 reductions with fixed-order block partials
// (mesh_eval.cu, traj_eval.cu) are built on it.
template <int K, int Threads>
__device__ __forceinline__ void gs_block_sum(double (&v)[K], double (*sh)[Threads]) {
#pragma unroll
  for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = v[k];
  __syncthreads();
  for (int h = Threads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
#pragma unroll
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = __dadd_rn(sh[k][threadIdx.x], sh[k][threadIdx.x + h]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = sh[k][0];
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
