// api.cu — library identification / error strings for the C-ABI in include/goslam_b200.h, and the host-side runtime
// policies every operator shares: error notes, per-device setup, the tensor-map encoder.
#include "common.cuh"

static thread_local cudaError_t g_last_cuda_error = cudaSuccess;
void gs_note_cuda_error(cudaError_t e) { g_last_cuda_error = e; }

int gs_device_setup_once(int (*setup)(int dev), bool* done, int* dev_out) {
  static std::mutex mu;
  int dev = -1;
  GS_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kGsMaxDevices) { gs_note_cuda_error(cudaErrorInvalidDevice); return GOSLAM_ELAUNCH; }
  if (dev_out) *dev_out = dev;
  std::lock_guard<std::mutex> lock(mu);
  if (done[dev]) return GOSLAM_OK;
  const int rc = setup(dev);
  done[dev] = rc == GOSLAM_OK;
  return rc;
}

namespace {
int g_sm_count[kGsMaxDevices];
int read_sm_count(int dev) {
  GS_CUDA(cudaDeviceGetAttribute(&g_sm_count[dev], cudaDevAttrMultiProcessorCount, dev));
  return GOSLAM_OK;
}
}  // namespace

int gs_sm_count(int* sms) {
  int dev = 0;
  const int rc = gs_device_setup<read_sm_count>(&dev);
  if (rc == GOSLAM_OK) *sms = g_sm_count[dev];
  return rc;
}

int gs_encode_tiled(GsEncodeTiled* fn) {
  static std::mutex mu;
  static GsEncodeTiled found = nullptr;
  std::lock_guard<std::mutex> lock(mu);
  if (!found) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    GS_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess) { gs_note_cuda_error(cudaErrorSymbolNotFound); return GOSLAM_ELAUNCH; }
    found = reinterpret_cast<GsEncodeTiled>(p);
  }
  *fn = found;
  return GOSLAM_OK;
}

extern "C" {

const char* goslam_last_cuda_error(void) {
  return g_last_cuda_error == cudaSuccess ? "" : cudaGetErrorString(g_last_cuda_error);
}

int goslam_version(void) { return 100; }

int goslam_sm_arch(void) {
#if defined(GOSLAM_SM_ARCH)
  return GOSLAM_SM_ARCH;
#else
  return 90;
#endif
}

const char* goslam_strerror(int code) {
  switch (code) {
    case GOSLAM_OK: return "ok";
    case GOSLAM_EINVAL: return "invalid argument or shape";
    case GOSLAM_ELAUNCH: return "CUDA launch failed";
    case GOSLAM_EWORKSPACE: return "workspace missing or too small";
    case GOSLAM_EUNSUPPORTED: return "entry point not supported (training-only backward)";
    default: return "unknown error";
  }
}

}  // extern "C"
