// The host protocol shared by the C-ABI handles (host.h): the one definition of the last error and its setters, the
// device probe and the error-word read.
#include <cstdarg>
#include <cstdio>

#include "host.h"

namespace ie {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

int cuda_fail(cudaError_t e, const char* what) {
  const int code = (e == cudaErrorMemoryAllocation) ? IE_ERR_OOM : IE_ERR_CUDA;
  if (e == cudaErrorMemoryAllocation) cudaGetLastError();  // clear the sticky-free OOM
  return fail(code, "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
}

int open_device(int device, int* sms) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(IE_ERR_CUDA, "no CUDA device available (%s): this library has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(IE_ERR_INVALID, "device %d not in [0,%d)", device, ndev);
  CK(cudaSetDevice(device));
  int major = 0;
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  CK(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, device));
  if (major != 9) return fail(IE_ERR_CUDA, "device compute capability %d.x is not sm_90 (H100)", major);
  return IE_OK;
}

int read_errors(const StreamOrder& order, const DevBuf& err, int* w, int n) {
  CK(order.wait());
  CK(cudaMemcpy(w, err.p, n * sizeof(int), cudaMemcpyDeviceToHost));
  if (std::any_of(w, w + n, [](int v) { return v != 0; })) {
    CK(cudaMemset(err.p, 0, n * sizeof(int)));
    CK(cudaDeviceSynchronize());
  }
  return IE_OK;
}

}  // namespace ie
