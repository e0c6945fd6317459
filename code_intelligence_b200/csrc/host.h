// The host protocol every C-ABI handle (api_*.cu) follows: error reporting, device buffers, the device probe, the
// stream a call runs on, the order of calls across streams and the device-side error words.
#pragma once
// the standard library and the kernel interfaces every handle's host code uses
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/issue_emb_b200.h"
#include "kernels.h"

namespace ie {

// the calling thread's last error (ie_last_error); fail and cuda_fail set it and return the code
extern thread_local std::string g_last_error;
int fail(int code, const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define CK(expr)                                                \
  do {                                                          \
    cudaError_t _e = (expr);                                    \
    if (_e != cudaSuccess) return ie::cuda_fail(_e, #expr);     \
  } while (0)

inline long long round_up(long long x, long long m) { return (x + m - 1) / m * m; }

// grow-only device buffer; owns its allocation (freed on destruction, so error paths do not leak)
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t reserve(size_t bytes, bool zero = false) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) { p = nullptr; return e; }
    cap = bytes;
    if (zero) {
      // the handle's streams are non-blocking: make the (legacy-stream) memset complete before anyone uses it
      e = cudaMemset(p, 0, bytes);
      if (e != cudaSuccess) return e;
      return cudaDeviceSynchronize();
    }
    return cudaSuccess;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// the device probe of every entry point that names a device: it exists and is an sm_90 part (this library has no CPU
// fallback); makes it current and returns its SM count in *sms
int open_device(int device, int* sms);

// the stream of a call: in device-pointer mode `stream` is used verbatim (NULL = the legacy default stream, e.g.
// torch's default); in host-pointer mode NULL selects the handle's own stream
inline cudaStream_t call_stream(int flags, void* stream, cudaStream_t own) {
  return (stream || (flags & IE_FLAG_DEVICE_PTRS)) ? static_cast<cudaStream_t>(stream) : own;
}

// One workspace per handle: a call on another stream than the last call's first waits for the last call to end.
struct StreamOrder {
  cudaEvent_t ev = nullptr;      // end of the last call (created by the first call)
  cudaStream_t last = nullptr;   // its stream
  bool has_done = false;
  StreamOrder() = default;
  StreamOrder(const StreamOrder&) = delete;
  StreamOrder& operator=(const StreamOrder&) = delete;
  ~StreamOrder() { if (ev) cudaEventDestroy(ev); }
  // before a call's first work on s
  cudaError_t begin(cudaStream_t s) {
    cudaError_t e = ev ? cudaSuccess : cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (e == cudaSuccess && has_done && last != s) e = cudaStreamWaitEvent(s, ev, 0);
    return e;
  }
  // after a call's last work on s
  cudaError_t end(cudaStream_t s) {
    const cudaError_t e = cudaEventRecord(ev, s);
    if (e == cudaSuccess) { has_done = true; last = s; }
    return e;
  }
  // the host waits for the last call
  cudaError_t wait() const { return has_done ? cudaEventSynchronize(ev) : cudaSuccess; }
};

// The n device error words of a handle's last call: waits for the call and copies them to w; when any is set, clears
// them and waits for the clear (the handles' streams do not wait for the legacy stream).  Each handle reports its own.
int read_errors(const StreamOrder& order, const DevBuf& err, int* w, int n);

// host array -> buf (reserved for n elements; host == nullptr: only reserved) on s
template <typename T>
int stage(DevBuf& buf, const T* host, size_t n, cudaStream_t s) {
  CK(buf.reserve(n * sizeof(T)));
  if (host != nullptr) CK(cudaMemcpyAsync(buf.p, host, n * sizeof(T), cudaMemcpyHostToDevice, s));
  return IE_OK;
}

// the row map of an unpermuted matrix of n rows padded to n_pad (upload_sliced): row i, then -1 for zero rows
inline std::vector<int> padded_identity(int n, int n_pad) {
  std::vector<int> perm(n_pad);
  for (int i = 0; i < n_pad; ++i) perm[i] = i < n ? i : -1;
  return perm;
}

}  // namespace ie
