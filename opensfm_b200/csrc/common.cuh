// Shared host/device helpers for the opensfm_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/opensfm_b200.h"

namespace osfm {

void set_last_error(const char* fmt, ...);
extern std::atomic<int64_t> g_kernel_launches;

struct CudaError : std::runtime_error {
  using std::runtime_error::runtime_error;
};
struct ArgError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

#define OSFM_CUDA(expr)                                                                   \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      char _buf[512];                                                                     \
      snprintf(_buf, sizeof(_buf), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
               __FILE__, __LINE__);                                                       \
      throw ::osfm::CudaError(_buf);                                                      \
    }                                                                                     \
  } while (0)

#define OSFM_LAUNCH_CHECK()                 \
  do {                                      \
    ::osfm::g_kernel_launches.fetch_add(1); \
    OSFM_CUDA(cudaGetLastError());          \
  } while (0)

// Wrap a C-ABI body: exceptions -> error codes + thread-local message.
#define OSFM_API_BEGIN try {
#define OSFM_API_END                                  \
  }                                                   \
  catch (const ::osfm::ArgError& e) {                 \
    ::osfm::set_last_error("%s", e.what());           \
    return OSFM_ERR_ARG;                              \
  }                                                   \
  catch (const ::osfm::CudaError& e) {                \
    ::osfm::set_last_error("%s", e.what());           \
    return OSFM_ERR_CUDA;                             \
  }                                                   \
  catch (const std::exception& e) {                   \
    ::osfm::set_last_error("%s", e.what());           \
    return OSFM_ERR_RUNTIME;                          \
  }                                                   \
  return OSFM_OK;

// Growable device buffer.
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  ~DevBuf() { release(); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  void reserve(size_t n) {
    if (n <= cap) return;
    release();
    size_t want = n + n / 4 + 16;
    OSFM_CUDA(cudaMalloc(&p, want * sizeof(T)));
    cap = want;
  }
};

// Growable pinned host buffer.
template <class T>
struct PinnedBuf {
  T* p = nullptr;
  size_t cap = 0;
  ~PinnedBuf() {
    if (p) cudaFreeHost(p);
  }
  void reserve(size_t n) {
    if (n <= cap) return;
    if (p) cudaFreeHost(p);
    p = nullptr;
    size_t want = n + n / 4 + 16;
    OSFM_CUDA(cudaMallocHost(&p, want * sizeof(T)));
    cap = want;
  }
};

// Copies of n elements on stream st.  The device buffer grows to hold at least one element, so that its pointer is
// never null, even for an empty upload.
template <class T>
void upload(DevBuf<T>& d, const T* h, size_t n, cudaStream_t st) {
  d.reserve(std::max<size_t>(n, 1));
  if (n) OSFM_CUDA(cudaMemcpyAsync(d.p, h, sizeof(T) * n, cudaMemcpyHostToDevice, st));
}
template <class T>
void upload(DevBuf<T>& d, const std::vector<T>& h, cudaStream_t st) {
  upload(d, h.data(), h.size(), st);
}
template <class T>
void download(T* h, const T* d, size_t n, cudaStream_t st) {
  if (n) OSFM_CUDA(cudaMemcpyAsync(h, d, sizeof(T) * n, cudaMemcpyDeviceToHost, st));
}
template <class T>
void download(std::vector<T>& h, const T* d, size_t n, cudaStream_t st) {
  h.resize(n);
  download(h.data(), d, n, st);
}

// The kernels an engine has opted into more than 48 KB of dynamic shared memory, each once, at a fixed byte count.
// The attribute is set for the current device, so an engine keeps one record per handle (= per device).
struct SmemOptIn {
  std::vector<const void*> opted;
  template <class Kernel>
  void operator()(Kernel* kernel, int bytes) {
    const void* k = (const void*)kernel;
    if (std::find(opted.begin(), opted.end(), k) != opted.end()) return;
    OSFM_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    opted.push_back(k);
  }
};

// An engine's device, its non-blocking stream there and NEV timing events, with the copies on that stream.
template <int NEV>
struct DeviceStream {
  int device;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[NEV] = {};

  explicit DeviceStream(int dev) : device(dev) {
    OSFM_CUDA(cudaSetDevice(device));
    OSFM_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    for (auto& e : ev) OSFM_CUDA(cudaEventCreate(&e));
  }
  ~DeviceStream() {
    for (auto& e : ev)
      if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }
  DeviceStream(const DeviceStream&) = delete;
  DeviceStream& operator=(const DeviceStream&) = delete;

  template <class T>
  void upload(DevBuf<T>& d, const T* h, size_t n) {
    ::osfm::upload(d, h, n, stream);
  }
  template <class T>
  void download(T* h, const T* d, size_t n) {
    ::osfm::download(h, d, n, stream);
  }
};

// What stands behind one C-ABI handle (osfm_ba, osfm_matcher, osfm_tracks, osfm_rotransac): the engine object and the
// lock that serialises calls on it.  The engine's methods expect its device to be current: with_handle makes it so
// for every entry point, and the destructor for the engine's own destructor, which frees its device memory.
template <class Engine>
struct Handle {
  std::mutex mu;
  Engine impl;
  explicit Handle(int device) : impl(device) {}
  ~Handle() { cudaSetDevice(impl.device); }
};

// osfm_<kind>_create and osfm_<kind>_destroy.
template <class H>
int create_handle(int device, H** out) {
  OSFM_API_BEGIN
  if (!out) throw ArgError("null out");
  int count = 0;
  OSFM_CUDA(cudaGetDeviceCount(&count));
  if (device < 0 || device >= count) throw ArgError("no such CUDA device");
  *out = new H(device);
  OSFM_API_END
}
template <class H>
int destroy_handle(H* h) {
  OSFM_API_BEGIN
  delete h;
  OSFM_API_END
}

// Every other entry point on a handle: body(engine) under the handle's lock with its device current, exceptions
// turned into error codes.  The lock is not recursive, so body must not re-enter the same handle.
template <class H, class F>
int with_handle(H* h, F&& body) {
  OSFM_API_BEGIN
  if (!h) throw ArgError(H::null_message);
  std::lock_guard<std::mutex> lock(h->mu);
  OSFM_CUDA(cudaSetDevice(h->impl.device));
  body(h->impl);
  OSFM_API_END
}

}  // namespace osfm
