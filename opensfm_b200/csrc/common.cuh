// Shared host/device helpers for the opensfm_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>

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

}  // namespace osfm
