// Shared host-side plumbing for libfeiscan: error state, CUDA call checking, RAII
// device buffers, stream/event helpers.  No torch, no exceptions across the C ABI.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string>
#include "../../include/feiscan.h"

namespace fei {

// thread-local last error (fei_last_error, include/feiscan.h)
void set_error(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
const char* last_error();

struct Status {
  int code;
  Status(int c = FEI_OK) : code(c) {}
  bool ok() const { return code == FEI_OK; }
};

}  // namespace fei

#ifdef __CUDACC__
#include <cuda_runtime.h>

namespace fei {

int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define FEI_CUDA(call)                                                     \
  do {                                                                     \
    cudaError_t e__ = (call);                                              \
    if (e__ != cudaSuccess) return ::fei::cuda_fail(e__, #call, __FILE__, __LINE__); \
  } while (0)

#define FEI_TRY(expr)                 \
  do {                                \
    int rc__ = (expr);                \
    if (rc__ != FEI_OK) return rc__;  \
  } while (0)

// Owning device buffer (cudaMalloc / cudaFree).  Not copyable.
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  int alloc(size_t n);        // frees previous contents
  int ensure(size_t n);       // grow-only
  void release();
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Queues a host-to-device copy of bytes into b (grown to bytes + zero_slack + 16, so never empty) and zeroes the zero_slack
// bytes behind them.
int upload(DevBuf& b, const void* src, size_t bytes, size_t zero_slack, cudaStream_t s);

// process-wide state
struct Context {
  int device = -1;
  int sm_count = 0;
  size_t hbm_bytes = 0;
  int cc_major = 0, cc_minor = 0;
  cudaStream_t stream = nullptr;       // compute stream
  cudaStream_t copy_stream = nullptr;  // H2D / D2H overlap
  bool ready = false;
};
Context& ctx();
int require_ready();

size_t total_device_bytes();   // bytes currently held through DevBuf

}  // namespace fei
#endif
