// Process/device context, error state and device buffers for libfeiscan.
#include "common.h"
#include <stdarg.h>
#include <stdio.h>
#include <atomic>

namespace fei {

static thread_local char g_err[1024] = "";
static std::atomic<size_t> g_dev_bytes{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d in %s", (int)e, cudaGetErrorString(e), file, line, what);
  cudaGetLastError();  // clear sticky-less errors so the next call reports its own
  return FEI_E_CUDA;
}

int DevBuf::alloc(size_t n) {
  (void)ctx();
  release();
  if (n == 0) return FEI_OK;
  cudaError_t e = cudaMalloc(&p, n);
  if (e != cudaSuccess) { p = nullptr; return cuda_fail(e, "cudaMalloc", __FILE__, __LINE__); }
  bytes = n;
  g_dev_bytes += n;
  return FEI_OK;
}
int DevBuf::ensure(size_t n) {
  if (n <= bytes) return FEI_OK;
  return alloc(n);
}
void DevBuf::release() {
  if (p) { cudaFree(p); g_dev_bytes -= bytes; }
  p = nullptr; bytes = 0;
}
size_t total_device_bytes() { return g_dev_bytes.load(); }

int upload(DevBuf& b, const void* src, size_t bytes, size_t zero_slack, cudaStream_t s) {
  FEI_TRY(b.ensure(bytes + zero_slack + 16));
  if (bytes) FEI_CUDA(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, s));
  if (zero_slack) FEI_CUDA(cudaMemsetAsync((uint8_t*)b.p + bytes, 0, zero_slack, s));
  return FEI_OK;
}

// Simple three-phase exclusive scan of u32 -> u64 (n up to 2^40): per-block sums,
// serial scan of the block sums by one thread block, then per-block rescan.
constexpr int kScanBlock = 1024;
__global__ void k_scan_block_sums(const uint32_t* __restrict__ in, uint64_t n, uint64_t* __restrict__ sums) {
  __shared__ uint64_t sh[32];
  uint64_t i = blockIdx.x * (uint64_t)kScanBlock + threadIdx.x;
  uint64_t v = i < n ? in[i] : 0;
  for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    uint64_t s = sh[threadIdx.x];
    for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) sums[blockIdx.x] = s;
  }
}
__global__ void k_scan_sums_inplace(uint64_t* sums, uint64_t nb) {
  // single block; nb block sums -> exclusive prefix, chunked by blockDim
  __shared__ uint64_t carry;
  __shared__ uint64_t sh[1024];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint64_t base = 0; base < nb; base += blockDim.x) {
    uint64_t i = base + threadIdx.x;
    uint64_t v = i < nb ? sums[i] : 0;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < blockDim.x; o <<= 1) {
      uint64_t t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    uint64_t incl = sh[threadIdx.x];
    if (i < nb) sums[i] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry += incl;
    __syncthreads();
  }
}
__global__ void k_scan_finish(const uint32_t* __restrict__ in, uint64_t n, const uint64_t* __restrict__ sums, uint64_t* __restrict__ out) {
  __shared__ uint64_t sh[kScanBlock];
  uint64_t i = blockIdx.x * (uint64_t)kScanBlock + threadIdx.x;
  uint64_t v = i < n ? in[i] : 0;
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int o = 1; o < kScanBlock; o <<= 1) {
    uint64_t t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
    __syncthreads();
    sh[threadIdx.x] += t;
    __syncthreads();
  }
  uint64_t excl = sums[blockIdx.x] + sh[threadIdx.x] - v;
  if (i < n) out[i] = excl;
  if (i == n - 1) out[n] = excl + v;
}

// out has n+1 entries.  tmp grows to ceil(n/1024) u64.
static int exclusive_scan_u32_u64(const uint32_t* in, uint64_t n, uint64_t* out, DevBuf& tmp, cudaStream_t s) {
  if (n == 0) { FEI_CUDA(cudaMemsetAsync(out, 0, sizeof(uint64_t), s)); return FEI_OK; }
  uint64_t nb = (n + kScanBlock - 1) / kScanBlock;
  FEI_TRY(tmp.ensure(nb * sizeof(uint64_t)));
  k_scan_block_sums<<<(unsigned)nb, kScanBlock, 0, s>>>(in, n, tmp.as<uint64_t>());
  k_scan_sums_inplace<<<1, 1024, 0, s>>>(tmp.as<uint64_t>(), nb);
  k_scan_finish<<<(unsigned)nb, kScanBlock, 0, s>>>(in, n, tmp.as<uint64_t>(), out);
  FEI_CUDA(cudaGetLastError());
  return FEI_OK;
}

int queue_offsets(const uint32_t* len, uint64_t n, uint64_t* off, uint64_t* host, bool whole, DevBuf& tmp, cudaStream_t s) {
  FEI_TRY(exclusive_scan_u32_u64(len, n, off, tmp, s));
  FEI_CUDA(cudaMemcpyAsync(host, whole ? off : off + n, (whole ? n + 1 : 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  return FEI_OK;
}

/* The CUDA "current device" is per host thread: a worker thread of the caller (a thread pool loading batches, Flask's request
 * threads) starts on device 0 whatever fei_init bound.  Every path that touches the device goes through ctx() or DevBuf::alloc, so
 * this is where the calling thread is put on the bound device. */
static inline void bind_thread(const Context& c) {
  int d = -1;
  if (c.ready && (cudaGetDevice(&d) != cudaSuccess || d != c.device)) cudaSetDevice(c.device);
}
Context& ctx() { static Context c; bind_thread(c); return c; }

int require_ready() {
  if (!ctx().ready) { set_error("fei_init() has not been called (or failed): no CUDA device bound; there is no CPU path"); return FEI_E_CUDA; }
  return FEI_OK;
}

}  // namespace fei

using namespace fei;

extern "C" int fei_abi_version(void) { return FEI_ABI_VERSION; }
extern "C" const char* fei_last_error(void) { return last_error(); }

extern "C" int fei_init(int device) {
  Context& c = ctx();
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error("no usable CUDA device (%s); libfeiscan has no CPU fallback", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    cudaGetLastError();
    return FEI_E_CUDA;
  }
  if (device < 0 || device >= ndev) { set_error("device %d out of range (0..%d)", device, ndev - 1); return FEI_E_BADARG; }
  if (c.ready && c.device == device) return FEI_OK;
  FEI_CUDA(cudaSetDevice(device));
  cudaDeviceProp p;
  FEI_CUDA(cudaGetDeviceProperties(&p, device));
  c.device = device;
  c.sm_count = p.multiProcessorCount;
  c.hbm_bytes = p.totalGlobalMem;
  c.cc_major = p.major; c.cc_minor = p.minor;
  if (p.major != 9 || p.minor != 0) {              // sm_90a code loads on compute capability 9.0 only
    set_error("device %d is sm_%d%d; libfeiscan is built for sm_90a only", device, p.major, p.minor);
    return FEI_E_CUDA;
  }
  if (!c.stream) FEI_CUDA(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
  if (!c.copy_stream) FEI_CUDA(cudaStreamCreateWithFlags(&c.copy_stream, cudaStreamNonBlocking));
  c.ready = true;
  return FEI_OK;
}

namespace fei { void chain_release_scratch(); }

extern "C" int fei_shutdown(void) {
  fei::chain_release_scratch();
  Context& c = ctx();
  if (c.stream) { cudaStreamDestroy(c.stream); c.stream = nullptr; }
  if (c.copy_stream) { cudaStreamDestroy(c.copy_stream); c.copy_stream = nullptr; }
  c.ready = false;
  return FEI_OK;
}

extern "C" int fei_device_info(int* sm_count, uint64_t* hbm_bytes, int* cc_major, int* cc_minor) {
  FEI_TRY(require_ready());
  Context& c = ctx();
  if (sm_count) *sm_count = c.sm_count;
  if (hbm_bytes) *hbm_bytes = c.hbm_bytes;
  if (cc_major) *cc_major = c.cc_major;
  if (cc_minor) *cc_minor = c.cc_minor;
  return FEI_OK;
}

extern "C" int fei_host_register(void* p, uint64_t bytes) {
  FEI_TRY(require_ready());
  if (!p || !bytes) return FEI_OK;
  FEI_CUDA(cudaHostRegister(p, bytes, cudaHostRegisterDefault));
  return FEI_OK;
}

extern "C" int fei_host_unregister(void* p) {
  FEI_TRY(require_ready());
  if (!p) return FEI_OK;
  FEI_CUDA(cudaHostUnregister(p));
  return FEI_OK;
}

/* Measured host <-> device copy bandwidth of a caller buffer (pinned with fei_host_register for the PCIe rate): best of
 * `reps` timed copies each way, CUDA events on the copy stream.  The roofline of every "from host buffers" number. */
extern "C" int fei_host_copy_bench(void* host, uint64_t bytes, int reps, float* h2d_gbs, float* d2h_gbs) {
  FEI_TRY(require_ready());
  if (!host || !bytes || reps < 1) { set_error("bad argument"); return FEI_E_BADARG; }
  cudaStream_t s = ctx().copy_stream;
  DevBuf d;
  FEI_TRY(d.alloc(bytes));
  cudaEvent_t e0, e1;
  FEI_CUDA(cudaEventCreate(&e0)); FEI_CUDA(cudaEventCreate(&e1));
  float best[2] = {0.f, 0.f};
  for (int dir = 0; dir < 2; ++dir)
    for (int r = 0; r < reps + 1; ++r) {
      FEI_CUDA(cudaEventRecord(e0, s));
      if (dir == 0) FEI_CUDA(cudaMemcpyAsync(d.p, host, bytes, cudaMemcpyHostToDevice, s));
      else FEI_CUDA(cudaMemcpyAsync(host, d.p, bytes, cudaMemcpyDeviceToHost, s));
      FEI_CUDA(cudaEventRecord(e1, s));
      FEI_CUDA(cudaStreamSynchronize(s));
      float ms = 0; FEI_CUDA(cudaEventElapsedTime(&ms, e0, e1));
      const float gbs = (float)((double)bytes / 1e9 / (ms * 1e-3));
      if (r > 0 && gbs > best[dir]) best[dir] = gbs;
    }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (h2d_gbs) *h2d_gbs = best[0];
  if (d2h_gbs) *d2h_gbs = best[1];
  return FEI_OK;
}
