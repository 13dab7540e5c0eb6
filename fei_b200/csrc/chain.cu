// K3: batched SHA-256 link-hash validation of a Memorychain (sm_90a).
//
// Replaces the loop of MemoryChain.validate_chain (memdir_tools/memorychain.py:596-618):
//   for i in 1..n-1:
//     block[i].hash != sha256(canonical_json(block[i])).hexdigest()  -> "invalid hash"  (kind 1)
//     block[i].previous_hash != block[i-1].hash                      -> "broken link"   (kind 2)
// Both comparisons are string comparisons in the reference; stored strings that are
// not 64 lowercase hex digits can never equal a hexdigest, and links between
// arbitrary strings are compared byte-wise on the device.
//
// Device layout ("pack once"): every message is pre-padded to whole 64-byte SHA-256
// blocks (0x80, zeros, 64-bit big-endian bit length) so the hash kernel is a pure
// compression loop over 16-byte aligned loads; stored hashes are kept as 32-byte
// binary digests.  One message per thread; the 64 round constants are immediates
// of the fully unrolled rounds (no table loads at all).  The kernel is INT32-issue
// bound (about 1.4k integer ops per compression), not HBM bound: see DESIGN.md.
#include "common.h"
#include "chain_json.h"
#include "jsonfmt.cuh"
#include <vector>
#include <string.h>
#include <mutex>
#include <chrono>
#include <stdlib.h>
#include <stdio.h>

namespace fei {

// ------------------------------------------------------------------ device SHA-256
__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }
__device__ __forceinline__ uint32_t bswap(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

#define SHA_K_LIST \
  0x428a2f98u,0x71374491u,0xb5c0fbcfu,0xe9b5dba5u,0x3956c25bu,0x59f111f1u,0x923f82a4u,0xab1c5ed5u, \
  0xd807aa98u,0x12835b01u,0x243185beu,0x550c7dc3u,0x72be5d74u,0x80deb1feu,0x9bdc06a7u,0xc19bf174u, \
  0xe49b69c1u,0xefbe4786u,0x0fc19dc6u,0x240ca1ccu,0x2de92c6fu,0x4a7484aau,0x5cb0a9dcu,0x76f988dau, \
  0x983e5152u,0xa831c66du,0xb00327c8u,0xbf597fc7u,0xc6e00bf3u,0xd5a79147u,0x06ca6351u,0x14292967u, \
  0x27b70a85u,0x2e1b2138u,0x4d2c6dfcu,0x53380d13u,0x650a7354u,0x766a0abbu,0x81c2c92eu,0x92722c85u, \
  0xa2bfe8a1u,0xa81a664bu,0xc24b8b70u,0xc76c51a3u,0xd192e819u,0xd6990624u,0xf40e3585u,0x106aa070u, \
  0x19a4c116u,0x1e376c08u,0x2748774cu,0x34b0bcb5u,0x391c0cb3u,0x4ed8aa4au,0x5b9cca4fu,0x682e6ff3u, \
  0x748f82eeu,0x78a5636fu,0x84c87814u,0x8cc70208u,0x90befffau,0xa4506cebu,0xbef9a3f7u,0xc67178f2u

// One compression: state += F(state, 16 big-endian message words).  Fully unrolled so
// K[t] folds into IADD3 immediates and w[] lives in registers.
__device__ __forceinline__ void sha256_compress(uint32_t (&st)[8], uint32_t (&w)[16]) {
  constexpr uint32_t K[64] = {SHA_K_LIST};
  uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
  for (int t = 0; t < 64; ++t) {
    uint32_t wt;
    if (t < 16) {
      wt = w[t];
    } else {
      uint32_t w15 = w[(t - 15) & 15], w2 = w[(t - 2) & 15];
      uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3);
      uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10);
      wt = w[t & 15] + s0 + w[(t - 7) & 15] + s1;
      w[t & 15] = wt;
    }
    uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
    uint32_t ch = (e & f) ^ (~e & g);
    uint32_t t1 = h + S1 + ch + K[t] + wt;
    uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
    uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
    uint32_t t2 = S0 + mj;
    h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

__device__ __forceinline__ uint4 ldg_nc16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// ------------------------------------------------------------------ kernels
// Pad tight messages into whole SHA-256 blocks.  blk_off[i] (in 64-byte blocks) is the
// exclusive prefix sum of ceil((len+9)/64).
__global__ void k_count_blocks(const uint64_t* __restrict__ msg_off, uint64_t n, uint32_t* __restrict__ nblk) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t len = msg_off[i + 1] - msg_off[i];
  nblk[i] = (uint32_t)((len + 9 + 63) >> 6);
}

__global__ void k_pad_messages(const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ msg_off,
                               const uint64_t* __restrict__ blk_off, uint64_t n, uint8_t* __restrict__ padded) {
  // one warp per message: lanes stride the padded area byte-wise in 4-byte words
  uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= n) return;
  const uint8_t* src = msgs + msg_off[warp];
  uint64_t len = msg_off[warp + 1] - msg_off[warp];
  uint64_t total = (blk_off[warp + 1] - blk_off[warp]) << 6;
  uint8_t* dst = padded + (blk_off[warp] << 6);
  uint64_t bits = len << 3;
  for (uint64_t o = lane; o < total; o += 32) {
    uint8_t v;
    if (o < len) v = src[o];
    else if (o == len) v = 0x80;
    else if (o >= total - 8) v = (uint8_t)(bits >> (8 * (total - 1 - o)));
    else v = 0;
    dst[o] = v;
  }
}

__device__ __forceinline__ int hexval(uint8_t c) {
  if (c >= '0' && c <= '9') return c - '0';
  if (c >= 'a' && c <= 'f') return c - 'a' + 10;
  return -1;
}

// Stored strings -> binary digests + flags; link strings compared byte-wise.
//   flags bit0: stored hash is a canonical hexdigest (64 lowercase hex)
//   flags bit1: previous_hash[i] == hash[i-1] (string equality); bit set for i == 0
__global__ void k_prepare_links(const uint8_t* __restrict__ hash, const uint64_t* __restrict__ hash_off,
                                const uint8_t* __restrict__ prev, const uint64_t* __restrict__ prev_off,
                                uint64_t n, uint8_t* __restrict__ stored_bin, uint8_t* __restrict__ flags) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* h = hash + hash_off[i];
  uint64_t hl = hash_off[i + 1] - hash_off[i];
  uint8_t fl = 0;
  bool canon = hl == 64;
  if (canon) {
    for (int k = 0; k < 32; ++k) {
      int hi = hexval(h[2 * k]), lo = hexval(h[2 * k + 1]);
      if ((hi | lo) < 0) { canon = false; break; }
      stored_bin[i * 32 + k] = (uint8_t)(hi << 4 | lo);
    }
  }
  if (canon) fl |= 1;
  if (i == 0) fl |= 2;
  else {
    const uint8_t* p = prev + prev_off[i];
    uint64_t pl = prev_off[i + 1] - prev_off[i];
    const uint8_t* q = hash + hash_off[i - 1];
    uint64_t ql = hash_off[i] - hash_off[i - 1];
    bool eq = pl == ql;
    for (uint64_t k = 0; eq && k < pl; ++k) eq = p[k] == q[k];
    if (eq) fl |= 2;
  }
  flags[i] = fl;
}

// Hash + validate.  One message per thread.  verdict = min over failing i of (i*4 + kind).
template <bool kWriteDigests>
__global__ void __launch_bounds__(128)
k_sha256_validate(const uint8_t* __restrict__ padded, const uint64_t* __restrict__ blk_off,
                  const uint8_t* __restrict__ stored_bin, const uint8_t* __restrict__ flags,
                  uint64_t n, uint8_t* __restrict__ digests, unsigned long long* __restrict__ verdict) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!kWriteDigests && i == 0) return;     // genesis is never checked (memorychain.py:604)
  uint64_t b0 = blk_off[i], b1 = blk_off[i + 1];
  uint32_t st[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
  const uint4* p = reinterpret_cast<const uint4*>(padded + (b0 << 6));
  for (uint64_t b = b0; b < b1; ++b, p += 4) {
    uint4 q0 = ldg_nc16(p), q1 = ldg_nc16(p + 1), q2 = ldg_nc16(p + 2), q3 = ldg_nc16(p + 3);
    uint32_t w[16] = {bswap(q0.x), bswap(q0.y), bswap(q0.z), bswap(q0.w), bswap(q1.x), bswap(q1.y), bswap(q1.z), bswap(q1.w),
                      bswap(q2.x), bswap(q2.y), bswap(q2.z), bswap(q2.w), bswap(q3.x), bswap(q3.y), bswap(q3.z), bswap(q3.w)};
    sha256_compress(st, w);
  }
  if (kWriteDigests) {
    uint4* d = reinterpret_cast<uint4*>(digests + i * 32);
    d[0] = make_uint4(bswap(st[0]), bswap(st[1]), bswap(st[2]), bswap(st[3]));
    d[1] = make_uint4(bswap(st[4]), bswap(st[5]), bswap(st[6]), bswap(st[7]));
    if (i == 0) return;
  }
  uint8_t fl = flags[i];
  bool ok = fl & 1;
  if (ok) {
    const uint4* s = reinterpret_cast<const uint4*>(stored_bin + i * 32);
    uint4 s0 = s[0], s1 = s[1];
    ok = s0.x == bswap(st[0]) && s0.y == bswap(st[1]) && s0.z == bswap(st[2]) && s0.w == bswap(st[3]) &&
         s1.x == bswap(st[4]) && s1.y == bswap(st[5]) && s1.z == bswap(st[6]) && s1.w == bswap(st[7]);
  }
  int kind = !ok ? 1 : ((fl & 2) ? 0 : 2);
  if (kind) atomicMin(verdict, (unsigned long long)(i * 4 + kind));
}

// ------------------------------------------------------------------ proof of work ("next" row 2)
// MemoryBlock.mine_block (memdir_tools/memorychain.py:132-143): smallest nonce >= the current one whose
// hexdigest starts with `difficulty` zeros.  The canonical text is prefix + decimal(nonce) + suffix (the
// nonce sits between "memory_id" and "previous_hash" in the sorted key order); one candidate per thread.
constexpr int kMineMaxFixed = 1024;                    // prefix + suffix bytes kept in shared memory

__global__ void __launch_bounds__(256)
k_mine(const uint8_t* __restrict__ fixed, uint32_t plen, uint32_t slen, unsigned long long base, unsigned long long count,
       uint32_t zero_nibbles, unsigned long long* __restrict__ best) {
  __shared__ uint8_t sh[kMineMaxFixed];
  for (uint32_t k = threadIdx.x; k < plen + slen; k += blockDim.x) sh[k] = fixed[k];
  __syncthreads();
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long idx = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; idx < count; idx += stride) {
    const unsigned long long nonce = base + idx;
    if (nonce >= *reinterpret_cast<volatile unsigned long long*>(best)) continue;   // a smaller winner is already known
    char dg[20]; uint32_t nd = 0;
    { unsigned long long v = nonce; char tmp[20]; do { tmp[nd++] = (char)('0' + v % 10); v /= 10; } while (v); for (uint32_t k = 0; k < nd; ++k) dg[k] = tmp[nd - 1 - k]; }
    const uint32_t total = plen + nd + slen;
    const uint32_t nblk = (total + 9 + 63) >> 6;
    const unsigned long long bits = (unsigned long long)total << 3;
    uint32_t st[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    for (uint32_t b = 0; b < nblk; ++b) {
      uint32_t w[16];
#pragma unroll
      for (int t = 0; t < 16; ++t) {
        uint32_t word = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t pos = b * 64 + t * 4 + j;
          uint32_t byte;
          if (pos < plen) byte = sh[pos];
          else if (pos < plen + nd) byte = (uint8_t)dg[pos - plen];
          else if (pos < total) byte = sh[pos - nd];
          else if (pos == total) byte = 0x80;
          else if (pos >= nblk * 64 - 8) byte = (uint32_t)(bits >> (8 * (nblk * 64 - 1 - pos))) & 0xFFu;
          else byte = 0;
          word = word << 8 | byte;
        }
        w[t] = word;
      }
      sha256_compress(st, w);
    }
    bool ok = true;                                       // `zero_nibbles` leading hex zeros
    for (uint32_t k = 0; ok && k < zero_nibbles; ++k) ok = ((st[k >> 3] >> (28 - 4 * (k & 7))) & 0xFu) == 0;
    if (ok) atomicMin(best, nonce);
  }
}

// ------------------------------------------------------------------ resident chain
}  // namespace fei

struct fei_chain {
  uint64_t n = 0, first_index = 0;
  uint64_t msg_bytes = 0, total_blocks = 0;
  fei::DevBuf msgs, msg_off;          // tight canonical JSON (kept for fetch / debugging)
  fei::DevBuf padded, blk_off;        // SHA-ready
  fei::DevBuf hash, hash_off, prev, prev_off;
  fei::DevBuf stored_bin, flags, digests, verdict, nblk, scan_tmp;
  fei::DevBuf col_tag[FEI_CHAIN_NCOLS], col_num[FEI_CHAIN_NCOLS], col_str[FEI_CHAIN_NCOLS], col_off[FEI_CHAIN_NCOLS], json_len, json_err;   // column form (fei_chain_load_cols)
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

namespace fei {

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

// out has n+1 entries.  tmp must hold ceil(n/1024) u64.
int exclusive_scan_u32_u64(const uint32_t* in, uint64_t n, uint64_t* out, DevBuf& tmp, cudaStream_t s) {
  if (n == 0) { FEI_CUDA(cudaMemsetAsync(out, 0, sizeof(uint64_t), s)); return FEI_OK; }
  uint64_t nb = (n + kScanBlock - 1) / kScanBlock;
  FEI_TRY(tmp.ensure(nb * sizeof(uint64_t)));
  k_scan_block_sums<<<(unsigned)nb, kScanBlock, 0, s>>>(in, n, tmp.as<uint64_t>());
  k_scan_sums_inplace<<<1, 1024, 0, s>>>(tmp.as<uint64_t>(), nb);
  k_scan_finish<<<(unsigned)nb, kScanBlock, 0, s>>>(in, n, tmp.as<uint64_t>(), out);
  FEI_CUDA(cudaGetLastError());
  return FEI_OK;
}

static int chain_prepare(fei_chain* ch) {
  // msgs/msg_off/hash/hash_off/prev/prev_off are on the device: build padded blocks + link flags
  Context& c = ctx();
  uint64_t n = ch->n;
  FEI_TRY(ch->nblk.ensure(n * sizeof(uint32_t)));
  FEI_TRY(ch->blk_off.ensure((n + 1) * sizeof(uint64_t)));
  unsigned g = (unsigned)((n + 255) / 256);
  k_count_blocks<<<g, 256, 0, c.stream>>>(ch->msg_off.as<uint64_t>(), n, ch->nblk.as<uint32_t>());
  FEI_TRY(exclusive_scan_u32_u64(ch->nblk.as<uint32_t>(), n, ch->blk_off.as<uint64_t>(), ch->scan_tmp, c.stream));
  uint64_t total = 0;
  FEI_CUDA(cudaMemcpyAsync(&total, ch->blk_off.as<uint64_t>() + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, c.stream));
  FEI_CUDA(cudaStreamSynchronize(c.stream));
  ch->total_blocks = total;
  FEI_TRY(ch->padded.ensure(total * 64));
  uint64_t warps_per_block = 8;
  unsigned gp = (unsigned)((n + warps_per_block - 1) / warps_per_block);
  k_pad_messages<<<gp, 256, 0, c.stream>>>(ch->msgs.as<uint8_t>(), ch->msg_off.as<uint64_t>(), ch->blk_off.as<uint64_t>(), n, ch->padded.as<uint8_t>());
  FEI_TRY(ch->stored_bin.ensure(n * 32));
  FEI_TRY(ch->flags.ensure(n));
  k_prepare_links<<<g, 256, 0, c.stream>>>(ch->hash.as<uint8_t>(), ch->hash_off.as<uint64_t>(), ch->prev.as<uint8_t>(), ch->prev_off.as<uint64_t>(), n,
                                           ch->stored_bin.as<uint8_t>(), ch->flags.as<uint8_t>());
  FEI_CUDA(cudaGetLastError());
  FEI_TRY(ch->verdict.ensure(sizeof(unsigned long long)));
  return FEI_OK;
}

}  // namespace fei

using namespace fei;

static std::mutex g_scratch_mu;
static fei_chain* g_scratch = nullptr;

extern "C" int fei_chain_create(fei_chain** out) {
  if (!out) { set_error("null out"); return FEI_E_BADARG; }
  FEI_TRY(require_ready());
  fei_chain* ch = new fei_chain();
  cudaEventCreate(&ch->ev0); cudaEventCreate(&ch->ev1);
  *out = ch;
  return FEI_OK;
}

extern "C" int fei_chain_destroy(fei_chain* ch) {
  if (!ch) return FEI_OK;
  if (ch->ev0) cudaEventDestroy(ch->ev0);
  if (ch->ev1) cudaEventDestroy(ch->ev1);
  delete ch;
  return FEI_OK;
}

extern "C" int fei_chain_load_msgs(fei_chain* ch, const uint8_t* msgs, const uint64_t* msg_off,
                                   const uint8_t* hash, const uint64_t* hash_off,
                                   const uint8_t* prev, const uint64_t* prev_off, uint64_t n, uint64_t first_index) {
  FEI_TRY(require_ready());
  if (!ch || !msg_off || !hash_off || !prev_off) { set_error("null argument"); return FEI_E_BADARG; }
  Context& c = ctx();
  ch->n = n; ch->first_index = first_index;
  ch->msg_bytes = n ? msg_off[n] - msg_off[0] : 0;
  if (n && msg_off[0] != 0) { set_error("msg_off[0] must be 0"); return FEI_E_BADARG; }
  FEI_TRY(upload(ch->msgs, msgs, ch->msg_bytes, 0, c.stream));
  FEI_TRY(upload(ch->msg_off, msg_off, (n + 1) * 8, 0, c.stream));
  FEI_TRY(upload(ch->hash, hash, n ? hash_off[n] : 0, 0, c.stream));
  FEI_TRY(upload(ch->hash_off, hash_off, (n + 1) * 8, 0, c.stream));
  FEI_TRY(upload(ch->prev, prev, n ? prev_off[n] : 0, 0, c.stream));
  FEI_TRY(upload(ch->prev_off, prev_off, (n + 1) * 8, 0, c.stream));
  if (n == 0) return FEI_OK;
  return chain_prepare(ch);
}

extern "C" int fei_chain_validate(fei_chain* ch, int64_t* first_bad, int32_t* bad_kind, uint8_t* digests, float* kernel_ms) {
  FEI_TRY(require_ready());
  if (!ch) { set_error("null chain"); return FEI_E_BADARG; }
  Context& c = ctx();
  uint64_t n = ch->n;
  if (first_bad) *first_bad = -1;
  if (bad_kind) *bad_kind = 0;
  if (kernel_ms) *kernel_ms = 0.f;
  if (n == 0) return FEI_OK;
  FEI_CUDA(cudaMemsetAsync(ch->verdict.p, 0xFF, sizeof(unsigned long long), c.stream));
  unsigned g = (unsigned)((n + 127) / 128);
  FEI_CUDA(cudaEventRecord(ch->ev0, c.stream));
  if (digests) {
    FEI_TRY(ch->digests.ensure(n * 32));
    k_sha256_validate<true><<<g, 128, 0, c.stream>>>(ch->padded.as<uint8_t>(), ch->blk_off.as<uint64_t>(), ch->stored_bin.as<uint8_t>(),
                                                     ch->flags.as<uint8_t>(), n, ch->digests.as<uint8_t>(), ch->verdict.as<unsigned long long>());
  } else {
    k_sha256_validate<false><<<g, 128, 0, c.stream>>>(ch->padded.as<uint8_t>(), ch->blk_off.as<uint64_t>(), ch->stored_bin.as<uint8_t>(),
                                                      ch->flags.as<uint8_t>(), n, nullptr, ch->verdict.as<unsigned long long>());
  }
  FEI_CUDA(cudaEventRecord(ch->ev1, c.stream));
  FEI_CUDA(cudaGetLastError());
  unsigned long long v = 0;
  FEI_CUDA(cudaMemcpyAsync(&v, ch->verdict.p, sizeof(v), cudaMemcpyDeviceToHost, c.stream));
  if (digests) FEI_CUDA(cudaMemcpyAsync(digests, ch->digests.p, n * 32, cudaMemcpyDeviceToHost, c.stream));
  FEI_CUDA(cudaStreamSynchronize(c.stream));
  if (kernel_ms) FEI_CUDA(cudaEventElapsedTime(kernel_ms, ch->ev0, ch->ev1));
  if (v != ~0ull) {
    if (first_bad) *first_bad = (int64_t)(v >> 2) + (int64_t)ch->first_index;
    if (bad_kind) *bad_kind = (int32_t)(v & 3);
  }
  return FEI_OK;
}

extern "C" int fei_chain_validate_msgs(const uint8_t* msgs, const uint64_t* msg_off,
                                       const uint8_t* hash, const uint64_t* hash_off,
                                       const uint8_t* prev, const uint64_t* prev_off,
                                       uint64_t n, uint64_t first_index,
                                       int64_t* first_bad, int32_t* bad_kind, uint8_t* digests) {
  // one-shot calls (MemoryChain.validate_chain on Python block objects, receive_chain_update) reuse one scratch chain:
  // its device buffers only grow, so a validation costs copies and kernels, not a dozen cudaMalloc / cudaFree pairs
  std::lock_guard<std::mutex> lk(g_scratch_mu);
  if (!g_scratch) FEI_TRY(fei_chain_create(&g_scratch));
  const bool dbg = getenv("FEI_DEBUG_TIMING") != nullptr;
  auto t0 = std::chrono::steady_clock::now();
  int rc = fei_chain_load_msgs(g_scratch, msgs, msg_off, hash, hash_off, prev, prev_off, n, first_index);
  auto t1 = std::chrono::steady_clock::now();
  if (rc == FEI_OK) rc = fei_chain_validate(g_scratch, first_bad, bad_kind, digests, nullptr);
  if (dbg) fprintf(stderr, "[feiscan] chain load (H2D + pad + links): %.2f ms, validate: %.2f ms\n", std::chrono::duration<double, std::milli>(t1 - t0).count(),
                   std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count());
  if (g_scratch->padded.bytes + g_scratch->msgs.bytes > (2ull << 30)) { fei_chain_destroy(g_scratch); g_scratch = nullptr; }   // do not sit on GBs
  return rc;
}

namespace fei {
void chain_release_scratch() {
  std::lock_guard<std::mutex> lk(g_scratch_mu);
  if (g_scratch) { fei_chain_destroy(g_scratch); g_scratch = nullptr; }
}
}

extern "C" int fei_chain_validate_cols(const fei_json_col* cols, const uint8_t* hash, const uint64_t* hash_off,
                                       uint64_t n, uint64_t first_index,
                                       int64_t* first_bad, int32_t* bad_kind, uint8_t* digests,
                                       uint8_t* msgs_out, uint64_t msgs_cap, uint64_t* msg_off_out) {
  FEI_TRY(require_ready());
  if (!cols || !hash_off) { set_error("null argument"); return FEI_E_BADARG; }
  ByteVec msgs; std::vector<uint64_t> off;
  const bool dbg = getenv("FEI_DEBUG_TIMING") != nullptr;
  auto t0 = std::chrono::steady_clock::now();
  FEI_TRY(serialize_chain_cols(cols, n, msgs, off));
  if (dbg) fprintf(stderr, "[feiscan] serialize_chain_cols: %.2f ms for %llu blocks, %zu bytes\n",
                   std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(), (unsigned long long)n, msgs.size());
  if (msg_off_out) memcpy(msg_off_out, off.data(), (n + 1) * sizeof(uint64_t));
  if (msgs_out) {
    if (msgs.size() > msgs_cap) { set_error("message buffer too small: need %zu bytes", msgs.size()); return FEI_E_CAPACITY; }
    if (!msgs.empty()) memcpy(msgs_out, msgs.data(), msgs.size());
  }
  // previous_hash strings come from column 4 (must be strings to ever equal a stored hash;
  // non-string values are rendered as their JSON text, which never equals a hexdigest)
  const fei_json_col& pc = cols[4];
  std::vector<uint8_t> prev_blob; std::vector<uint64_t> prev_off(n + 1, 0);
  const uint8_t* prev_ptr; const uint64_t* prev_off_ptr;
  bool all_str = !pc.tag && pc.uniform_tag == FEI_J_STR;
  if (all_str) { prev_ptr = pc.str; prev_off_ptr = pc.str_off; }
  else {
    for (uint64_t i = 0; i < n; ++i) {
      int tag = pc.tag ? pc.tag[i] : pc.uniform_tag;
      if (tag == FEI_J_STR) prev_blob.insert(prev_blob.end(), pc.str + pc.str_off[i], pc.str + pc.str_off[i + 1]);
      else prev_blob.push_back(0xFF);   // not a str: can never equal a stored hash string
      prev_off[i + 1] = prev_blob.size();
    }
    prev_ptr = prev_blob.data(); prev_off_ptr = prev_off.data();
  }
  std::vector<uint64_t> prev_rebased;
  if (n && prev_off_ptr[0] != 0) {
    prev_rebased.resize(n + 1);
    for (uint64_t i = 0; i <= n; ++i) prev_rebased[i] = prev_off_ptr[i] - prev_off_ptr[0];
    prev_ptr += prev_off_ptr[0]; prev_off_ptr = prev_rebased.data();
  }
  return fei_chain_validate_msgs(msgs.data(), off.data(), hash, hash_off, prev_ptr, prev_off_ptr, n, first_index, first_bad, bad_kind, digests);
}

// ---------------------------------------------------------------- canonical JSON of the column form on the GPU
// One thread per block serialises the ten hashed fields (jsonfmt.cuh: json.dumps(..., sort_keys=True) incl. the shortest
// round-trip float repr) -- a counting pass, a prefix sum, a writing pass -- straight into the resident chain's message blob: the
// host ships typed columns (~100 B per block) instead of building and copying 360-byte texts (memorychain.py:117-128).
namespace fei {
struct DevCols { fei_json_col c[FEI_CHAIN_NCOLS]; };

__global__ void __launch_bounds__(128) k_json_size(DevCols cols, uint64_t n, uint32_t* __restrict__ len, int* __restrict__ err) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  feijson::CountSink s;
  if (feijson::put_block(s, cols.c, i) != 0) atomicExch(err, 1);
  len[i] = s.n;
}
__global__ void __launch_bounds__(128) k_json_write(DevCols cols, uint64_t n, const uint64_t* __restrict__ off, uint8_t* __restrict__ out) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  feijson::WriteSink s{out + off[i]};
  feijson::put_block(s, cols.c, i);
}
}  // namespace fei

/* Resident chain from the column form (fei_chain_validate_cols' layout): typed columns are uploaded, the canonical JSON texts are
 * produced on the GPU, then padded and linked like fei_chain_load_msgs does.  previous_hash must be all strings (column 4).      */
extern "C" int fei_chain_load_cols(fei_chain* ch, const fei_json_col* cols, const uint8_t* hash, const uint64_t* hash_off, uint64_t n, uint64_t first_index) {
  FEI_TRY(require_ready());
  if (!ch || !cols || !hash_off) { set_error("null argument"); return FEI_E_BADARG; }
  Context& c = ctx();
  cudaStream_t s = c.stream;
  ch->n = n; ch->first_index = first_index; ch->msg_bytes = 0;
  if (n == 0) return FEI_OK;
  const fei_json_col& pc = cols[4];
  if (pc.tag || pc.uniform_tag != FEI_J_STR) { set_error("previous_hash column must hold strings only for the resident column form"); return FEI_E_UNSUPPORTED; }
  DevCols dc;
  std::vector<std::vector<uint64_t>> rebased(FEI_CHAIN_NCOLS);
  for (int k = 0; k < FEI_CHAIN_NCOLS; ++k) {
    const fei_json_col& h = cols[k];
    fei_json_col d; d.tag = nullptr; d.uniform_tag = h.uniform_tag; d.num = nullptr; d.str = nullptr; d.str_off = nullptr;
    if (!h.tag && (h.uniform_tag < FEI_J_NULL || h.uniform_tag > FEI_J_BIGINT)) { set_error("column %d: bad uniform tag %d", k, h.uniform_tag); return FEI_E_BADARG; }
    if (h.tag) { FEI_TRY(upload(ch->col_tag[k], h.tag, n, 0, s)); d.tag = ch->col_tag[k].as<uint8_t>(); }
    if (h.num) { FEI_TRY(upload(ch->col_num[k], h.num, n * 8, 0, s)); d.num = ch->col_num[k].as<uint64_t>(); }
    if (h.str_off) {
      const uint64_t base = h.str_off[0];
      const uint64_t* off = h.str_off;
      if (base) { rebased[k].resize(n + 1); for (uint64_t i = 0; i <= n; ++i) rebased[k][i] = h.str_off[i] - base; off = rebased[k].data(); }
      FEI_TRY(upload(ch->col_off[k], off, (n + 1) * 8, 0, s));
      FEI_TRY(upload(ch->col_str[k], h.str ? h.str + base : nullptr, h.str ? h.str_off[n] - base : 0, 0, s));
      d.str = ch->col_str[k].as<uint8_t>(); d.str_off = ch->col_off[k].as<uint64_t>();
    }
    dc.c[k] = d;
  }
  FEI_TRY(ch->json_len.ensure(n * 4));
  FEI_TRY(ch->json_err.ensure(16));
  FEI_CUDA(cudaMemsetAsync(ch->json_err.p, 0, 4, s));
  FEI_TRY(ch->msg_off.ensure((n + 1) * 8));
  const unsigned g = (unsigned)((n + 127) / 128);
  k_json_size<<<g, 128, 0, s>>>(dc, n, ch->json_len.as<uint32_t>(), ch->json_err.as<int>());
  FEI_TRY(exclusive_scan_u32_u64(ch->json_len.as<uint32_t>(), n, ch->msg_off.as<uint64_t>(), ch->scan_tmp, s));
  uint64_t total = 0; int err = 0;
  FEI_CUDA(cudaMemcpyAsync(&total, ch->msg_off.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaMemcpyAsync(&err, ch->json_err.p, 4, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));                               // (also: the rebased offset vectors may go now)
  if (err) { set_error("unsupported JSON tag in chain columns"); return FEI_E_BADARG; }
  ch->msg_bytes = total;
  FEI_TRY(ch->msgs.ensure(total + 16));
  k_json_write<<<g, 128, 0, s>>>(dc, n, ch->msg_off.as<uint64_t>(), ch->msgs.as<uint8_t>());
  FEI_CUDA(cudaGetLastError());
  FEI_TRY(upload(ch->hash, hash, hash_off[n], 0, s));
  FEI_TRY(upload(ch->hash_off, hash_off, (n + 1) * 8, 0, s));
  // previous_hash strings = column 4, already on the device
  FEI_TRY(ch->prev.ensure(ch->col_str[4].bytes ? ch->col_str[4].bytes : 16));
  FEI_TRY(ch->prev_off.ensure((n + 1) * 8));
  const uint64_t pbytes = cols[4].str_off[n] - cols[4].str_off[0];
  if (pbytes) FEI_CUDA(cudaMemcpyAsync(ch->prev.p, ch->col_str[4].p, pbytes, cudaMemcpyDeviceToDevice, s));
  FEI_CUDA(cudaMemcpyAsync(ch->prev_off.p, ch->col_off[4].p, (n + 1) * 8, cudaMemcpyDeviceToDevice, s));
  return chain_prepare(ch);
}

extern "C" int fei_chain_fetch(fei_chain* ch, uint64_t first, uint64_t n, uint8_t* msgs, uint64_t msgs_cap, uint64_t* msg_off,
                               uint8_t* hash_hex, uint8_t* prev_hex) {
  FEI_TRY(require_ready());
  if (!ch || first + n > ch->n) { set_error("range out of bounds"); return FEI_E_BADARG; }
  Context& c = ctx();
  std::vector<uint64_t> off(n + 1), hoff(n + 1), poff(n + 1);
  FEI_CUDA(cudaMemcpyAsync(off.data(), ch->msg_off.as<uint64_t>() + first, (n + 1) * 8, cudaMemcpyDeviceToHost, c.stream));
  FEI_CUDA(cudaMemcpyAsync(hoff.data(), ch->hash_off.as<uint64_t>() + first, (n + 1) * 8, cudaMemcpyDeviceToHost, c.stream));
  FEI_CUDA(cudaMemcpyAsync(poff.data(), ch->prev_off.as<uint64_t>() + first, (n + 1) * 8, cudaMemcpyDeviceToHost, c.stream));
  FEI_CUDA(cudaStreamSynchronize(c.stream));
  uint64_t bytes = off[n] - off[0];
  if (msgs) {
    if (bytes > msgs_cap) { set_error("message buffer too small: need %llu bytes", (unsigned long long)bytes); return FEI_E_CAPACITY; }
    FEI_CUDA(cudaMemcpyAsync(msgs, ch->msgs.as<uint8_t>() + off[0], bytes, cudaMemcpyDeviceToHost, c.stream));
  }
  if (msg_off) for (uint64_t i = 0; i <= n; ++i) msg_off[i] = off[i] - off[0];
  if (hash_hex) {
    if (hoff[n] - hoff[0] != 64 * n) { set_error("stored hashes are not all 64 characters"); return FEI_E_UNSUPPORTED; }
    FEI_CUDA(cudaMemcpyAsync(hash_hex, ch->hash.as<uint8_t>() + hoff[0], 64 * n, cudaMemcpyDeviceToHost, c.stream));
  }
  if (prev_hex) {
    if (poff[n] - poff[0] != 64 * n) { set_error("previous hashes are not all 64 characters"); return FEI_E_UNSUPPORTED; }
    FEI_CUDA(cudaMemcpyAsync(prev_hex, ch->prev.as<uint8_t>() + poff[0], 64 * n, cudaMemcpyDeviceToHost, c.stream));
  }
  FEI_CUDA(cudaStreamSynchronize(c.stream));
  return FEI_OK;
}

extern "C" int fei_chain_mine(const uint8_t* prefix, uint32_t prefix_len, const uint8_t* suffix, uint32_t suffix_len,
                              uint64_t start_nonce, uint32_t difficulty, uint64_t max_tries,
                              uint64_t* nonce_out, uint8_t* digest_out, uint64_t* tried_out) {
  FEI_TRY(require_ready());
  if (!nonce_out || (prefix_len && !prefix) || (suffix_len && !suffix)) { set_error("null argument"); return FEI_E_BADARG; }
  if (prefix_len + suffix_len > kMineMaxFixed) { set_error("block text longer than %d bytes is not supported by the miner", kMineMaxFixed); return FEI_E_UNSUPPORTED; }
  if (difficulty > 64) { set_error("difficulty above 64 hex digits can never be met"); return FEI_E_BADARG; }
  Context& c = ctx();
  cudaStream_t s = c.stream;
  DevBuf fixed, best;
  FEI_TRY(fixed.alloc(kMineMaxFixed)); FEI_TRY(best.alloc(16));
  std::vector<uint8_t> host(prefix_len + suffix_len + 1);
  if (prefix_len) memcpy(host.data(), prefix, prefix_len);
  if (suffix_len) memcpy(host.data() + prefix_len, suffix, suffix_len);
  FEI_CUDA(cudaMemcpyAsync(fixed.p, host.data(), prefix_len + suffix_len, cudaMemcpyHostToDevice, s));
  FEI_CUDA(cudaMemsetAsync(best.p, 0xFF, sizeof(unsigned long long), s));
  const unsigned long long batch = 1ull << 22;
  unsigned long long tried = 0, found = ~0ull, base = start_nonce;
  while (tried < max_tries) {
    unsigned long long cnt = max_tries - tried < batch ? max_tries - tried : batch;
    if (base + cnt < base) cnt = ~0ull - base;             // do not wrap the 64-bit nonce space
    if (cnt == 0) break;
    k_mine<<<c.sm_count * 8, 256, 0, s>>>(fixed.as<uint8_t>(), prefix_len, suffix_len, base, cnt, difficulty, best.as<unsigned long long>());
    FEI_CUDA(cudaGetLastError());
    FEI_CUDA(cudaMemcpyAsync(&found, best.p, sizeof(found), cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaStreamSynchronize(s));
    tried += cnt; base += cnt;
    if (found != ~0ull) break;
  }
  if (tried_out) *tried_out = tried;
  if (found == ~0ull) { set_error("no nonce found within %llu tries", (unsigned long long)max_tries); return FEI_E_CAPACITY; }
  *nonce_out = found;
  if (digest_out) {                                        // hash of the winning text, through the validate kernel's path
    char dg[24]; int nd = snprintf(dg, sizeof dg, "%llu", found);
    std::vector<uint8_t> msg(prefix_len + nd + suffix_len);
    if (prefix_len) memcpy(msg.data(), prefix, prefix_len);
    memcpy(msg.data() + prefix_len, dg, nd);
    if (suffix_len) memcpy(msg.data() + prefix_len + nd, suffix, suffix_len);
    uint64_t moff[2] = {0, msg.size()}, hoff[2] = {0, 1};
    uint8_t dummy = '0';
    int64_t fb; int32_t kind;
    FEI_TRY(fei_chain_validate_msgs(msg.data(), moff, &dummy, hoff, &dummy, hoff, 1, 0, &fb, &kind, digest_out));
  }
  return FEI_OK;
}
