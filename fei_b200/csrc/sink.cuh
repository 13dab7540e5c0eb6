// Byte sinks for the writers that run twice over an item, once with CountSink to size it and once with WriteSink to write it at
// its offset (the device calls that return text, the host copies of the chain JSON and the synthetic records).  Host and device.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define FEI_HD __host__ __device__ __forceinline__
#define FEI_HD_NI __host__ __device__ inline
#else
#define FEI_HD inline
#define FEI_HD_NI inline
#endif

namespace fei {

struct CountSink {
  uint32_t n = 0;
  FEI_HD void put(uint8_t) { ++n; }
  FEI_HD void put(const uint8_t*, uint32_t l) { n += l; }
};
// p advances past every byte written: after a writer ran, p is the end of what it wrote
struct WriteSink {
  uint8_t* p;
  FEI_HD void put(uint8_t c) { *p++ = c; }
  FEI_HD void put(const uint8_t* s, uint32_t l) { for (uint32_t k = 0; k < l; ++k) *p++ = s[k]; }
};

template <class S> FEI_HD void put_lit(S& o, const char* s) { while (*s) o.put((uint8_t)*s++); }
template <class S> FEI_HD void put_bytes(S& o, const uint8_t* s, uint64_t n) { for (uint64_t i = 0; i < n; ++i) o.put(s[i]); }

}  // namespace fei
