// Threaded host driver for the canonical-JSON writer of Memorychain blocks (jsonfmt.cuh), in chain_json.cpp.
#pragma once
#include <stdint.h>
#include <vector>
#include "../../include/feiscan.h"

#include <cstdlib>
#include <new>
#include <utility>

namespace fei {
// byte vector whose resize() does not zero-fill (the serialiser overwrites every byte; tens of MB per call)
template <class T> struct NoInitAlloc {
  using value_type = T;
  NoInitAlloc() = default;
  template <class U> NoInitAlloc(const NoInitAlloc<U>&) {}
  T* allocate(size_t n) { void* p = malloc(n * sizeof(T)); if (!p) throw std::bad_alloc(); return (T*)p; }
  void deallocate(T* p, size_t) { free(p); }
  template <class U> void construct(U* p) { (void)p; }                                   // default-init: leave as is
  template <class U, class A0, class... A> void construct(U* p, A0&& a0, A&&... a) { ::new ((void*)p) U(std::forward<A0>(a0), std::forward<A>(a)...); }
  template <class U> bool operator==(const NoInitAlloc<U>&) const { return true; }
  template <class U> bool operator!=(const NoInitAlloc<U>&) const { return false; }
};
using ByteVec = std::vector<uint8_t, NoInitAlloc<uint8_t>>;

// msgs = concatenated canonical JSON texts, off[n+1] = offsets.  Returns FEI_OK or FEI_E_*.
int serialize_chain_cols(const fei_json_col* cols, uint64_t n, ByteVec& msgs, std::vector<uint64_t>& off);
}
