// Canonical JSON of Memorychain blocks on the host, multi-threaded; the GPU then hashes the texts (chain.cu).  Every block
// goes through the writer in jsonfmt.cuh, the source chain.cu's k_json_* kernels format the resident image with, so
// one-shot and resident validation hash the same bytes.
#include "common.h"
#include "chain_json.h"
#include "jsonfmt.cuh"

#include <cstring>
#include <cstdlib>
#include <thread>
#include <vector>
#include <algorithm>

namespace fei {

// upper bound of one block's text: every string byte can become a 6-byte \\uXXXX escape (a 4-byte character two of them)
static size_t block_bound(const fei_json_col* cols, uint64_t i) {
  size_t b = 2 + FEI_CHAIN_NCOLS * 56;                          // braces; per field: ", " + quoted key (<= 18) + ": " + a number / literal (<= 26 chars)
  for (int k = 0; k < FEI_CHAIN_NCOLS; ++k) {
    const fei_json_col& c = cols[k];
    const int tag = c.tag ? c.tag[i] : c.uniform_tag;
    if (tag == FEI_J_STR || tag == FEI_J_BIGINT) b += 6 * (size_t)(c.str_off[i + 1] - c.str_off[i]) + 2;
  }
  return b;
}

// One block's text at dst; returns its end, or nullptr on an unsupported tag.  flatten inlines the whole writer so the sink's
// pointer can live in a register; otherwise every byte store, which may alias the pointer, forces a store and reload of it.
__attribute__((flatten)) static uint8_t* write_block(uint8_t* dst, const fei_json_col* cols, uint64_t i) {
  WriteSink o{dst};
  return feijson::put_block(o, cols, i) == 0 ? o.p : nullptr;
}

int serialize_chain_cols(const fei_json_col* cols, uint64_t n, ByteVec& msgs, std::vector<uint64_t>& off) {
  for (int k = 0; k < FEI_CHAIN_NCOLS; ++k) {
    const fei_json_col& c = cols[k];
    if (!c.tag && (c.uniform_tag < FEI_J_NULL || c.uniform_tag > FEI_J_BIGINT)) { set_error("column %d (%s): bad uniform tag %d", k, feijson::key_name(k), c.uniform_tag); return FEI_E_BADARG; }
  }
  unsigned hw = std::thread::hardware_concurrency();
  unsigned nt = (unsigned)std::min<uint64_t>(std::min(std::max(1u, hw), 32u), std::max<uint64_t>(1, n / 4096));
  // each worker writes into its own malloc'ed buffer (no zero fill), grown by doubling with the block bound as the guard
  struct Part { uint8_t* buf = nullptr; size_t len = 0, cap = 0; };
  std::vector<Part> parts(nt);
  std::vector<int> rc(nt, 0);
  off.assign(n + 1, 0);
  auto work = [&](unsigned t) {
    uint64_t lo = n * t / nt, hi = n * (t + 1) / nt;
    Part& pt = parts[t];
    pt.cap = (hi - lo) * 400 + 4096;
    pt.buf = (uint8_t*)malloc(pt.cap);
    if (!pt.buf) { rc[t] = -2; return; }
    for (uint64_t i = lo; i < hi; ++i) {
      const size_t need = block_bound(cols, i);
      if (pt.len + need > pt.cap) {
        size_t ncap = std::max(pt.cap * 2, pt.len + need);
        uint8_t* nb = (uint8_t*)realloc(pt.buf, ncap);
        if (!nb) { rc[t] = -2; return; }
        pt.buf = nb; pt.cap = ncap;
      }
      const uint8_t* end = write_block(pt.buf + pt.len, cols, i);
      if (!end) { rc[t] = -1; return; }
      const size_t wrote = (size_t)(end - (pt.buf + pt.len));
      off[i + 1] = wrote;                                       // length for now; prefix-summed below
      pt.len += wrote;
    }
  };
  if (nt == 1) work(0);
  else {
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; ++t) th.emplace_back(work, t);
    for (auto& x : th) x.join();
  }
  int bad = 0;
  for (unsigned t = 0; t < nt; ++t) if (rc[t]) bad = rc[t];
  if (bad) {
    for (auto& pt : parts) free(pt.buf);
    if (bad == -2) { set_error("out of host memory serialising the chain"); return FEI_E_CAPACITY; }
    set_error("unsupported JSON tag in chain columns"); return FEI_E_BADARG;
  }
  for (uint64_t i = 0; i < n; ++i) off[i + 1] += off[i];
  msgs.resize(off[n]);
  {
    std::vector<std::thread> th;
    auto copy = [&](unsigned t) { uint64_t lo = n * t / nt; if (parts[t].len) memcpy(msgs.data() + off[lo], parts[t].buf, parts[t].len); free(parts[t].buf); };
    if (nt == 1) copy(0);
    else { for (unsigned t = 0; t < nt; ++t) th.emplace_back(copy, t); for (auto& x : th) x.join(); }
  }
  return FEI_OK;
}

}  // namespace fei

extern "C" int fei_chain_serialize_cols(const fei_json_col* cols, uint64_t n, uint8_t* msgs_out, uint64_t msgs_cap, uint64_t* msg_off_out) {
  if (!cols || !msg_off_out) { fei::set_error("null argument"); return FEI_E_BADARG; }
  fei::ByteVec msgs; std::vector<uint64_t> off;
  int rc = fei::serialize_chain_cols(cols, n, msgs, off);
  if (rc != FEI_OK) return rc;
  memcpy(msg_off_out, off.data(), (n + 1) * sizeof(uint64_t));
  if (msgs.size() > msgs_cap) { fei::set_error("message buffer too small: need %zu bytes", msgs.size()); return FEI_E_CAPACITY; }
  if (msgs_out && !msgs.empty()) memcpy(msgs_out, msgs.data(), msgs.size());
  return FEI_OK;
}
