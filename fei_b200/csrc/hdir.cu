// Header directory, built once at pack time (fei_corpus_load / load_raw / synth):
// for every record, one entry per header line that holds a colon, in line order -- the dict that utils.py:113-118
// builds (`for line in header.split("\n"): if ":" in line: key, value = line.split(":", 1);
// headers[key.strip()] = value.strip()`), minus the dict's collapsing of repeated keys, which depends on the queried
// field and stays in the scan (header_lookup in scan.cu).  Keys are interned: the corpus keeps a dictionary of its distinct
// stripped key spellings (a few dozen in a real Memdir) and an entry names its key by dictionary slot, so a scan
// runs the key automaton once per distinct key (k_key_lut) instead of once per header line of every record, and then
// touches only the one value it needs.
#include "corpus.h"
#include "pyws.cuh"
#include <stdlib.h>
#include <vector>

namespace fei {

// entry.x = key slot | val_len << 16, entry.y = val_off (offset of the stripped value from the start of the record's
// header text).  Headers longer than 65535 bytes get the single entry text_record_entry(): "parse the text".
__device__ __forceinline__ unsigned long long key_hash(const uint8_t* p, uint32_t n) {
  unsigned long long h = 0xcbf29ce484222325ull;                       // FNV-1a, then a finaliser
  for (uint32_t i = 0; i < n; ++i) { h ^= p[i]; h *= 0x100000001b3ull; }
  h ^= h >> 29; h *= 0xbf58476d1ce4e5b9ull; h ^= h >> 32;
  return h | 1ull;                                                    // 0 marks an empty slot
}

struct KeyDict { unsigned long long* tag; unsigned long long* rep; uint32_t* len; uint32_t* flag; uint32_t* cnt; };

// slot of `h` (inserting it if new); ~0u when the table is over-full
__device__ __forceinline__ uint32_t key_slot(const KeyDict& d, unsigned long long h, bool insert) {
  uint32_t s = (uint32_t)(h >> 17) & (kKeySlots - 1);
  for (uint32_t probe = 0; probe < kKeySlots / 2; ++probe, s = (s + 1) & (kKeySlots - 1)) {
    unsigned long long t = d.tag[s];
    if (t == h) return s;
    if (t == 0) {
      if (!insert) return 0xFFFFFFFFu;
      t = atomicCAS(d.tag + s, 0ull, h);
      if (t == 0 || t == h) return s;
    }
  }
  return 0xFFFFFFFFu;
}

// kPass 0: count the entries of every record and intern the keys.  kPass 1: write the entries, checking every key
// against its slot's representative spelling (a 64-bit hash collision would set flag bit 1 and the directory is
// rebuilt as "parse the text" for everybody).
template <int kPass>
__global__ void __launch_bounds__(256) k_hdir(const uint8_t* __restrict__ hdr, const uint64_t* __restrict__ hdr_off, uint64_t n,
                                              uint32_t* __restrict__ cnt, const uint64_t* __restrict__ dir_off, uint2* __restrict__ dir,
                                              KeyDict kd, bool force_text) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* h = hdr + hdr_off[i];
  const uint64_t hlen = hdr_off[i + 1] - hdr_off[i];
  uint2* out = kPass ? dir + dir_off[i] : nullptr;
  if (hlen > 65535 || force_text) {
    if (kPass) out[0] = text_record_entry(); else { cnt[i] = 1; kd.cnt[kKeySlots] = 1u; }   // [kKeySlots]: some record's keys are not in the dictionary
    return;
  }
  uint32_t k = 0;
  HeaderLine l;
  for (const uint8_t* p = h; p < h + hlen;) {
    if (!next_header_line(p, h + hlen, l)) continue;
    const uint32_t klen = (uint32_t)(l.kb - l.ka);
    const unsigned long long kh = key_hash(l.ka, klen);
    if (!kPass) {
      const uint32_t s = key_slot(kd, kh, true);
      if (s == 0xFFFFFFFFu) atomicOr(kd.flag, 1u);
      else {
        const unsigned long long at = (unsigned long long)(l.ka - hdr);
        if (at < kd.rep[s]) atomicMin(kd.rep + s, at);                   // representative = smallest offset; the plain read skips almost every atomic
        kd.len[s] = klen;                                                // same hash => same length unless colliding (checked in pass 1)
        if ((i & 63) == 0) atomicAdd(kd.cnt + s, 1u);                    // sampled frequency: which keys deserve a value column
      }
    } else {
      const uint32_t s = key_slot(kd, kh, false);
      bool same = s != 0xFFFFFFFFu && kd.len[s] == klen;
      if (same) { const uint8_t* r = hdr + kd.rep[s]; for (uint32_t b = 0; same && b < klen; ++b) same = r[b] == l.ka[b]; }
      if (!same) atomicOr(kd.flag, 2u);
      out[k] = make_uint2((s & 0xFFFFu) | (uint32_t)(l.vb - l.va) << 16, (uint32_t)(l.va - h));
    }
    ++k;
  }
  if (!kPass) cnt[i] = k;
}

// ---------------------------------------------------------------- value columns
// Thread per record: for every directory entry whose key has a column, store the value (the last line with that key wins,
// like the dict assignment of utils.py:118) as 16-byte units in the column's planes.
__global__ void __launch_bounds__(256) k_hdir_cols(const uint8_t* __restrict__ hdr, const uint64_t* __restrict__ hdr_off, uint64_t n,
                                                   const uint2* __restrict__ dir, const uint64_t* __restrict__ dir_off,
                                                   const int8_t* __restrict__ kid_col, uint32_t n_cols,
                                                   uint16_t* __restrict__ col_len, uint8_t* __restrict__ planes) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint2* ent = dir + dir_off[i];
  const uint32_t n_ent = (uint32_t)(dir_off[i + 1] - dir_off[i]);
  if (text_record(ent, n_ent)) {                                        // every column defers to the walk
    for (uint32_t c = 0; c < n_cols; ++c) col_len[(uint64_t)c * n + i] = kColWalk;
    return;
  }
  const uint8_t* h = hdr + hdr_off[i];
  for (uint32_t j = 0; j < n_ent; ++j) {
    const uint2 e = ent[j];
    const int c = kid_col[e.x & 0xFFFFu];
    if (c < 0) continue;
    const uint32_t len = e.x >> 16;
    if (len > kColUnits * 16) { col_len[(uint64_t)c * n + i] = kColWalk; continue; }
    col_len[(uint64_t)c * n + i] = (uint16_t)len;
    uint8_t* base = planes + (uint64_t)c * kColUnits * n * 16 + i * 16;
    for (uint32_t k = 0; k * 16 < len; ++k)
      *reinterpret_cast<uint4*>(base + (uint64_t)k * n * 16) = load16(h + e.y + k * 16);     // bytes past `len` are never looked at
  }
}

static int build_value_columns(fei_corpus* c, const uint32_t* d_cnt, bool no_directory, cudaStream_t s) {
  const uint64_t n = c->n;
  c->n_cols = 0;
  const char* env = getenv("FEI_HCOLS");
  if (no_directory || n == 0 || (env && env[0] == '0')) return FEI_OK;
  // keys that (by the 1-in-64 sample of pass 0) at least every 8th record carries, most frequent first
  std::vector<uint32_t> cnt(kKeySlots);
  FEI_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt, kKeySlots * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  std::vector<int8_t> kid_col(kKeySlots, (int8_t)-1);
  const uint64_t sampled = (n + 63) / 64;
  for (uint32_t col = 0; col < kMaxCols; ++col) {
    uint32_t best = 0, arg = 0;
    for (uint32_t k = 0; k < kKeySlots; ++k) if (kid_col[k] < 0 && cnt[k] > best) { best = cnt[k]; arg = k; }
    if (best == 0 || (uint64_t)best * 8 < sampled) break;
    kid_col[arg] = (int8_t)col; c->n_cols = col + 1;
  }
  FEI_TRY(c->kid_col.ensure(kKeySlots));
  FEI_CUDA(cudaMemcpyAsync(c->kid_col.p, kid_col.data(), kKeySlots, cudaMemcpyHostToDevice, s));
  if (c->n_cols == 0) { FEI_CUDA(cudaStreamSynchronize(s)); return FEI_OK; }
  FEI_TRY(c->col_len.ensure((uint64_t)c->n_cols * n * sizeof(uint16_t)));
  FEI_TRY(c->col_planes.ensure((uint64_t)c->n_cols * kColUnits * n * 16 + 64));
  FEI_CUDA(cudaMemsetAsync(c->col_len.p, 0xFF, (uint64_t)c->n_cols * n * sizeof(uint16_t), s));      // kColAbsent
  k_hdir_cols<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), n, c->hdir.as<uint2>(), c->hdir_off.as<uint64_t>(),
                                                          c->kid_col.as<int8_t>(), c->n_cols, c->col_len.as<uint16_t>(), c->col_planes.as<uint8_t>());
  FEI_CUDA(cudaGetLastError());
  FEI_CUDA(cudaStreamSynchronize(s));      // kid_col (host vector) must outlive the copy
  return FEI_OK;
}

int build_header_dir(fei_corpus* c, cudaStream_t s) {
  const uint64_t n = c->n;
  FEI_TRY(c->hdir_off.ensure((n + 1) * sizeof(uint64_t)));
  FEI_TRY(c->key_tag.ensure(kKeySlots * sizeof(unsigned long long)));
  FEI_TRY(c->key_rep.ensure(kKeySlots * sizeof(unsigned long long)));
  FEI_TRY(c->key_len.ensure((2 * kKeySlots + 2) * sizeof(uint32_t)));      // len[kKeySlots], flag word, sampled count[kKeySlots], text-record word
  if (n == 0) { FEI_CUDA(cudaMemsetAsync(c->hdir_off.p, 0, sizeof(uint64_t), s)); c->hdir_entries = 0; return FEI_OK; }
  DevBuf& cnt = c->tmp_len;
  FEI_TRY(cnt.ensure(n * sizeof(uint32_t)));
  const unsigned blocks = (unsigned)((n + 255) / 256);
  // FEI_HDIR=0 (read at load time): mark every record "parse the text", so tests can hold the in-scan text parser
  // (normally only reached by > 64 KiB headers) against the directory path on the same corpus
  const char* env = getenv("FEI_HDIR");
  bool force_text = env && env[0] == '0';
  KeyDict kd{c->key_tag.as<unsigned long long>(), c->key_rep.as<unsigned long long>(), c->key_len.as<uint32_t>(), c->key_len.as<uint32_t>() + kKeySlots,
             c->key_len.as<uint32_t>() + kKeySlots + 1};
  for (int attempt = 0; attempt < 2; ++attempt) {
    FEI_CUDA(cudaMemsetAsync(kd.tag, 0, kKeySlots * sizeof(unsigned long long), s));
    FEI_CUDA(cudaMemsetAsync(kd.rep, 0xFF, kKeySlots * sizeof(unsigned long long), s));
    FEI_CUDA(cudaMemsetAsync(kd.len, 0, (2 * kKeySlots + 2) * sizeof(uint32_t), s));
    k_hdir<0><<<blocks, 256, 0, s>>>(c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), n, cnt.as<uint32_t>(), nullptr, nullptr, kd, force_text);
    uint64_t total = 0;
    FEI_TRY(queue_offsets(cnt.as<uint32_t>(), n, c->hdir_off.as<uint64_t>(), &total, false, c->scan_tmp, s));
    FEI_CUDA(cudaStreamSynchronize(s));
    c->hdir_entries = total;
    FEI_TRY(c->hdir.ensure((total + 1) * sizeof(uint2)));
    k_hdir<1><<<blocks, 256, 0, s>>>(c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), n, nullptr, c->hdir_off.as<uint64_t>(), c->hdir.as<uint2>(), kd, force_text);
    uint32_t flag = 0, any_text = 0;
    FEI_CUDA(cudaMemcpyAsync(&any_text, kd.cnt + kKeySlots, 4, cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaMemcpyAsync(&flag, kd.flag, 4, cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaStreamSynchronize(s));
    FEI_CUDA(cudaGetLastError());
    c->has_text_records = any_text != 0;
    if (flag == 0 || force_text) break;
    force_text = true;      // more than kKeySlots / 2 distinct keys, or a 64-bit hash collision: no directory for this corpus
  }
  return build_value_columns(c, kd.cnt, force_text, s);
}

}  // namespace fei
