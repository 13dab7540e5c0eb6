// Raw ingest ("next" row 1 of SURVEY.md 8(f)): file bytes -> packed corpus, on the GPU.
//
// Replaces the per-file text work of utils.list_memories + parse_memory_content
// (memdir_tools/utils.py:229-232, :97-120) that the host packer otherwise does in Python:
//   open(path, "r").read()      -> strict UTF-8 validation (an undecodable file is reported and
//                                  skipped, utils.py:247-248) + universal-newline translation
//                                  ("\r\n" and lone "\r" become "\n")
//   content.split("---", 1)     -> first "---" anywhere in the text (utils.py:105)
//   body.strip()                -> Python's str.strip() whitespace set (utils.py:109,120)
// plus the record bits the scan needs (no separator / non-ASCII / context-dependent str.lower()).
// The host keeps the directory walk, the file-name grammar and the listing order.
//
// k_raw_measure : one warp per file: validate + measure the normalised header / stripped body (the file is read once, coalesced).
// k_raw_write   : one warp per valid file: write normalised header text and stripped body into
//                 the canonical blobs (offsets from an exclusive scan over the valid files), 16-byte stores.
#include "corpus.h"
#include "pyws.cuh"
#include <vector>
#include <string.h>

namespace fei {

// All spans are in RAW bytes.  Universal-newline translation only touches '\r' ("\r\n" -> "\n", lone "\r" -> "\n"),
// never '-' and never the whitespace-ness of a character, so the "---" search and the strip can run on the raw bytes;
// the translated length of a span is its raw length minus the number of "\r\n" pairs inside it (spans start and end at
// non-whitespace bytes or at the separator, so no pair is ever cut).
// summary[0] = files that are not valid UTF-8, summary[1] = 1 + index of the last record whose body exceeds kMaxBodyBytes (0 = none):
// the host needs these two numbers, not the per-record measures
constexpr uint32_t kMaxBodyBytes = 32u << 20;
struct RawMeasure {
  uint32_t hdr_raw_len;               // header = raw[0, hdr_raw_len)
  uint32_t body_raw_begin, body_raw_end;
  uint32_t hdr_len, body_len;         // translated lengths
  uint32_t flags;                     // bit0 valid UTF-8, bit1 has separator, bit2 non-ASCII, bit3 U+03A3 present, bit4 U+0130 present, bit5 a '\r' somewhere
};

// ---- one warp per file.  A file is read once, in rows of 32 x 16 bytes (16-byte aligned, coalesced); every lane also sees the
// 4 bytes before and after its 16 (the neighbours' cache lines), which is all the context the per-byte rules need:
//   strict UTF-8 (what bytes.decode("utf-8") accepts: no overlongs, no surrogates, <= U+10FFFF): a decoder state of
//       (continuation bytes still owed, allowed range of the next one) is a function of the three preceding bytes in valid text,
//       so a lane replays its 3 bytes of context without judging them and then judges its own 16;
//   first "---", "\r\n" pairs before / after it, U+03A3 / U+0130: bit masks over the 16 positions.
// Bytes outside the file are read as 0 (the staging buffer is padded), which is neither '-', '\r', '\n' nor a continuation byte.
__device__ __forceinline__ uint32_t eq4(uint32_t w, uint32_t c4) {       // bit k = (byte k of w == byte of c4), k = 0..3
  uint32_t x = w ^ c4;
  uint32_t t = ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu);     // 0x80 exactly where a byte of x is 0
  return ((t >> 7) * 0x10204080u) >> 28;
}
__device__ __forceinline__ uint32_t keep_bytes(uint32_t w, long long wp, long long o0, long long o1) {   // zero the bytes of the word at offset wp outside [o0, o1)
  long long lo = wp > o0 ? wp : o0, hi = wp + 4 < o1 ? wp + 4 : o1;
  if (hi <= lo) return 0u;
  uint32_t m = 0xFFFFFFFFu;
  m >>= 8 * (4 - (int)(hi - lo));
  m <<= 8 * (int)(lo - wp);
  return w & m;
}
struct Utf8State {
  int owed; uint32_t lo, hi; bool bad;
  __device__ __forceinline__ void feed(uint32_t b, bool judge) {
    if (owed) {
      bool ok = b >= lo && b <= hi;
      if (!ok && judge) bad = true;
      owed = ok ? owed - 1 : 0; lo = 0x80u; hi = 0xBFu;
    } else if (b < 0x80u) {
    } else if (b >= 0xC2u && b <= 0xDFu) { owed = 1; lo = 0x80u; hi = 0xBFu; }
    else if (b >= 0xE0u && b <= 0xEFu) { owed = 2; lo = b == 0xE0u ? 0xA0u : 0x80u; hi = b == 0xEDu ? 0x9Fu : 0xBFu; }   // overlong / surrogates
    else if (b >= 0xF0u && b <= 0xF4u) { owed = 3; lo = b == 0xF0u ? 0x90u : 0x80u; hi = b == 0xF4u ? 0x8Fu : 0xBFu; }   // overlong / > U+10FFFF
    else if (judge) bad = true;                                           // a continuation byte with nothing owed, C0, C1, F5..FF
  }
};

constexpr int kIngestThreads = 256;
constexpr uint64_t kH2DPiece = 64ull << 20;       // = packer._Arena.BLOCK
// raw_len == nullptr: file i = raw[raw_off[i], raw_off[i+1]); else raw[raw_off[i], raw_off[i] + raw_len[i])
__global__ void __launch_bounds__(kIngestThreads) k_raw_measure(const uint8_t* __restrict__ raw, const uint64_t* __restrict__ raw_off,
                                                                 const uint64_t* __restrict__ raw_len, uint64_t n, RawMeasure* __restrict__ out, uint32_t* __restrict__ hdr_len, uint32_t* __restrict__ body_len,
                                                                 unsigned long long* __restrict__ summary) {
  const uint64_t i = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const long long o0 = (long long)raw_off[i], o1 = raw_len ? o0 + (long long)raw_len[i] : (long long)raw_off[i + 1];
  const long long a0 = o0 & ~15ll;
  bool bad = false, nonascii = false, sigma = false, idot = false, any_cr = false;
  long long sep = -1;                                  // offset of the first "---", warp-uniform
  uint32_t pre = 0, post = 0;                          // "\r\n" pairs before the separator (all pairs while none is known) / from 3 bytes after it
  for (long long row = a0; row <= o1; row += 512) {
    const long long c = row + lane * 16;
    uint32_t w[6] = {0, 0, 0, 0, 0, 0};                // w[0]: bytes c-4..c-1, w[1..4]: own, w[5]: c+16..c+19
    if (c + 16 > o0 && c < o1) { uint4 v = *reinterpret_cast<const uint4*>(raw + c); w[1] = v.x; w[2] = v.y; w[3] = v.z; w[4] = v.w; }
    if (c > o0 && c - 4 < o1) w[0] = *reinterpret_cast<const uint32_t*>(raw + c - 4);
    if (c + 20 > o0 && c + 16 < o1) w[5] = *reinterpret_cast<const uint32_t*>(raw + c + 16);
    if (c - 4 < o0 || c + 20 > o1) {
#pragma unroll
      for (int k = 0; k < 6; ++k) w[k] = keep_bytes(w[k], c - 4 + 4 * k, o0, o1);
    }
    // ---- UTF-8: only lanes with a non-ASCII byte in sight (own 16 or the 3 before) run the decoder
    if (((w[0] & 0x80808000u) | ((w[1] | w[2] | w[3] | w[4]) & 0x80808080u)) != 0u) {
      Utf8State st{0, 0x80u, 0xBFu, false};
      st.feed((w[0] >> 8) & 0xFFu, false); st.feed((w[0] >> 16) & 0xFFu, false); st.feed(w[0] >> 24, false);
      uint32_t prev = w[0] >> 24;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const uint32_t b = (w[1 + (k >> 2)] >> (8 * (k & 3))) & 0xFFu;
        if (c + k >= o1) { if (c + k == o1 && st.owed) st.bad = true; st.owed = 0; }   // the file ends inside a sequence
        else {
          st.feed(b, true);
          if (b >= 0x80u) nonascii = true;
          if (prev == 0xCEu && b == 0xA3u) sigma = true;       // U+03A3: lower() depends on the context (final sigma)
          if (prev == 0xC4u && b == 0xB0u) idot = true;        // U+0130: lower() is two characters (handled by the automata)
        }
        prev = b;
      }
      bad |= st.bad;
    }
    // ---- '-', '\r', '\n' masks: bit k = own byte k, bits 16..19 = the 4 bytes after
    uint32_t dash = 0, cr = 0, lf = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      dash |= eq4(w[1 + k], 0x2D2D2D2Du) << (4 * k);
      cr |= eq4(w[1 + k], 0x0D0D0D0Du) << (4 * k);
      lf |= eq4(w[1 + k], 0x0A0A0A0Au) << (4 * k);
    }
    cr &= 0xFFFFu;
    any_cr |= cr != 0;
    const uint32_t pairs = cr & (lf >> 1);
    if (sep < 0) {
      const uint32_t hits = dash & (dash >> 1) & (dash >> 2) & 0xFFFFu;
      const uint32_t ball = __ballot_sync(0xffffffffu, hits != 0);
      if (ball) {
        const int fl = __ffs(ball) - 1;
        sep = __shfl_sync(0xffffffffu, c + (__ffs(hits) - 1), fl);
      }
    }
    if (sep < 0) pre += __popc(pairs);
    else {
      const long long nb = sep - c, na = sep + 3 - c;        // own positions < nb are before the separator, >= na are after it
      const uint32_t mb = nb <= 0 ? 0u : nb >= 16 ? 0xFFFFu : ((1u << nb) - 1u);
      const uint32_t ma = na <= 0 ? 0xFFFFu : na >= 16 ? 0u : (0xFFFFu & ~((1u << na) - 1u));
      pre += __popc(pairs & mb); post += __popc(pairs & ma);
    }
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) { pre += __shfl_xor_sync(0xffffffffu, pre, d); post += __shfl_xor_sync(0xffffffffu, post, d); }
  bad = __ballot_sync(0xffffffffu, bad) != 0; nonascii = __ballot_sync(0xffffffffu, nonascii) != 0;
  sigma = __ballot_sync(0xffffffffu, sigma) != 0; idot = __ballot_sync(0xffffffffu, idot) != 0; any_cr = __ballot_sync(0xffffffffu, any_cr) != 0;
  if (lane != 0) return;
  RawMeasure m{0, 0, 0, 0, 0, 0};
  if (!bad) {
    const uint8_t* p = raw + o0;
    const uint8_t* end = raw + o1;
    m.flags = 1u | (nonascii ? 4u : 0u) | (sigma ? 8u : 0u) | (idot ? 16u : 0u) | (any_cr ? 32u : 0u);
    const uint8_t* ba = sep >= 0 ? raw + sep + 3 : p;        // no separator: the whole text is the body (utils.py:107-109)
    const uint8_t* bb = end;
    uint32_t cut = 0;                                         // "\r\n" pairs inside the stripped margins
    for (;;) { if (ba >= bb) break; int k = ws_len_at(ba, bb); if (!k) break; if (ba[0] == '\r' && ba + 1 < bb && ba[1] == '\n') ++cut; ba += k; }
    for (;;) { if (ba >= bb) break; int k = ws_len_before(ba, bb); if (!k) break; if (bb[-1] == '\n' && bb - 2 >= ba && bb[-2] == '\r') ++cut; bb -= k; }
    uint32_t body_pairs = sep >= 0 ? post : pre;
    if (sep >= 0) { m.flags |= 2u; m.hdr_raw_len = (uint32_t)(sep - o0); m.hdr_len = m.hdr_raw_len - pre; }
    m.body_raw_begin = (uint32_t)(ba - p); m.body_raw_end = (uint32_t)(bb - p);
    m.body_len = ba < bb ? (uint32_t)(bb - ba) - (body_pairs - cut) : 0u;
    if (m.body_len > kMaxBodyBytes) atomicMax(summary + 1, (unsigned long long)i + 1ull);
  } else {
    atomicAdd(summary, 1ull);
  }
  out[i] = m;
  hdr_len[i] = m.hdr_len;
  body_len[i] = m.body_len;
}

// ---- warp copy of one span with universal-newline translation
// no '\r' in the file: a plain copy with 16-byte stores (the source is read 16-byte aligned and funnel-shifted into place)
__device__ __forceinline__ void warp_copy_plain(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t len, int lane) {
  uint32_t head = (uint32_t)((16u - (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u);
  if (head > len) head = len;
  if ((uint32_t)lane < head) dst[lane] = src[lane];
  const uint32_t nvec = (len - head) >> 4;
  const uint8_t* s0 = src + head;
  uint8_t* d0 = dst + head;
  const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(s0) & 15u), ws = sh >> 2, bs = (sh & 3u) * 8u;
  const uint8_t* sa = s0 - sh;
  for (uint32_t v = lane; v < nvec; v += 32) {
    const uint4 A = *reinterpret_cast<const uint4*>(sa + 16ull * v);
    uint4 o = A;
    if (sh) {
      const uint4 B = *reinterpret_cast<const uint4*>(sa + 16ull * v + 16);
      const uint32_t W[8] = {A.x, A.y, A.z, A.w, B.x, B.y, B.z, B.w};
      switch (ws) {
        case 0: o = make_uint4(__funnelshift_r(W[0], W[1], bs), __funnelshift_r(W[1], W[2], bs), __funnelshift_r(W[2], W[3], bs), __funnelshift_r(W[3], W[4], bs)); break;
        case 1: o = make_uint4(__funnelshift_r(W[1], W[2], bs), __funnelshift_r(W[2], W[3], bs), __funnelshift_r(W[3], W[4], bs), __funnelshift_r(W[4], W[5], bs)); break;
        case 2: o = make_uint4(__funnelshift_r(W[2], W[3], bs), __funnelshift_r(W[3], W[4], bs), __funnelshift_r(W[4], W[5], bs), __funnelshift_r(W[5], W[6], bs)); break;
        default: o = make_uint4(__funnelshift_r(W[3], W[4], bs), __funnelshift_r(W[4], W[5], bs), __funnelshift_r(W[5], W[6], bs), __funnelshift_r(W[6], W[7], bs)); break;
      }
    }
    *reinterpret_cast<uint4*>(d0 + 16ull * v) = o;
  }
  const uint32_t done = head + (nvec << 4);
  if (done + lane < len) dst[done + lane] = src[done + lane];
}
// with '\r': rows of 32 bytes, one per lane; a '\r' followed by '\n' is dropped, a lone one becomes '\n' (hard_end bounds the look-ahead)
__device__ __forceinline__ void warp_copy_translated(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t len, const uint8_t* hard_end, int lane) {
  uint32_t outpos = 0;
  for (uint32_t base = 0; base < len; base += 128) {
    uint32_t b[4], nx[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const uint32_t q = base + 32 * r + lane;
      b[r] = q < len ? src[q] : 0u;
      nx[r] = (q < len && src + q + 1 < hard_end) ? src[q + 1] : 0u;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const uint32_t q = base + 32 * r + lane;
      const bool in = q < len;
      const bool drop = in && b[r] == '\r' && nx[r] == '\n';
      const uint32_t dm = __ballot_sync(0xffffffffu, drop), im = __ballot_sync(0xffffffffu, in);
      if (in && !drop) dst[outpos + lane - __popc(dm & ((1u << lane) - 1u))] = b[r] == '\r' ? (uint8_t)'\n' : (uint8_t)b[r];
      outpos += __popc(im) - __popc(dm);
    }
  }
}

__global__ void __launch_bounds__(kIngestThreads) k_raw_write(const uint8_t* __restrict__ raw, const uint64_t* __restrict__ raw_off,
                                                               const uint64_t* __restrict__ raw_len, uint64_t n, const RawMeasure* __restrict__ ms, const uint64_t* __restrict__ hdr_off,
                                                               const uint64_t* __restrict__ body_off, uint8_t* __restrict__ hdr, uint8_t* __restrict__ body) {
  const uint64_t i = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const RawMeasure m = ms[i];
  if (!(m.flags & 1u)) return;
  const uint8_t* p = raw + raw_off[i];
  const uint8_t* end = raw_len ? p + raw_len[i] : raw + raw_off[i + 1];
  if (m.flags & 32u) {
    warp_copy_translated(hdr + hdr_off[i], p, m.hdr_raw_len, end, lane);
    warp_copy_translated(body + body_off[i], p + m.body_raw_begin, m.body_raw_end - m.body_raw_begin, end, lane);
  } else {
    warp_copy_plain(hdr + hdr_off[i], p, m.hdr_raw_len, lane);
    warp_copy_plain(body + body_off[i], p + m.body_raw_begin, m.body_raw_end - m.body_raw_begin, lane);
  }
}

__global__ void k_fix_fsb(const RawMeasure* __restrict__ ms, uint64_t n, uint32_t* __restrict__ fsb) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t f = ms[i].flags;
  uint32_t bits = ((f & 2u) ? 0u : FEI_REC_NO_SEPARATOR) | ((f & 4u) ? FEI_REC_NONASCII : 0u) | ((f & 8u) ? FEI_REC_HAS_SIGMA : 0u) | ((f & 16u) ? FEI_REC_HAS_IDOT : 0u);
  fsb[i] = (fsb[i] & 0x00FFFFFFu) | (bits << 24);
}

}  // namespace fei

using namespace fei;

// All n files must be valid records to be loaded; the call first reports validity so the host can drop the
// undecodable ones (and print the reference's message) and call again with the survivors.
static int load_raw_impl(fei_corpus* c, const fei_corpus_host* h, const uint8_t* raw, uint64_t raw_bytes_in, const uint64_t* raw_off,
                         const uint64_t* raw_len, uint8_t* valid_out) {
  if (!c || !h || !raw_off) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(check_load(h->n, h));
  const bool staged = h->n && !raw;                                     // raw == NULL: the text was put on the device by fei_corpus_stage_text
  // loads run on the copy stream: a batch can be uploaded / normalised / tiled into one handle while another handle is being
  // scanned on the compute stream (streaming e2e use); the staging buffers live in the handle (grow-only) because a
  // cudaFree in the middle of a pipeline synchronises the whole device
  cudaStream_t s = corpus_load_stream(c);
  uint64_t n = h->n;
  c->loaded = false;
  uint64_t raw_bytes = raw_len ? raw_bytes_in : (n ? raw_off[n] : 0);
  if (raw_len)
    for (uint64_t i = 0; i < n; ++i)
      if (raw_off[i] > raw_bytes || raw_len[i] > raw_bytes - raw_off[i]) { set_error("record %llu: span outside the %llu raw bytes", (unsigned long long)i, (unsigned long long)raw_bytes); return FEI_E_BADARG; }
  c->load_raw_bytes = raw_bytes;
  if (staged && (c->staged_text_bytes != raw_bytes || c->stage_raw.bytes < raw_bytes + 64)) {
    set_error("raw == NULL but the staged text (%llu bytes) is not the %llu bytes the offsets describe", (unsigned long long)c->staged_text_bytes, (unsigned long long)raw_bytes);
    return FEI_E_STATE;
  }
  FEI_TRY(corpus_load_events(c));
  DevBuf& d_raw = c->stage_raw; DevBuf& d_raw_off = c->stage_raw_off; DevBuf& d_ms = c->stage_ms; DevBuf& d_hlen = c->stage_hlen; DevBuf& d_blen = c->stage_blen;
  FEI_TRY(d_raw.ensure(raw_bytes + 64));
  FEI_TRY(d_ms.ensure((n ? n : 1) * sizeof(RawMeasure) + 16)); FEI_TRY(d_hlen.ensure((n ? n : 1) * 4)); FEI_TRY(d_blen.ensure((n ? n : 1) * 4));
  // The small host arrays go first: a second handle's multi-GB text copy may already sit in the copy engine's queue when this load
  // reaches its tail, and anything this load still had to upload then would wait behind it (and the next load behind this one).
  // meta columns + names come from the host (file-name grammar and listing order stay there)
  FEI_TRY(upload_meta(c, h, s));
  FEI_TRY(upload(d_raw_off, raw_off, (raw_len ? n : n + 1) * 8, 0, s));      // spans: n begins and n lengths; else n + 1 offsets
  if (raw_len) FEI_TRY(upload(c->stage_raw_len, raw_len, n * 8, 0, s));
  const uint64_t* d_len = raw_len ? c->stage_raw_len.as<uint64_t>() : nullptr;
  FEI_CUDA(cudaEventRecord(c->ev_load[0], s));
  // in pieces at fixed offsets: the host buffer may be page-locked block by block (the packer's arena: a copy must not straddle two
  // registrations), and a failed registration leaves one block pageable without slowing the others
  if (!staged) c->staged_text_bytes = ~0ull;                             // whatever was staged is overwritten now
  for (uint64_t o = 0; o < raw_bytes && !staged; o += kH2DPiece) {
    const uint64_t nb = raw_bytes - o < kH2DPiece ? raw_bytes - o : kH2DPiece;
    FEI_CUDA(cudaMemcpyAsync(d_raw.as<uint8_t>() + o, raw + o, nb, cudaMemcpyHostToDevice, s));
  }
  FEI_CUDA(cudaEventRecord(c->ev_load[1], s));
  FEI_CUDA(cudaMemsetAsync((uint8_t*)d_raw.p + raw_bytes, 0, 64, s));
  unsigned long long* d_summary = reinterpret_cast<unsigned long long*>(d_ms.as<uint8_t>() + (n ? n : 1) * sizeof(RawMeasure));
  FEI_CUDA(cudaMemsetAsync(d_summary, 0, 16, s));
  unsigned g = (unsigned)((n + 127) / 128);
  const unsigned gw = (unsigned)((n * 32 + kIngestThreads - 1) / kIngestThreads);       // one warp per file
  if (n) k_raw_measure<<<gw, kIngestThreads, 0, s>>>(d_raw.as<uint8_t>(), d_raw_off.as<uint64_t>(), d_len, n, d_ms.as<RawMeasure>(), d_hlen.as<uint32_t>(), d_blen.as<uint32_t>(), d_summary);
  // offsets of the normalised pieces (computed before the validity verdict is known: one host round trip instead of two)
  FEI_TRY(c->hdr_off.ensure((n + 1) * 8));
  DevBuf& body_off = c->stage_body_off; DevBuf& body = c->stage_body;
  FEI_TRY(body_off.ensure((n + 1) * 8));
  unsigned long long summary[2] = {0, 0};
  uint64_t hb = 0, bb = 0;
  FEI_TRY(queue_offsets(d_hlen.as<uint32_t>(), n, c->hdr_off.as<uint64_t>(), &hb, false, c->scan_tmp, s));
  FEI_TRY(queue_offsets(d_blen.as<uint32_t>(), n, body_off.as<uint64_t>(), &bb, false, c->scan_tmp, s));
  FEI_CUDA(cudaMemcpyAsync(summary, d_summary, 16, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  if (summary[0]) {
    if (valid_out) {
      std::vector<RawMeasure> ms(n);
      FEI_CUDA(cudaMemcpy(ms.data(), d_ms.p, n * sizeof(RawMeasure), cudaMemcpyDeviceToHost));
      for (uint64_t i = 0; i < n; ++i) valid_out[i] = ms[i].flags & 1u;
    }
    set_error("some files are not valid UTF-8 (see valid_out); drop them and load again");
    return FEI_E_BADARG;
  }
  if (valid_out && n) memset(valid_out, 1, n);
  if (summary[1]) { set_error("record %llu: body larger than 32 MiB is not supported", summary[1] - 1ull); return FEI_E_UNSUPPORTED; }
  c->n = n; c->global_base = h->global_base;
  c->hdr_bytes = hb; c->body_bytes = bb;
  FEI_TRY(c->hdr.ensure(hb + kBlobSlack)); FEI_TRY(body.ensure(bb + kBlobSlack));
  FEI_CUDA(cudaMemsetAsync((uint8_t*)c->hdr.p + hb, 0, kBlobSlack, s));
  FEI_CUDA(cudaMemsetAsync((uint8_t*)body.p + bb, 0, kBlobSlack, s));
  if (n) k_raw_write<<<gw, kIngestThreads, 0, s>>>(d_raw.as<uint8_t>(), d_raw_off.as<uint64_t>(), d_len, n, d_ms.as<RawMeasure>(), c->hdr_off.as<uint64_t>(), body_off.as<uint64_t>(),
                                       c->hdr.as<uint8_t>(), body.as<uint8_t>());
  if (n) k_fix_fsb<<<g, 128, 0, s>>>(d_ms.as<RawMeasure>(), n, c->fsb.as<uint32_t>());
  FEI_CUDA(cudaGetLastError());
  FEI_TRY(pack_canonical(c, body, body_off, s, false, c->ev_load[2]));
  c->load_timed = true;
  return FEI_OK;
}

/* Uploads a stretch of the file text ahead of fei_corpus_load_raw (which is then called with raw == NULL): the packer sends each
 * directory's bytes while it reads the next directory, so that the (pageable) copy is off the critical path.  total_bytes is the
 * size of the whole text; the stretches may come in any order and from any thread, one at a time per handle. */
extern "C" int fei_corpus_stage_text(fei_corpus* c, uint64_t total_bytes, const uint8_t* src, uint64_t offset, uint64_t bytes) {
  if (!c || (bytes && !src)) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_ready());
  if (offset > total_bytes || bytes > total_bytes - offset) { set_error("stretch outside the text"); return FEI_E_BADARG; }
  cudaStream_t s = corpus_load_stream(c);
  if (c->stage_raw.bytes < total_bytes + 64 || c->staged_text_bytes != total_bytes) {
    if (c->stage_raw.bytes < total_bytes + 64) { FEI_CUDA(cudaStreamSynchronize(s)); FEI_TRY(c->stage_raw.alloc(total_bytes + 64)); }
    c->staged_text_bytes = total_bytes;
  }
  for (uint64_t o = 0; o < bytes; o += kH2DPiece) {
    const uint64_t nb = bytes - o < kH2DPiece ? bytes - o : kH2DPiece;
    FEI_CUDA(cudaMemcpyAsync(c->stage_raw.as<uint8_t>() + offset + o, src + o, nb, cudaMemcpyHostToDevice, s));
  }
  return FEI_OK;
}

extern "C" int fei_corpus_load_raw(fei_corpus* c, const fei_corpus_host* h, const uint8_t* raw, const uint64_t* raw_off, uint8_t* valid_out) {
  return load_raw_impl(c, h, raw, 0, raw_off, nullptr, valid_out);
}
extern "C" int fei_corpus_load_raw_spans(fei_corpus* c, const fei_corpus_host* h, const uint8_t* raw, uint64_t raw_bytes, const uint64_t* begin,
                                         const uint64_t* len, uint8_t* valid_out) {
  if (h && h->n && (!begin || !len)) { set_error("null argument"); return FEI_E_BADARG; }
  static const uint64_t none = 0;
  return load_raw_impl(c, h, raw, raw_bytes, begin ? begin : &none, len ? len : &none, valid_out);
}

/* Device-side stage times of the last fei_corpus_load_raw on this handle (CUDA events on the load stream): out[0] = the text's
 * host-to-device copy, out[1] = everything after it (measure, offsets, normalise, tiling, header directory), out[2] = bytes of that
 * copy / out[0] in GB/s.  Waits for the load stream. */
extern "C" int fei_corpus_last_load_timing(fei_corpus* c, float* out) {
  if (!c || !out) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_ready());
  if (!c->load_timed) { set_error("no fei_corpus_load_raw has completed on this handle"); return FEI_E_BADARG; }
  FEI_CUDA(cudaEventSynchronize(c->ev_load[2]));
  FEI_CUDA(cudaEventElapsedTime(out + 0, c->ev_load[0], c->ev_load[1]));
  FEI_CUDA(cudaEventElapsedTime(out + 1, c->ev_load[1], c->ev_load[2]));
  out[2] = out[0] > 0 ? (float)(c->load_raw_bytes / (out[0] * 1e6)) : 0.f;
  return FEI_OK;
}
