// Python's str.strip() / str.isspace() whitespace set on UTF-8 bytes (shared by the scan and ingest kernels).
#pragma once
#include <stdint.h>

namespace fei {

// str.isspace(): U+0009-000D, 001C-001F, 0020, 0085, 00A0, 1680, 2000-200A, 2028, 2029, 202F, 205F, 3000
__device__ __forceinline__ int ws_len_at(const uint8_t* p, const uint8_t* end) {   // bytes of the whitespace char at p, or 0
  uint32_t c = p[0];
  if (c < 0x80) return ((c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x20)) ? 1 : 0;
  if (c == 0xC2) return (p + 1 < end && (p[1] == 0x85 || p[1] == 0xA0)) ? 2 : 0;
  if (p + 2 >= end) return 0;
  uint32_t c1 = p[1], c2 = p[2];
  if (c == 0xE1) return (c1 == 0x9A && c2 == 0x80) ? 3 : 0;
  if (c == 0xE2) {
    if (c1 == 0x80) return ((c2 >= 0x80 && c2 <= 0x8A) || c2 == 0xA8 || c2 == 0xA9 || c2 == 0xAF) ? 3 : 0;
    if (c1 == 0x81) return c2 == 0x9F ? 3 : 0;
    return 0;
  }
  if (c == 0xE3) return (c1 == 0x80 && c2 == 0x80) ? 3 : 0;
  return 0;
}
__device__ __forceinline__ int ws_len_before(const uint8_t* begin, const uint8_t* p) {   // whitespace char ending right before p
  if (p <= begin) return 0;
  uint32_t c = p[-1];
  if (c < 0x80) return ((c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x20)) ? 1 : 0;
  if ((c & 0xC0) != 0x80) return 0;
  if (p - begin >= 2 && p[-2] == 0xC2) return (c == 0x85 || c == 0xA0) ? 2 : 0;
  if (p - begin >= 3) { int n = ws_len_at(p - 3, p); return n == 3 ? 3 : 0; }
  return 0;
}
__device__ __forceinline__ void strip_span(const uint8_t*& a, const uint8_t*& b) {
  for (;;) { if (a >= b) return; int n = ws_len_at(a, b); if (!n) break; a += n; }
  for (;;) { if (a >= b) return; int n = ws_len_before(a, b); if (!n) break; b -= n; }
}

// One line of a header text, as utils.py:113-118 splits it: advances p past the line and its '\n'; false for a line without a
// colon, else the key (before the first colon) and the value, both stripped.
struct HeaderLine { const uint8_t *ka, *kb, *va, *vb; };
__device__ __forceinline__ bool next_header_line(const uint8_t*& p, const uint8_t* end, HeaderLine& l) {
  const uint8_t* eol = p; const uint8_t* colon = nullptr;
  while (eol < end && *eol != '\n') { if (!colon && *eol == ':') colon = eol; ++eol; }
  const uint8_t* line = p;
  p = eol + 1;
  if (!colon) return false;
  l = HeaderLine{line, colon, colon + 1, eol};
  strip_span(l.ka, l.kb); strip_span(l.va, l.vb);
  return true;
}

}  // namespace fei
