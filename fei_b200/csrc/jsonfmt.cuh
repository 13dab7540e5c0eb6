// Canonical JSON of a Memorychain block's hashed fields, usable from host and device:
//   json.dumps({...ten fields...}, sort_keys=True)          (memdir_tools/memorychain.py:117-128)
// keys in sorted order, separators ", " and ": ", ensure_ascii=True, Python float repr (shortest digits that round-trip:
// Ryu, U. Adams, PLDI 2018; then float.__repr__'s layout rules, Python/pystrtod.c format_float_short mode 'r').
// The same source formats the column form on the GPU (chain.cu k_json_*) and on the host (chain_json.cpp).
#pragma once
#include <stdint.h>
#include <string.h>
#include "../../include/feiscan.h"
#include "sink.cuh"

namespace feijson {
using fei::put_bytes;
using fei::put_lit;

#define FEI_RYU_TABLE static const
namespace tab_host {
#include "ryu_tables.h"
}
#undef FEI_RYU_TABLE
#if defined(__CUDACC__)
#define FEI_RYU_TABLE __device__ const
namespace tab_dev {
#include "ryu_tables.h"
}
#undef FEI_RYU_TABLE
#endif

FEI_HD const uint64_t* pow5_inv(int i) {
#if defined(__CUDA_ARCH__)
  return tab_dev::kRyuPow5Inv[i];
#else
  return tab_host::kRyuPow5Inv[i];
#endif
}
FEI_HD const uint64_t* pow5(int i) {
#if defined(__CUDA_ARCH__)
  return tab_dev::kRyuPow5[i];
#else
  return tab_host::kRyuPow5[i];
#endif
}

// ---------------------------------------------------------------- Ryu: double -> shortest decimal (digits, exponent)
FEI_HD uint64_t umul128(uint64_t a, uint64_t b, uint64_t* hi) {
#if defined(__CUDA_ARCH__)
  *hi = __umul64hi(a, b);
  return a * b;
#else
  unsigned __int128 p = (unsigned __int128)a * b;
  *hi = (uint64_t)(p >> 64);
  return (uint64_t)p;
#endif
}
FEI_HD uint64_t shiftright128(uint64_t lo, uint64_t hi, uint32_t dist) { return (hi << (64 - dist)) | (lo >> dist); }   // 0 < dist < 64
FEI_HD uint64_t mul_shift64(uint64_t m, const uint64_t* mul, int j) {
  uint64_t high1, high0;
  const uint64_t low1 = umul128(m, mul[1], &high1);
  umul128(m, mul[0], &high0);
  const uint64_t sum = high0 + low1;
  if (sum < high0) ++high1;
  return shiftright128(sum, high1, (uint32_t)(j - 64));
}
FEI_HD uint32_t pow5_factor(uint64_t v) { uint32_t c = 0; while (v && v % 5 == 0) { v /= 5; ++c; } return c; }
FEI_HD bool multiple_of_pow5(uint64_t v, uint32_t p) { return pow5_factor(v) >= p; }
FEI_HD bool multiple_of_pow2(uint64_t v, uint32_t p) { return (v & ((1ull << p) - 1)) == 0; }
FEI_HD int pow5bits(int e) { return (int)(((uint32_t)e * 1217359u) >> 19) + 1; }
FEI_HD int log10_pow2(int e) { return (int)(((uint32_t)e * 78913u) >> 18); }
FEI_HD int log10_pow5(int e) { return (int)(((uint32_t)e * 732923u) >> 20); }

// value = mantissa * 10^exponent, mantissa without trailing zeros beyond what shortest round-trip leaves
FEI_HD_NI void ryu_d2d(uint64_t ieee_mantissa, uint32_t ieee_exponent, uint64_t* out_mantissa, int* out_exponent) {
  const int kMant = 52, kBias = 1023;
  int e2; uint64_t m2;
  if (ieee_exponent == 0) { e2 = 1 - kBias - kMant - 2; m2 = ieee_mantissa; }
  else { e2 = (int)ieee_exponent - kBias - kMant - 2; m2 = (1ull << kMant) | ieee_mantissa; }
  const bool accept_bounds = (m2 & 1) == 0;
  const uint64_t mv = 4 * m2;
  const uint32_t mm_shift = ieee_mantissa != 0 || ieee_exponent <= 1;
  uint64_t vr, vp, vm;
  int e10;
  bool vm_tz = false, vr_tz = false;
  if (e2 >= 0) {
    const uint32_t q = (uint32_t)log10_pow2(e2) - (e2 > 3);
    e10 = (int)q;
    const int k = 125 + pow5bits((int)q) - 1;
    const int i = -e2 + (int)q + k;
    const uint64_t* mul = pow5_inv((int)q);
    vr = mul_shift64(4 * m2, mul, i); vp = mul_shift64(4 * m2 + 2, mul, i); vm = mul_shift64(4 * m2 - 1 - mm_shift, mul, i);
    if (q <= 21) {
      const uint32_t mod5 = (uint32_t)(mv % 5);
      if (mod5 == 0) vr_tz = multiple_of_pow5(mv, q);
      else if (accept_bounds) vm_tz = multiple_of_pow5(mv - 1 - mm_shift, q);
      else vp -= multiple_of_pow5(mv + 2, q);
    }
  } else {
    const uint32_t q = (uint32_t)log10_pow5(-e2) - (-e2 > 1);
    e10 = (int)q + e2;
    const int i = -e2 - (int)q;
    const int k = pow5bits(i) - 125;
    const int j = (int)q - k;
    const uint64_t* mul = pow5(i);
    vr = mul_shift64(4 * m2, mul, j); vp = mul_shift64(4 * m2 + 2, mul, j); vm = mul_shift64(4 * m2 - 1 - mm_shift, mul, j);
    if (q <= 1) {
      vr_tz = true;
      if (accept_bounds) vm_tz = mm_shift == 1;
      else --vp;
    } else if (q < 63) {
      vr_tz = multiple_of_pow2(mv, q);
    }
  }
  int removed = 0;
  uint8_t last = 0;
  uint64_t output;
  if (vm_tz || vr_tz) {
    while (vp / 10 > vm / 10) {
      vm_tz &= vm % 10 == 0;
      vr_tz &= last == 0;
      last = (uint8_t)(vr % 10);
      vr /= 10; vp /= 10; vm /= 10; ++removed;
    }
    if (vm_tz) {
      while (vm % 10 == 0) {
        vr_tz &= last == 0;
        last = (uint8_t)(vr % 10);
        vr /= 10; vp /= 10; vm /= 10; ++removed;
      }
    }
    if (vr_tz && last == 5 && vr % 2 == 0) last = 4;                      // exactly halfway: round to even
    output = vr + ((vr == vm && (!accept_bounds || !vm_tz)) || last >= 5);
  } else {
    bool round_up = false;
    while (vp / 10 > vm / 10) {
      round_up = vr % 10 >= 5;
      vr /= 10; vp /= 10; vm /= 10; ++removed;
    }
    output = vr + (vr == vm || round_up);
  }
  *out_mantissa = output; *out_exponent = e10 + removed;
}

// float.__repr__: exponent form iff decpt <= -4 or decpt > 16; ".0" appended to integers; exponent of at least two digits.
// json.dumps spells the non-finite values NaN / Infinity / -Infinity (allow_nan=True).
template <class S> FEI_HD_NI void put_float(S& o, uint64_t bits) {
  const bool neg = (bits >> 63) != 0;
  const uint64_t mant = bits & ((1ull << 52) - 1);
  const uint32_t expo = (uint32_t)((bits >> 52) & 0x7FF);
  if (expo == 0x7FF) { if (mant) put_lit(o, "NaN"); else put_lit(o, neg ? "-Infinity" : "Infinity"); return; }
  if (expo == 0 && mant == 0) { put_lit(o, neg ? "-0.0" : "0.0"); return; }
  uint64_t m; int e;
  ryu_d2d(mant, expo, &m, &e);
  while (m % 10 == 0) { m /= 10; ++e; }                                       // the general path can leave trailing zeros (e.g. 1e23 family)
  char digits[20]; int nd = 0;
  { char tmp[20]; int k = 0; while (m) { tmp[k++] = (char)('0' + m % 10); m /= 10; } while (k) digits[nd++] = tmp[--k]; }
  const int decpt = nd + e;
  if (neg) o.put('-');
  if (decpt <= -4 || decpt > 16) {
    o.put((uint8_t)digits[0]);
    if (nd > 1) { o.put('.'); for (int k = 1; k < nd; ++k) o.put((uint8_t)digits[k]); }
    o.put('e');
    int x = decpt - 1;
    o.put(x < 0 ? '-' : '+');
    if (x < 0) x = -x;
    char eb[4]; int ne = 0;
    do { eb[ne++] = (char)('0' + x % 10); x /= 10; } while (x);
    if (ne < 2) eb[ne++] = '0';
    while (ne) o.put((uint8_t)eb[--ne]);
  } else if (decpt <= 0) {
    o.put('0'); o.put('.');
    for (int k = 0; k < -decpt; ++k) o.put('0');
    for (int k = 0; k < nd; ++k) o.put((uint8_t)digits[k]);
  } else if (decpt >= nd) {
    for (int k = 0; k < nd; ++k) o.put((uint8_t)digits[k]);
    for (int k = nd; k < decpt; ++k) o.put('0');
    o.put('.'); o.put('0');
  } else {
    for (int k = 0; k < decpt; ++k) o.put((uint8_t)digits[k]);
    o.put('.');
    for (int k = decpt; k < nd; ++k) o.put((uint8_t)digits[k]);
  }
}

template <class S> FEI_HD void put_int(S& o, int64_t v) {
  uint64_t u = v < 0 ? 0ull - (uint64_t)v : (uint64_t)v;
  if (v < 0) o.put('-');
  char tmp[20]; int k = 0;
  do { tmp[k++] = (char)('0' + u % 10); u /= 10; } while (u);
  while (k) o.put((uint8_t)tmp[--k]);
}

template <class S> FEI_HD void put_u4(S& o, uint32_t cp) {      // \uXXXX, lowercase hex like json.encoder
  const char* hx = "0123456789abcdef";
  o.put('\\'); o.put('u'); o.put((uint8_t)hx[(cp >> 12) & 15]); o.put((uint8_t)hx[(cp >> 8) & 15]); o.put((uint8_t)hx[(cp >> 4) & 15]); o.put((uint8_t)hx[cp & 15]);
}

// one ASCII character as py_encode_basestring_ascii writes it (put_json_string keeps its own copy of this switch: routing it
// through here changes the SASS of the chain kernels that instantiate it)
template <class S> FEI_HD void put_json_ascii(S& o, uint32_t c) {
  switch (c) {
    case '"': o.put('\\'); o.put('"'); break;
    case '\\': o.put('\\'); o.put('\\'); break;
    case '\n': o.put('\\'); o.put('n'); break;
    case '\r': o.put('\\'); o.put('r'); break;
    case '\t': o.put('\\'); o.put('t'); break;
    case '\b': o.put('\\'); o.put('b'); break;
    case '\f': o.put('\\'); o.put('f'); break;
    default: if (c >= 0x20 && c <= 0x7E) o.put((uint8_t)c); else put_u4(o, c);
  }
}

// py_encode_basestring_ascii: everything outside ' '..'~' plus '"' and '\\' is escaped.  Input is UTF-8 (lone surrogates
// arrive as 3-byte "surrogatepass" sequences).
template <class S> FEI_HD_NI void put_json_string(S& o, const uint8_t* s, uint64_t n) {
  o.put('"');
  uint64_t i = 0;
  while (i < n) {
    const uint32_t c = s[i];
    if (c < 0x80) {
      ++i;
      switch (c) {
        case '"': o.put('\\'); o.put('"'); break;
        case '\\': o.put('\\'); o.put('\\'); break;
        case '\n': o.put('\\'); o.put('n'); break;
        case '\r': o.put('\\'); o.put('r'); break;
        case '\t': o.put('\\'); o.put('t'); break;
        case '\b': o.put('\\'); o.put('b'); break;
        case '\f': o.put('\\'); o.put('f'); break;
        default: if (c >= 0x20 && c <= 0x7E) o.put((uint8_t)c); else put_u4(o, c);
      }
      continue;
    }
    uint32_t cp; int len;
    if ((c & 0xE0) == 0xC0) { cp = c & 0x1F; len = 2; }
    else if ((c & 0xF0) == 0xE0) { cp = c & 0x0F; len = 3; }
    else { cp = c & 0x07; len = 4; }
    for (int k = 1; k < len && i + k < n; ++k) cp = (cp << 6) | (s[i + k] & 0x3F);
    i += len;
    if (cp >= 0x10000) { const uint32_t v = cp - 0x10000; put_u4(o, 0xD800 | (v >> 10)); put_u4(o, 0xDC00 | (v & 0x3FF)); }
    else put_u4(o, cp);
  }
  o.put('"');
}

// Length of the well-formed UTF-8 sequence at s[0..n) (Python's strict decoder: no overlongs, surrogates or code points past
// U+10FFFF), or 0 when s[0] does not start one.
FEI_HD uint32_t utf8_seq_len(const uint8_t* s, uint64_t n) {
  const uint32_t c = s[0];
  if (c < 0x80) return 1;
  uint32_t len, lo = 0x80, hi = 0xBF;
  if (c >= 0xC2 && c <= 0xDF) len = 2;
  else if (c >= 0xE0 && c <= 0xEF) { len = 3; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
  else if (c >= 0xF0 && c <= 0xF4) { len = 4; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
  else return 0;
  if (n < len || s[1] < lo || s[1] > hi) return 0;
  for (uint32_t k = 2; k < len; ++k) if ((s[k] & 0xC0) != 0x80) return 0;
  return len;
}

// put_json_string of a file-system name as os.fsdecode gives it: bytes that are not part of well-formed UTF-8 become the lone
// surrogates U+DC80..U+DCFF (surrogateescape), which json.dumps writes as \udcXX.
template <class S> FEI_HD void put_json_fsname(S& o, const uint8_t* s, uint64_t n) {
  o.put('"');
  for (uint64_t i = 0; i < n;) {
    const uint32_t len = utf8_seq_len(s + i, n - i);
    if (len == 0) { put_u4(o, 0xDC00u | s[i]); ++i; continue; }
    if (len == 1) {                                                  // ASCII: the escapes of put_json_string
      put_json_ascii(o, s[i++]);
      continue;
    }
    uint32_t cp = s[i] & (0x7Fu >> len);
    for (uint32_t k = 1; k < len; ++k) cp = (cp << 6) | (s[i + k] & 0x3F);
    i += len;
    if (cp >= 0x10000) { const uint32_t v = cp - 0x10000; put_u4(o, 0xD800 | (v >> 10)); put_u4(o, 0xDC00 | (v & 0x3FF)); }
    else put_u4(o, cp);
  }
  o.put('"');
}

template <class S> FEI_HD_NI int put_value(S& o, const fei_json_col& c, uint64_t i) {
  const int tag = c.tag ? c.tag[i] : c.uniform_tag;
  switch (tag) {
    case FEI_J_NULL: put_lit(o, "null"); return 0;
    case FEI_J_TRUE: put_lit(o, "true"); return 0;
    case FEI_J_FALSE: put_lit(o, "false"); return 0;
    case FEI_J_INT: put_int(o, (int64_t)c.num[i]); return 0;
    case FEI_J_FLOAT: put_float(o, c.num[i]); return 0;
    case FEI_J_STR: put_json_string(o, c.str + c.str_off[i], c.str_off[i + 1] - c.str_off[i]); return 0;
    case FEI_J_BIGINT: put_bytes(o, c.str + c.str_off[i], c.str_off[i + 1] - c.str_off[i]); return 0;
    default: return -1;
  }
}

FEI_HD const char* key_name(int k) {
  switch (k) {
    case 0: return "difficulty"; case 1: return "index"; case 2: return "memory_id"; case 3: return "nonce"; case 4: return "previous_hash";
    case 5: return "proposer_node"; case 6: return "responsible_node"; case 7: return "solver_node"; case 8: return "task_state"; default: return "timestamp";
  }
}

template <class S> FEI_HD_NI int put_block(S& o, const fei_json_col* cols, uint64_t i) {
  o.put('{');
  for (int k = 0; k < FEI_CHAIN_NCOLS; ++k) {
    if (k) { o.put(','); o.put(' '); }
    o.put('"'); put_lit(o, key_name(k)); o.put('"'); o.put(':'); o.put(' ');
    if (put_value(o, cols[k], i) != 0) return -1;
  }
  o.put('}');
  return 0;
}

}  // namespace feijson
