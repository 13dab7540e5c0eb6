// K1/K2: the Memdir scan kernels (sm_90a).
//
// Replaces the per-record loops of the reference:
//   search_memories -> _memory_matches_query -> _get_field_value / _compare_values
//       (memdir_tools/search.py:361-367, :244-335, :97-139, :141-242)
//   FilterManager.process_memories -> MemoryFilter.matches      (memdir_tools/filter.py:229-233, :67-109)
//   parse_memory_content header parsing                          (memdir_tools/utils.py:113-118)
//
// k_head_meta / k_head_parse : meta predicates (flags / date / folder / status) over the 20-byte meta columns, four
//          records per thread; records that still need a header or name field go to a work list and get one thread
//          each in k_head_parse, which applies the reference's dict semantics (header_lookup: a repeated key keeps its
//          last value, a case-insensitive field lookup takes the first matching spelling) to the record's header lines:
//          its header directory (hdir.cu: interned key + stripped value span per line; k_key_lut maps the corpus'
//          distinct keys to the program's fields once per scan), or, for headers the directory cannot address, its
//          text split / stripped like utils.py:113-118.  Every string condition is an output bit of a byte DFA (or of the field's
//          position automaton, head_nfa_run, for patterns the DFA refuses; k_head_meta<kFused, true, *> / k_head_parse<true, *>); the
//          program head (conditions + small automata + folder-set bitmaps) is staged into shared memory by a TMA bulk copy per CTA.
//          A folder set with a folder id of 64 or above is a bitmap in the head, read by the kFolderBits instances only.
//          Writes alive[i] = bitmask of queries whose non-content conditions all hold.
// k_body : one warp per group of 32 records in the warp-transposed body tiles (corpus.h): each
//          row is one contiguous coalesced request (ld.global.nc 16 B per lane); each lane walks
//          its own record through the multi-pattern DFA whose tables were staged into shared
//          memory with 1-D TMA bulk copies (cp.async.bulk + mbarrier).  Groups with no live
//          record are skipped without touching their bytes.  hits[i] = alive[i] & content bits.
//          In a list-building scan every warp stores its group's per-query hit counts (store_group_counts),
//          and the warp that completes a window of 4096 records adds them up and appends the window's hits
//          to the per-query ordered lists of 32-bit corpus-local indices (build_window_lists: decoupled
//          look-back over the windows); warps with no group left help write the last windows' lists (help_tail).
// k_body_nfa : content patterns too large for the DFA, stepped per code point as a bit-parallel position automaton (next to the
//          DFA of the program's other content patterns); same group loop, lists compacted after it.
// k_count / k_scan_blocks / k_emit : order-preserving compaction of hits[] into per-query lists
//          (warp ballots + popc prefix, block offsets from a scan): corpus-local 32-bit indices for the
//          single-pattern kernels and header-only programs, 64-bit global ones for gathered multi-GPU masks.
#include "corpus.h"
#include "../../include/feiscan_prog.h"
#include "pyws.cuh"
#include "datefmt.cuh"
#include "sink.cuh"
#include <string.h>
#include <stdlib.h>
#include <vector>
#include <algorithm>

namespace fei {

// ---------------------------------------------------------------- short automaton runs (header fields, names, flags)
// Where an automaton's tables live.  SmemTables: the shared-memory copy of the program head (stage_prog_head), 32-bit shared
// addresses and ld.shared (a generic-pointer loop costs 29 instructions per byte in SASS, this one about 8).  GlobalTables: the
// program blob in global memory.
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) { uint32_t r; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(r) : "r"(a)); return r; }
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) { uint32_t r; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(r) : "r"(a)); return r; }
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) { uint32_t r; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(a)); return r; }
struct SmemTables {
  using Addr = uint32_t;
  static __device__ __forceinline__ Addr at(const uint8_t* blob) { return (uint32_t)__cvta_generic_to_shared(blob); }
  static __device__ __forceinline__ uint32_t u8(Addr a) { return lds_u8(a); }
  static __device__ __forceinline__ uint32_t u16(Addr a) { return lds_u16(a); }
  static __device__ __forceinline__ uint32_t u32(Addr a) { return lds_u32(a); }
};
struct GlobalTables {
  using Addr = const uint8_t*;
  static __device__ __forceinline__ Addr at(const uint8_t* blob) { return blob; }
  static __device__ __forceinline__ uint32_t u8(Addr a) { return *a; }
  static __device__ __forceinline__ uint32_t u16(Addr a) { return *reinterpret_cast<const uint16_t*>(a); }
  static __device__ __forceinline__ uint32_t u32(Addr a) { return *reinterpret_cast<const uint32_t*>(a); }
};

// One automaton run.  out[] has an entry (0) for every non-accepting state too (feiscan_prog.h), so there is no branch around
// the lookup and the byte loads of an unrolled group issue ahead of the table walk.
template <class M> struct Dfa {
  typename M::Addr trans, out, endout, cls;
  uint32_t stride2, empty_acc, s, acc;
  bool direct;
  __device__ __forceinline__ Dfa(const uint8_t* blob, uint32_t off) {
    const fei_prog_dfa* d = reinterpret_cast<const fei_prog_dfa*>(blob + off);
    const typename M::Addr base = M::at(blob);
    trans = base + d->off_trans; out = base + d->off_out; endout = base + d->off_endout; cls = base + d->off_cls;
    stride2 = d->row_stride * 2u; empty_acc = d->empty_acc; direct = d->n_cols == 256;
    s = d->start; acc = M::u32(out + 4u * s);
  }
  __device__ __forceinline__ void step(uint32_t b) {
    const uint32_t col = direct ? b : M::u8(cls + b);
    s = M::u16(trans + s * stride2 + col * 2u);
    acc |= M::u32(out + 4u * s);
  }
  __device__ __forceinline__ uint32_t result() const { return acc | M::u32(endout + 4u * s); }
  // a byte span.  (Fetching it as aligned 4- or 16-byte words was measured slower on the header workloads: per-lane skip /
  // tail predicates diverge.)
  __device__ __forceinline__ uint32_t span(const uint8_t* p, uint32_t len) {
    if (len == 0) return empty_acc;
    uint32_t i = 0;
    for (; i + 4 <= len; i += 4) {
      const uint32_t b0 = p[i], b1 = p[i + 1], b2 = p[i + 2], b3 = p[i + 3];
      step(b0); step(b1); step(b2); step(b3);
    }
    for (; i < len; ++i) step(p[i]);
    return result();
  }
  // up to 8 bytes held in a register (the flags string of a record: flags8)
  __device__ __forceinline__ uint32_t u64(unsigned long long bytes, uint32_t len) {
    if (len == 0) return empty_acc;
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) if (k < len) step((uint32_t)(bytes >> (8 * k)) & 0xFFu);
    return result();
  }
  // a column value: unit k (16 bytes) of the value at base + k * plane_stride (hdir.cu), LDG.128 per unit
  __device__ __forceinline__ uint32_t units(const uint8_t* base, uint64_t plane_stride, uint32_t len) {
    if (len == 0) return empty_acc;
    for (uint32_t k = 0; k * 16 < len; ++k) {
      const uint4 c = *reinterpret_cast<const uint4*>(base + k * plane_stride);
      const uint32_t w[4] = {c.x, c.y, c.z, c.w};
      const uint32_t nb = len - k * 16;
#pragma unroll
      for (uint32_t j = 0; j < 16; ++j) if (j < nb) step((w[j >> 2] >> (8 * (j & 3))) & 0xFFu);
    }
    return result();
  }
};
// `run(dfa)` with the tables where they are: `in_smem` is uniform for the grid (stage_prog_head staged the head for every CTA or for none)
template <class Run> __device__ __forceinline__ uint32_t dfa_run_at(const uint8_t* blob, uint32_t off, bool in_smem, Run run) {
  if (in_smem) return run(Dfa<SmemTables>(blob, off));
  return run(Dfa<GlobalTables>(blob, off));
}
__device__ __forceinline__ uint32_t dfa_run_at(const uint8_t* blob, uint32_t off, bool in_smem, const uint8_t* p, uint32_t len) {
  return dfa_run_at(blob, off, in_smem, [&](auto d) { return d.span(p, len); });
}

// ---------------------------------------------------------------- position automaton step (content and head fields)
// One code point of a fei_prog_nfa (feiscan_prog.h) over a W-word bit vector of NFA positions:
//     D' = (((D << 1) & SHIFT) | (D & SELF) | OR_g [(D & src_g) && ctx ok] dst_g) & B[class]
// The tables are read through generic pointers: k_body_nfa's staged shared-memory copy, or a head field's section in the staged
// program head or in the global program.
struct NfaTables {
  const uint16_t* ascii; const uint32_t* range_lo; const uint16_t* range_ck; const uint32_t* cls_b;
  const uint32_t* masks; const uint32_t* follow; const uint32_t* accept;
  uint32_t n_ranges, n_follow, n_accept;
  // the tables of section nd, whose bytes [off_ascii, off_ascii + table_bytes) start at tab
  __device__ __forceinline__ NfaTables(const fei_prog_nfa* nd, const uint8_t* tab) {
    ascii = reinterpret_cast<const uint16_t*>(tab);
    range_lo = reinterpret_cast<const uint32_t*>(tab + (nd->off_range_lo - nd->off_ascii));
    range_ck = reinterpret_cast<const uint16_t*>(tab + (nd->off_range_ck - nd->off_ascii));
    cls_b = reinterpret_cast<const uint32_t*>(tab + (nd->off_cls_b - nd->off_ascii));
    masks = reinterpret_cast<const uint32_t*>(tab + (nd->off_masks - nd->off_ascii));
    follow = reinterpret_cast<const uint32_t*>(tab + (nd->off_follow - nd->off_ascii));
    accept = reinterpret_cast<const uint32_t*>(tab + (nd->off_accept - nd->off_ascii));
    n_ranges = nd->n_ranges; n_follow = nd->n_follow; n_accept = nd->n_accept;
  }
  __device__ __forceinline__ uint32_t class_kind(uint32_t cp) const {     // class | kind << 8
    if (cp < 0x80u) return ascii[cp];
    uint32_t lo = 0, hi = n_ranges - 1;
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) >> 1;
      if (range_lo[mid] <= cp) lo = mid; else hi = mid - 1;
    }
    return range_ck[lo];
  }
};

// Counter positions of a content automaton (feiscan_prog.h fei_prog_nfa_ctr), all in registers: position, bound and age of
// each.  Empty for the automata without counters.
template <bool kCtr> struct NfaCounters {};
template <> struct NfaCounters<true> {
  uint32_t n, pos[FEI_NFA_MAX_COUNTERS], bound[FEI_NFA_MAX_COUNTERS], age[FEI_NFA_MAX_COUNTERS];
};

template <int W, bool kCtr = false>
struct Nfa {
  uint32_t d[W];                     // active positions
  uint32_t prev;                     // context kind of the last code point (0: none yet)
  uint32_t cp, need;                 // UTF-8 decoder: code point so far, continuation bytes still to come
  uint32_t acc;                      // output bits of the accepts met so far (end-only accepts not included)
  NfaCounters<kCtr> ctr;
  // kCtr: the counter table (uint32[n][2]: position, bound), read once into registers
  __device__ __forceinline__ void load_counters(const uint32_t* tab, uint32_t n) {
    ctr.n = n;
#pragma unroll
    for (int i = 0; i < FEI_NFA_MAX_COUNTERS; ++i) {
      ctr.pos[i] = i < (int)n ? tab[2 * i] : 0u;
      ctr.bound[i] = i < (int)n ? tab[2 * i + 1] : 0u;
    }
  }
  __device__ __forceinline__ void reset(const NfaTables& t) {
#pragma unroll
    for (int k = 0; k < W; ++k) d[k] = t.masks[2 * W + k];
    prev = 0; cp = 0; need = 0; acc = 0;
    if constexpr (kCtr) {
#pragma unroll
      for (int i = 0; i < FEI_NFA_MAX_COUNTERS; ++i) ctr.age[i] = 0;
    }
  }
  // kCtr: n = Follow(D, ctx) gets the counter positions that continue their run, D[P] && age_P < k, and every age steps
  // (1 on entry).  A position's word is a run-time value: d[] and n[] are read and written with unrolled compares, so they
  // stay in registers.
  __device__ __forceinline__ void count(uint32_t* n) {
    uint32_t keep[W];
#pragma unroll
    for (int k = 0; k < W; ++k) keep[k] = 0;
#pragma unroll
    for (int i = 0; i < FEI_NFA_MAX_COUNTERS; ++i) {
      if (i < (int)ctr.n) {
        const uint32_t w = ctr.pos[i] >> 5, m = 1u << (ctr.pos[i] & 31u);
        uint32_t fw = 0, dw = 0;
#pragma unroll
        for (int k = 0; k < W; ++k) if (k == (int)w) { fw = n[k]; dw = d[k]; }
        const uint32_t cont = (dw & m) && ctr.age[i] < ctr.bound[i] ? m : 0u;
        ctr.age[i] = (fw & m) ? 1u : ctr.age[i] + 1u;
#pragma unroll
        for (int k = 0; k < W; ++k) if (k == (int)w) keep[k] |= cont;
      }
    }
#pragma unroll
    for (int k = 0; k < W; ++k) n[k] |= keep[k];
  }
  __device__ __forceinline__ bool any(const uint32_t* src) const {
    uint32_t x = 0;
#pragma unroll
    for (int k = 0; k < W; ++k) x |= d[k] & src[k];
    return x != 0;
  }
  __device__ __forceinline__ uint32_t accepts(const NfaTables& t, uint32_t ctx, bool at_end) const {
    uint32_t m = 0;
    for (uint32_t g = 0; g < t.n_accept; ++g) {
      const uint32_t* r = t.accept + g * (W + 2);
      const uint32_t info = r[W + 1];
      if ((r[W] & ctx) && (at_end || !(info >> 8)) && any(r)) m |= 1u << (info & 31u);
    }
    return m;
  }
  __device__ __forceinline__ void step_cp(const NfaTables& t, uint32_t c) {
    const uint32_t ck = t.class_kind(c);
    const uint32_t kind = ck >> 8;
    const uint32_t ctx = 1u << (prev * 5u + kind);
    acc |= accepts(t, ctx, false);
    uint32_t n[W];
#pragma unroll
    for (int k = 0; k < W; ++k) {
      const uint32_t sh = k ? __funnelshift_l(d[k - 1], d[k], 1) : d[0] << 1;
      n[k] = (sh & t.masks[k]) | (d[k] & t.masks[W + k]);
    }
    for (uint32_t g = 0; g < t.n_follow; ++g) {
      const uint32_t* r = t.follow + g * (2 * W + 1);
      if ((r[2 * W] & ctx) && any(r)) {
#pragma unroll
        for (int k = 0; k < W; ++k) n[k] |= r[W + k];
      }
    }
    if constexpr (kCtr) count(n);
    const uint32_t* b = t.cls_b + (ck & 0xFFu) * W;
#pragma unroll
    for (int k = 0; k < W; ++k) d[k] = n[k] & b[k];
    prev = kind;
  }
  // one byte of UTF-8 text
  __device__ __forceinline__ void byte(const NfaTables& t, uint32_t b) {
    if (b < 0x80u) { step_cp(t, b); return; }                        // ASCII: one byte, one code point
    if (b >= 0xC0u) { need = b >= 0xF0u ? 3u : b >= 0xE0u ? 2u : 1u; cp = b & (0x3Fu >> need); return; }
    cp = (cp << 6) | (b & 0x3Fu);
    if (--need == 0) step_cp(t, cp);
  }
  __device__ __forceinline__ uint32_t finish(const NfaTables& t) const { return acc | accepts(t, 1u << (prev * 5u), true); }
};

// A head field's position automaton (the section at `off` of the program at `prog`, staged or global) over one value of len
// bytes: byte j at p[(j >> 4) * stride + (j & 15)] -- a span of header text or a formatted buffer with stride 16, value-column
// units (Dfa::units) with the plane stride -- or, with p == nullptr, byte j of `reg` (flags8).  Out of line: the head kernels'
// DFA paths do not pay its registers, and one copy serves every caller.
template <int W>
__device__ __forceinline__ uint32_t nfa_run(const NfaTables& t, const uint8_t* p, uint64_t stride, uint32_t len, unsigned long long reg) {
  Nfa<W> nfa;
  nfa.reset(t);
  for (uint32_t j = 0; j < len; ++j) nfa.byte(t, p ? p[(j >> 4) * stride + (j & 15u)] : (uint32_t)(reg >> (8 * j)) & 0xFFu);
  return nfa.finish(t);
}
__device__ __noinline__ uint32_t head_nfa_run(const uint8_t* prog, uint32_t off, const uint8_t* p, uint64_t stride, uint32_t len,
                                              unsigned long long reg) {
  const fei_prog_nfa* nd = reinterpret_cast<const fei_prog_nfa*>(prog + off);
  const NfaTables t(nd, prog + nd->off_ascii);
  switch (nd->n_words) {                                               // check_prog: 1, 2, 4 or 8
    case 1: return nfa_run<1>(t, p, stride, len, reg);
    case 2: return nfa_run<2>(t, p, stride, len, reg);
    case 4: return nfa_run<4>(t, p, stride, len, reg);
    default: return nfa_run<8>(t, p, stride, len, reg);
  }
}
// A head field's verdict over one value: its DFA's bits, run(dfa), and its position automaton's over the same bytes (either
// part may be absent).  Only kHeadNfa instances call it; the others run the DFA alone, as before there were head automata.
template <class Run>
__device__ __forceinline__ uint32_t field_run(const uint8_t* prog, bool in_smem, uint32_t off_dfa, uint32_t off_nfa, Run run,
                                              const uint8_t* p, uint64_t stride, uint32_t len) {
  return (off_dfa ? dfa_run_at(prog, off_dfa, in_smem, run) : 0u) | (off_nfa ? head_nfa_run(prog, off_nfa, p, stride, len, 0) : 0u);
}
// fei_prog_head_nfa entry k (0 flags, 1 + name field)
__device__ __forceinline__ uint32_t head_nfa_off(const uint8_t* prog, const fei_prog_hdr* ph, int k) {
  return ph->off_head_nfa ? reinterpret_cast<const uint32_t*>(prog + ph->off_head_nfa)[k] : 0u;
}

// ---------------------------------------------------------------- header field lookup
// A record's header lines, in order, from its directory entries (hdir.cu).  A key is its dictionary slot.
struct DirLines {
  using Key = uint32_t;
  const uint2* ent; uint32_t n_ent; const uint32_t* key_lut;
  uint32_t j, key, val_off, val_len;
  __device__ __forceinline__ bool next() {
    if (j == n_ent) return false;
    const uint2 e = ent[j++];
    key = e.x & 0xFFFFu; val_off = e.y; val_len = e.x >> 16;
    return true;
  }
  __device__ __forceinline__ uint32_t key_mask() const { return key_lut[key]; }
  __device__ __forceinline__ bool same_key(Key k) const { return k == key; }
  __device__ __forceinline__ bool assigned_later() const {
    for (uint32_t k = j; k < n_ent; ++k) if ((ent[k].x & 0xFFFFu) == key) return true;
    return false;
  }
};
// The same lines split from the record's header text (next_header_line), for headers the directory cannot address.  A key is
// its span (offset, length) in the text; the key automaton gives its slots.
struct TextLines {
  using Key = uint2;
  const uint8_t *h, *p, *end;
  const uint8_t* prog; uint32_t key_dfa; bool in_smem;
  Key key; uint32_t val_off, val_len;
  __device__ __forceinline__ bool next() {
    for (HeaderLine l; p < end;)
      if (next_header_line(p, end, l)) {
        key = make_uint2((uint32_t)(l.ka - h), (uint32_t)(l.kb - l.ka)); val_off = (uint32_t)(l.va - h); val_len = (uint32_t)(l.vb - l.va);
        return true;
      }
    return false;
  }
  __device__ __forceinline__ uint32_t key_mask() const { return dfa_run_at(prog, key_dfa, in_smem, h + key.x, key.y); }
  __device__ __forceinline__ bool same_key(Key k) const {
    bool same = k.y == key.y;
    for (uint32_t b = 0; same && b < k.y; ++b) same = h[k.x + b] == h[key.x + b];
    return same;
  }
  __device__ __forceinline__ bool assigned_later() const {
    HeaderLine l;
    for (const uint8_t* q = p; q < end;)
      if (next_header_line(q, end, l) && same_key(make_uint2((uint32_t)(l.ka - h), (uint32_t)(l.kb - l.ka)))) return true;
    return false;
  }
};

// The reference's headers dict (filled line by line by utils.py:113-118, read by search.py:121-132 and utils.py:333-336), asked
// for program slots 0 .. kSlots-1 over one record's header lines, by the slot's mode(s):
//   0: the first key whose lower() equals the field fixes the spelling; the value is that of the last line with exactly that spelling;
//   1: exact key, the last line wins;
//   2: every value of the dict: each line whose key no later line assigns again goes to any(s, off, len).
// Returns the mode-0/1 slots found; their values are at val_off[s] / val_len[s] (offsets into the record's header text).  Both
// line sources give the same answers: k_hdir checks every interned key byte for byte against its slot's spelling.
template <uint32_t kSlots, class Lines, class Mode, class Any>
__device__ __forceinline__ uint32_t header_lookup(Lines lines, Mode mode, uint32_t* val_off, uint32_t* val_len, Any any) {
  typename Lines::Key first_key[kSlots];
  uint32_t found = 0, have_first = 0;
  while (lines.next()) {
    for (uint32_t km = lines.key_mask() & (kSlots < 32 ? (1u << kSlots) - 1u : ~0u); km; km &= km - 1) {
      const int s = kSlots == 1 ? 0 : __ffs(km) - 1;
      const uint32_t m = mode(s);
      if (m == 2) { if (!lines.assigned_later()) any(s, lines.val_off, lines.val_len); continue; }
      if (m == 0) {
        if (!(have_first >> s & 1u)) { have_first |= 1u << s; first_key[s] = lines.key; }
        else if (!lines.same_key(first_key[s])) continue;      // a different spelling of the key: not the dict entry we read
      }
      val_off[s] = lines.val_off; val_len[s] = lines.val_len;   // repeated key: last value wins (dict assignment)
      found |= 1u << s;
    }
  }
  return found;
}
__device__ __forceinline__ void no_values(int, uint32_t, uint32_t) {}   // `any` of a lookup without mode-2 slots

// ---------------------------------------------------------------- head kernel
struct HeadArgs {
  const uint8_t* prog;         // device copy of the program blob
  const uint8_t* hdr; const uint64_t* hdr_off;
  const uint8_t* name; const uint64_t* name_off; const uint16_t* name_spans;
  const int64_t* wall; const uint64_t* flags8; const uint32_t* fsb;
  uint64_t n;
  uint32_t* alive;
  const uint2* hdir; const uint64_t* hdir_off;     // header directory (hdir.cu)
  const uint32_t* key_lut;                         // dictionary slot of a header key -> mask of the program's slots it names (k_key_lut)
  bool prog_in_smem;                               // set by the kernels after stage_prog_head
  const int8_t* slot_col;                          // per program slot: value column to read (k_slot_cols), -1 walk the directory, -2 no record has the field
  const uint16_t* col_len; const uint8_t* col_planes;   // header value columns (hdir.cu)
  const int64_t* ts;                               // filename timestamps (metadata "timestamp")
  const uint8_t* aux[FEI_MAX_AUX];                 // host-computed per-record verdict bytes (fei_corpus_set_aux)
};

constexpr int kHeadThreads = 256;

__device__ __forceinline__ bool cmp_i64(int64_t v, int64_t o, uint32_t op) {
  switch (op) {
    case FEI_CMP_GT: return v > o; case FEI_CMP_LT: return v < o;
    case FEI_CMP_GE: return v >= o; case FEI_CMP_LE: return v <= o;
    case FEI_CMP_EQ: return v == o; default: return v != o;
  }
}
// kFolderBits: some folder set of the program is a bitmap (folder ids of 64 and above).  Only the instances of the head kernels for
// such programs read it; the others keep the set64 test alone, which costs the unrolled meta loop no registers.
template <bool kFolderBits>
__device__ __forceinline__ bool eval_meta_cond(const HeadArgs& a, uint64_t rec, const fei_prog_cond& cd, uint32_t flags_acc, int64_t wall, uint32_t fsb) {
  switch (cd.kind) {
    case FEI_C_RECBITS: {
      // selected, not indexed: a dynamic index into the by-value kernel argument makes ptxas copy the whole struct to local memory
      const uint32_t k = cd.ref & (FEI_MAX_AUX - 1);
      static_assert(FEI_MAX_AUX == 4, "aux column select below");
      const uint8_t* col = k == 0 ? a.aux[0] : k == 1 ? a.aux[1] : k == 2 ? a.aux[2] : a.aux[3];
      return (col[rec] != 0) != (cd.negate != 0);
    }
    case FEI_C_TS_CMP: return cmp_i64(a.ts[rec], cd.i64, cd.cmp_op);
    case FEI_C_CONST: return cd.bit != 0;
    case FEI_C_FLAGS: return ((flags_acc >> cd.bit) & 1u) != cd.negate;
    case FEI_C_DATE_CMP: {
      int64_t v = wall * 1000000ll, o = cd.i64;
      switch (cd.cmp_op) {
        case FEI_CMP_GT: return v > o; case FEI_CMP_LT: return v < o;
        case FEI_CMP_GE: return v >= o; case FEI_CMP_LE: return v <= o;
        case FEI_CMP_EQ: return v == o; default: return v != o;
      }
    }
    case FEI_C_FOLDER_SET:
      if constexpr (kFolderBits) {                             // set64, or the program's bitmap of the set (fei_prog_cond.off_set_words)
        const uint32_t fid = fsb & 0xFFFFu;
        if (!cd.off_set_words) return fid < 64u && (cd.set64 >> fid & 1ull) != 0;
        const uint32_t* words = reinterpret_cast<const uint32_t*>(a.prog + cd.off_set_words);     // staged with the head (check_prog)
        return fid < 32u * cd.n_set_words && (words[fid >> 5] >> (fid & 31u) & 1u) != 0;
      } else {
        return (cd.set64 >> (fsb & 0xFFFFu) & 1ull) != 0;
      }
    case FEI_C_STATUS_SET: return (cd.set64 >> ((fsb >> 16) & 0xFFu) & 1ull) != 0;
    default: return true;                                      // slot / name / body: decided later
  }
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count);
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes);
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar);
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity);

// str(int) of a non-negative integer; returns the length
__device__ __forceinline__ uint32_t format_u64(unsigned long long v, uint8_t* out) {
  uint8_t tmp[20]; int n = 0;
  do { tmp[n++] = (uint8_t)('0' + v % 10); v /= 10; } while (v);
  for (int i = 0; i < n; ++i) out[i] = tmp[n - 1 - i];
  return (uint32_t)n;
}

// File-name fields and the strings Python would format from the metadata (rare predicates): kept out of line so that their
// buffers and divisions do not cost the common header path registers.  (Arguments by value: a reference to the kernel's by-value
// HeadArgs, like a dynamic index into one of its arrays, makes ptxas copy the whole struct to local memory -- that, via the aux
// column array, more than doubled the time of the cfg2 head pass.)
struct NameArgs { const uint8_t* prog; const uint8_t* name; const uint64_t* name_off; const uint16_t* name_spans; const int64_t* ts; const int64_t* wall; bool prog_in_smem; };
template <bool kHeadNfa>
__device__ __noinline__ void eval_name_fields(const NameArgs a, const fei_prog_hdr* ph, uint64_t rec, uint32_t* name_acc) {
  if constexpr (!kHeadNfa) {
    for (int k = 0; k < 3; ++k) {
      if (!ph->off_name_dfa[k]) continue;
      const uint8_t* nb = a.name + a.name_off[rec];
      uint32_t nl = (uint32_t)(a.name_off[rec + 1] - a.name_off[rec]);
      if (k > 0) { const uint16_t* sp = a.name_spans + 4 * rec + 2 * (k - 1); nb += sp[0]; nl = sp[1]; }
      name_acc[k] = dfa_run_at(a.prog, ph->off_name_dfa[k], a.prog_in_smem, nb, nl);
    }
    // str(timestamp) and str(datetime.fromtimestamp(ts))
    if (ph->off_meta_dfa[0]) { uint8_t buf[24]; const uint32_t nl = format_u64(a.ts[rec] < 0 ? 0ull : (unsigned long long)a.ts[rec], buf); name_acc[3] = dfa_run_at(a.prog, ph->off_meta_dfa[0], a.prog_in_smem, buf, nl); }
    if (ph->off_meta_dfa[1]) { uint8_t buf[24]; const uint32_t nl = format_datetime(a.wall[rec], buf); name_acc[4] = dfa_run_at(a.prog, ph->off_meta_dfa[1], a.prog_in_smem, buf, nl); }
  } else {                                                     // the same fields, each through its DFA and / or position automaton
    for (int k = 0; k < FEI_NAME_FIELDS; ++k) {
      const uint32_t off_dfa = k < 3 ? ph->off_name_dfa[k] : ph->off_meta_dfa[k - 3], off_nfa = head_nfa_off(a.prog, ph, 1 + k);
      if (!off_dfa && !off_nfa) continue;
      uint8_t buf[24];
      const uint8_t* nb = buf;
      uint32_t nl;
      if (k == 3) nl = format_u64(a.ts[rec] < 0 ? 0ull : (unsigned long long)a.ts[rec], buf);
      else if (k == 4) nl = format_datetime(a.wall[rec], buf);
      else {
        nb = a.name + a.name_off[rec]; nl = (uint32_t)(a.name_off[rec + 1] - a.name_off[rec]);
        if (k > 0) { const uint16_t* sp = a.name_spans + 4 * rec + 2 * (k - 1); nb += sp[0]; nl = sp[1]; }
      }
      name_acc[k] = field_run(a.prog, a.prog_in_smem, off_dfa, off_nfa, [&](auto d) { return d.span(nb, nl); }, nb, 16, nl);
    }
  }
}

// Phase 2 for one record: header fields (if `parse`), name fields, evaluation of the queries left in `pre`.  kHeadNfa: the
// program has head position automata (a slot may then have no DFA); kFolderBits: see eval_meta_cond.
template <bool kHeadNfa, bool kFolderBits>
__device__ void head_finish(const HeadArgs& a, uint64_t rec, uint32_t pre, uint32_t flags_acc, bool parse) {
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const fei_prog_cond* conds = reinterpret_cast<const fei_prog_cond*>(a.prog + ph->off_conds);
  const fei_prog_query* queries = reinterpret_cast<const fei_prog_query*>(a.prog + ph->off_queries);
  const fei_prog_slot* slots = reinterpret_cast<const fei_prog_slot*>(a.prog + ph->off_slots);
  const uint32_t nslots = ph->n_slots;
  uint32_t slot_acc[FEI_MAX_SLOTS];
  uint32_t present = 0;
  if (parse) {
    // fields that have a value column: the record's value sits at plane k, offset 16 * rec -- consecutive threads read
    // consecutive units, and neither the directory nor the header text of the record is touched
    bool walk = false;
    for (uint32_t s = 0; s < nslots; ++s) {
      const int col = a.slot_col[s];
      if (col == -2) continue;                                 // no record of this corpus has the field
      if (col < 0) { walk = true; break; }
      const uint32_t len = a.col_len[(uint64_t)col * a.n + rec];
      if (len == kColAbsent) continue;
      if (len == kColWalk) { walk = true; break; }
      const uint8_t* unit = a.col_planes + (uint64_t)col * kColUnits * a.n * 16 + rec * 16;
      if constexpr (kHeadNfa)
        slot_acc[s] = field_run(a.prog, a.prog_in_smem, slots[s].off_val_dfa, slots[s].off_val_nfa, [&](auto d) { return d.units(unit, a.n * 16, len); },
                                unit, a.n * 16, len);
      else slot_acc[s] = dfa_run_at(a.prog, slots[s].off_val_dfa, a.prog_in_smem, [&](auto d) { return d.units(unit, a.n * 16, len); });
      present |= 1u << s;
    }
    if (walk) {
      // the record's header lines: its directory entries, or its text when the directory cannot address it
      const uint8_t* h = a.hdr + a.hdr_off[rec];
      const uint2* ent = a.hdir + a.hdir_off[rec];
      const uint32_t n_ent = (uint32_t)(a.hdir_off[rec + 1] - a.hdir_off[rec]);
      uint32_t val_off[FEI_MAX_SLOTS], val_len[FEI_MAX_SLOTS];
      uint32_t any_mask = 0;                                   // mode-2 slots ("any header value", utils.py:333-336) already accumulated
      auto any = [&](int s, uint32_t off, uint32_t len) {
        uint32_t acc;
        if constexpr (kHeadNfa)
          acc = field_run(a.prog, a.prog_in_smem, slots[s].off_val_dfa, slots[s].off_val_nfa, [&](auto d) { return d.span(h + off, len); }, h + off, 16, len);
        else acc = dfa_run_at(a.prog, slots[s].off_val_dfa, a.prog_in_smem, h + off, len);
        slot_acc[s] = (any_mask >> s & 1u) ? (slot_acc[s] | acc) : acc;
        any_mask |= 1u << s;
      };
      auto mode = [&](int s) { return slots[s].mode; };
      present = text_record(ent, n_ent)
          ? header_lookup<FEI_MAX_SLOTS>(TextLines{h, h, a.hdr + a.hdr_off[rec + 1], a.prog, ph->off_key_dfa, a.prog_in_smem}, mode, val_off, val_len, any)
          : header_lookup<FEI_MAX_SLOTS>(DirLines{ent, n_ent, a.key_lut}, mode, val_off, val_len, any);
      for (uint32_t m = present; m; m &= m - 1) {
        const int s = __ffs(m) - 1;
        const uint8_t* v = h + val_off[s];
        if constexpr (kHeadNfa)
          slot_acc[s] = field_run(a.prog, a.prog_in_smem, slots[s].off_val_dfa, slots[s].off_val_nfa, [&](auto d) { return d.span(v, val_len[s]); }, v, 16, val_len[s]);
        else slot_acc[s] = dfa_run_at(a.prog, slots[s].off_val_dfa, a.prog_in_smem, h + val_off[s], val_len[s]);
      }
      present |= any_mask;
    }
  }
  for (uint32_t s = 0; s < nslots; ++s)
    if (!(present >> s & 1) && slots[s].empty_if_missing) {   // headers.get("Status", "")
      if constexpr (!kHeadNfa) slot_acc[s] = reinterpret_cast<const fei_prog_dfa*>(a.prog + slots[s].off_val_dfa)->empty_acc;
      else slot_acc[s] = (slots[s].off_val_dfa ? reinterpret_cast<const fei_prog_dfa*>(a.prog + slots[s].off_val_dfa)->empty_acc : 0u) |
                         (slots[s].off_val_nfa ? head_nfa_run(a.prog, slots[s].off_val_nfa, nullptr, 0, 0, 0) : 0u);
      present |= 1u << s;
    }
  uint32_t name_acc[FEI_NAME_FIELDS] = {0, 0, 0, 0, 0};
  if (pre & ph->name_mask) eval_name_fields<kHeadNfa>(NameArgs{a.prog, a.name, a.name_off, a.name_spans, a.ts, a.wall, (bool)a.prog_in_smem}, ph, rec, name_acc);
  uint32_t alive = 0;
  for (uint32_t q = 0; q < ph->n_queries; ++q) {
    if (!(pre >> q & 1)) continue;
    bool ok = true;
    bool fallback = false;                                      // the condition is the fallback field of an absent header
    for (uint32_t c = queries[q].cond_begin; ok && c < queries[q].cond_end; ++c) {
      const fei_prog_cond& cd = conds[c];
      bool r;
      switch (cd.kind) {
        case FEI_C_BODY: continue;                              // evaluated by k_body
        case FEI_C_SLOT:
          if (present >> cd.ref & 1) { r = ((slot_acc[cd.ref] >> cd.bit) & 1u) != cd.negate; if (cd.if_missing == 2) ++c; }
          else if (cd.if_missing == 2) { fallback = true; continue; }   // header absent: the next condition is the fallback field
          else r = cd.if_missing != 0;
          break;
        case FEI_C_NAME: r = ((name_acc[cd.ref < FEI_NAME_FIELDS ? cd.ref : 0] >> cd.bit) & 1u) != cd.negate; break;
        default:
          // meta predicates of a query in `pre` already held in k_head_meta; only a fallback field (skipped there) is still open
          r = fallback ? eval_meta_cond<kFolderBits>(a, rec, cd, flags_acc, a.wall[rec], a.fsb[rec]) : true;
      }
      fallback = false;
      ok = r;
    }
    if (ok) alive |= 1u << q;
  }
  a.alive[rec] = alive;
}

// Per scan: run the key automaton over the corpus' distinct header keys (hdir.cu), one thread per dictionary slot.
__global__ void k_key_lut(const uint8_t* __restrict__ prog, const uint8_t* __restrict__ hdr, const unsigned long long* __restrict__ tag,
                          const unsigned long long* __restrict__ rep, const uint32_t* __restrict__ len, uint32_t* __restrict__ lut) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= kKeySlots) return;
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(prog);
  lut[s] = tag[s] ? Dfa<GlobalTables>(prog, ph->off_key_dfa).span(hdr + rep[s], len[s]) : 0u;
}

// One warp, after k_key_lut: a program slot whose field is spelled exactly one way in the whole corpus can be read from that
// key's value column (if it has one); a field no record carries is absent everywhere; anything else walks the directory.
__global__ void k_slot_cols(const uint8_t* __restrict__ prog, const uint32_t* __restrict__ lut, const int8_t* __restrict__ kid_col,
                            uint32_t n_cols, uint32_t any_text, int8_t* __restrict__ slot_col) {
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(prog);
  const int lane = threadIdx.x & 31;
  for (uint32_t s = 0; s < ph->n_slots && s < FEI_MAX_SLOTS; ++s) {
    uint32_t count = 0, kid = 0;
    for (uint32_t k = lane; k < kKeySlots; k += 32) if (lut[k] >> s & 1u) { ++count; kid = k; }
    for (int o = 16; o; o >>= 1) { count += __shfl_xor_sync(0xffffffffu, count, o); kid = max(kid, __shfl_xor_sync(0xffffffffu, kid, o)); }
    // (records whose header is parsed from its text keep their keys out of the dictionary: with any of those, nothing is "absent everywhere")
    if (lane == 0) slot_col[s] = count == 0 ? (any_text ? (int8_t)-1 : (int8_t)-2) : (count == 1 && n_cols ? kid_col[kid] : (int8_t)-1);
  }
}

// Every CTA of the head kernels first copies the "head" of the program (header, conditions, queries, slots and all
// automata except the big content one: fei_prog_hdr.head_bytes, a few KB) into shared memory with one TMA bulk copy,
// so that the interpretive condition loops and the short automaton runs read LDS instead of chasing global pointers.
constexpr uint32_t kHeadProgSmem = 32 * 1024;
__device__ __forceinline__ const uint8_t* stage_prog_head(const uint8_t* gprog, uint8_t* sprog, uint64_t* bar) {
  const uint32_t head_bytes = reinterpret_cast<const fei_prog_hdr*>(gprog)->head_bytes;
  if (head_bytes == 0 || head_bytes > kHeadProgSmem) return gprog;           // uniform for the whole grid
  if (threadIdx.x == 0) { mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  if (threadIdx.x == 0) { mbar_expect_tx(bar, head_bytes); bulk_g2s(sprog, gprog, head_bytes, bar); }
  mbar_wait(bar, 0);
  return sprog;
}

// k_head_meta streams the 20-byte meta columns, finalises every record that needs no header text and appends
// the others to a work list; k_head_parse then gives each survivor its own thread at full occupancy (a survivor's
// serial header walk does not pin a CTA full of already-finished threads), and the dead records' headers are never read.
struct Survivor { uint32_t rec, pre, flags_acc; };

constexpr int kMetaPer = 4;     // records per thread: the (uniform) condition fetch / decode is paid once for four records

template <bool kFused, bool kHeadNfa, bool kFolderBits>
__global__ void __launch_bounds__(256, 5) k_head_meta(HeadArgs a, Survivor* __restrict__ list, unsigned int* __restrict__ count) {
  __shared__ __align__(128) uint8_t sprog[kHeadProgSmem];
  __shared__ uint64_t bar;
  a.prog = stage_prog_head(a.prog, sprog, &bar);
  a.prog_in_smem = a.prog == sprog;
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const fei_prog_cond* conds = reinterpret_cast<const fei_prog_cond*>(a.prog + ph->off_conds);
  const fei_prog_query* queries = reinterpret_cast<const fei_prog_query*>(a.prog + ph->off_queries);
  const uint64_t base = blockIdx.x * (uint64_t)(256 * kMetaPer) + threadIdx.x;
  uint32_t fsb[kMetaPer], flags_acc[kMetaPer], pre[kMetaPer];
  int64_t wall[kMetaPer];
  uint64_t f8[kMetaPer];
  bool valid[kMetaPer];
#pragma unroll
  for (int r = 0; r < kMetaPer; ++r) {
    const uint64_t i = base + (uint64_t)r * 256;
    valid[r] = i < a.n;
    fsb[r] = valid[r] ? a.fsb[i] : 0u; wall[r] = valid[r] ? a.wall[i] : 0; f8[r] = valid[r] ? a.flags8[i] : 0ull;
    flags_acc[r] = 0; pre[r] = 0;
  }
  if (ph->off_flags_dfa) {                                     // flags string (search.py:105-106): up to 7 letters in flags8
#pragma unroll
    for (int r = 0; r < kMetaPer; ++r)
      flags_acc[r] = dfa_run_at(a.prog, ph->off_flags_dfa, a.prog_in_smem, [&](auto d) { return d.u64(f8[r], (uint32_t)(f8[r] >> 56)); });
  }
  if constexpr (kHeadNfa) {
    if (const uint32_t off = head_nfa_off(a.prog, ph, 0)) {
      for (int r = 0; r < kMetaPer; ++r) flags_acc[r] |= head_nfa_run(a.prog, off, nullptr, 0, (uint32_t)(f8[r] >> 56), f8[r]);
    }
  }
  for (uint32_t q = 0; q < ph->n_queries; ++q) {
    bool ok[kMetaPer];
#pragma unroll
    for (int r = 0; r < kMetaPer; ++r) ok[r] = true;
    for (uint32_t c = queries[q].cond_begin; c < queries[q].cond_end; ++c) {
      const fei_prog_cond cd = conds[c];
      if (cd.kind == FEI_C_SLOT && cd.if_missing == 2) { ++c; continue; }     // header-or-fallback pair: decided in phase 2
#pragma unroll
      for (int r = 0; r < kMetaPer; ++r) ok[r] = ok[r] && (!valid[r] || eval_meta_cond<kFolderBits>(a, base + (uint64_t)r * 256, cd, flags_acc[r], wall[r], fsb[r]));
    }
#pragma unroll
    for (int r = 0; r < kMetaPer; ++r) if (ok[r]) pre[r] |= 1u << q;
  }
  const uint32_t later_mask = ph->slot_mask | ph->name_mask;
  if (kFused) {
    // header / name fields right here: with value columns a record's fields are a couple of coalesced loads and short
    // automaton runs, so there is no long per-record walk that would pin the CTA, and the work list is not needed
    for (int r = 0; r < kMetaPer; ++r) {
      const uint64_t i = base + (uint64_t)r * 256;
      if (!valid[r]) continue;
      if ((pre[r] & later_mask) == 0) a.alive[i] = pre[r];
      else head_finish<kHeadNfa, kFolderBits>(a, i, pre[r], flags_acc[r], (pre[r] & ph->slot_mask) != 0);
    }
    return;
  }
  const int lane = threadIdx.x & 31;
  // survivors: slots are reserved per warp in shared memory and per CTA with ONE global atomic (a global atomic per
  // warp puts 260 k same-address atomics on the L2 for 10 M records, which costs more than streaming the columns)
  __shared__ unsigned int cta_count, cta_base;
  if (threadIdx.x == 0) cta_count = 0;
  __syncthreads();
  bool later[kMetaPer];
  uint32_t bal[kMetaPer];
  unsigned int warp_total = 0;
#pragma unroll
  for (int r = 0; r < kMetaPer; ++r) {
    const uint64_t i = base + (uint64_t)r * 256;
    later[r] = valid[r] && (pre[r] & later_mask) != 0;
    if (valid[r] && !later[r]) a.alive[i] = pre[r];            // no header / name condition left: pre is the verdict
    bal[r] = __ballot_sync(0xffffffffu, later[r]);
    warp_total += __popc(bal[r]);
  }
  unsigned int warp_base = 0;
  if (lane == 0 && warp_total) warp_base = atomicAdd(&cta_count, warp_total);
  warp_base = __shfl_sync(0xffffffffu, warp_base, 0);
  __syncthreads();
  if (threadIdx.x == 0 && cta_count) cta_base = atomicAdd(count, cta_count);
  __syncthreads();
  unsigned int slot = cta_base + warp_base;
#pragma unroll
  for (int r = 0; r < kMetaPer; ++r) {
    if (later[r]) list[slot + __popc(bal[r] & ((1u << lane) - 1u))] = Survivor{(uint32_t)(base + (uint64_t)r * 256), pre[r], flags_acc[r]};
    slot += __popc(bal[r]);
  }
}

template <bool kHeadNfa, bool kFolderBits>
__global__ void __launch_bounds__(256, 5) k_head_parse(HeadArgs a, const Survivor* __restrict__ list, const unsigned int* __restrict__ n_list) {
  __shared__ __align__(128) uint8_t sprog[kHeadProgSmem];
  __shared__ uint64_t bar;
  const unsigned int n_surv = *n_list;                         // written by k_head_meta earlier on this stream: no host round trip
  if (blockIdx.x * blockDim.x >= n_surv) return;               // the grid is sized for "every record survives"
  a.prog = stage_prog_head(a.prog, sprog, &bar);
  a.prog_in_smem = a.prog == sprog;
  const unsigned int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_surv) return;
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const Survivor sv = list[t];
  head_finish<kHeadNfa, kFolderBits>(a, sv.rec, sv.pre, sv.flags_acc, (sv.pre & ph->slot_mask) != 0);
}

// ---------------------------------------------------------------- body kernel
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  }
}
__device__ __forceinline__ uint4 ldg_stream16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
// Stage a content automaton into shared memory with TMA bulk copies (cp.async.bulk + mbarrier), at most 32 KiB per copy.
// Its __syncthreads also publishes to the CTA what any thread wrote to shared memory before the call.
__device__ __forceinline__ void stage_table(uint8_t* dst, const uint8_t* src, uint32_t bytes, uint64_t* bar) {
  if (threadIdx.x == 0) { mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, bytes);
    for (uint32_t o = 0; o < bytes; o += 32768u) {
      uint32_t nb = bytes - o < 32768u ? bytes - o : 32768u;
      bulk_g2s(dst + o, src + o, nb, bar);
    }
  }
  mbar_wait(bar, 0);
}

struct BodyArgs {
  const uint8_t* prog;
  const uint8_t* tiles; const uint64_t* grp_base; const uint32_t* grp_rec; const uint32_t* grp_len;
  uint64_t n_groups;
  uint32_t* hits;              // in: alive masks (when has_alive), out: final hit masks
  int has_alive;
  unsigned long long* counter; // [1] = tile bytes of the groups entered, [3] = tile bytes requested (k_body: 16 per lane and
                               // row it loaded), [4] = live records (gather), [5] = set when a list-building wait timed out
  unsigned long long gather_max;   // k_body_sticky stands down (and k_body_gather runs) when 0 < counter[4] <= gather_max
  unsigned long long* next;    // hands out the groups [0, n_groups) of the one launch
  // window w (groups [w * kWindow / 32, (w + 1) * kWindow / 32)) is finished when win_done[w] reaches kWindow / 32; null unless
  // the warp that finishes a window has work to do for it (ordered lists, peer push)
  unsigned int* win_done;
  // multi-GPU, fused exchange: the warp that completes a window stores the window's 4096 hit masks into every rank's rank-major
  // mask buffer (peer memory over NVLink / NVSwitch, mapped with CUDA IPC) -- the transfer of a finished window runs under the scan
  // of the next ones, from inside the scan kernel.  push_peers is a DEVICE array (a dynamic index into this by-value struct would
  // make ptxas copy it to local memory).
  uint32_t* const* push_peers; uint32_t push_n; unsigned long long push_off, n_records;
  // ordered hit lists (k_body): the warp that completes a window also writes the window's part of every query's list
  // (build_window_lists); win_state holds kWinBytes of look-back / count / emit state per window, zeroed once per scan.
  // List entries are corpus-local record indices (32-bit, like grp_rec).
  uint32_t* lists; unsigned long long list_stride;
  unsigned long long* totals; uint8_t* win_state; uint32_t nq;
};
constexpr uint32_t kGroupsPerWindow = kWindow / 32;
__device__ __noinline__ void publish_window(const uint32_t* __restrict__ hits, uint32_t* const* __restrict__ peers, uint32_t n_peers,
                                            unsigned long long off, unsigned long long n_records, unsigned long long w, int lane) {
  __threadfence();                                   // acquire side of the window counter: the other groups' masks are visible now
  const unsigned long long r0 = w * kWindow;
  const uint32_t cnt = (uint32_t)((n_records - r0) < kWindow ? (n_records - r0) : kWindow);
  const uint32_t* src = hits + r0;                   // 16 KiB aligned; the destination is 16-byte aligned too (n_max is a multiple of 4)
  for (uint32_t p = 0; p < n_peers; ++p) {
    uint32_t* dst = peers[(p + (uint32_t)w) % n_peers];        // successive windows start with different ranks
    if (!dst) continue;
    dst += off + r0;
    for (uint32_t i = lane * 4u; i < cnt; i += 128u) {
      if (i + 4u <= cnt) {
        const uint4 v = __ldcg(reinterpret_cast<const uint4*>(src + i));        // L2: another SM wrote them
        *reinterpret_cast<uint4*>(dst + i) = v;
      } else {
        for (uint32_t j = i; j < cnt; ++j) dst[j] = __ldcg(src + j);
      }
    }
  }
  __threadfence_system();                            // the remote stores are ordered before this kernel's completion is observed
}
// ---- ordered hit lists: the per-32-record pieces of the compaction, shared by k_count / k_emit and build_window_lists
// lane q (< nq) gets the number of the warp's 32 masks that have bit q
__device__ __forceinline__ uint32_t count_hits32(uint32_t m, uint32_t nq, int lane) {
  uint32_t cnt = 0;
#pragma unroll 8
  for (uint32_t q = 0; q < nq; ++q) {                // unrolled: independent ballots in flight together
    const uint32_t b = __popc(__ballot_sync(0xffffffffu, (m >> q) & 1u));
    if (lane == (int)q) cnt = b;
  }
  return cnt;
}
// one query over the warp's 32 records in lane order: a lane with `hit` stores `rec` at list[hits of the lanes below it]
// (the caller points `list` at the rank of the warp's first hit); returns the warp's hits
template <class T>
__device__ __forceinline__ uint32_t emit_hits32(bool hit, T* list, T rec, int lane) {
  const uint32_t bal = __ballot_sync(0xffffffffu, hit);
  if (hit) __stcs(list + __popc(bal & ((1u << lane) - 1u)), rec);       // nothing reads them back soon
  return __popc(bal);
}

// Per-window state of the list building, one record of kWinBytes per window, zeroed once per scan:
//   desc[32]  look-back descriptor of (window, query): flag in the top 2 bits over a 62-bit hit count;
//   ready     set (release) once excl[] below is written;   claim: query slices of the window's emit handed out so far;
//   excl[32]  hits of query q in all earlier windows;
//   cnt[128]  one 32-byte row per group of the window (store_group_counts): byte 4k + j = the group's hits of query 8j + k.
// The emit of a window is cut into slices of kEmitQueries queries, claimed one at a time: the completer of the window takes
// them, and so do warps that find no group left to scan (help_tail), so the last windows' lists are written by many warps
// instead of one each after the scan.  A slice spans the whole window: the length sort spreads the records of a group over
// the window, so the group counts give per-query window totals but not the offsets of record ranges inside it.
constexpr unsigned long long kDescAggregate = 1ull << 62, kDescPrefix = 2ull << 62, kDescCount = (1ull << 62) - 1;
constexpr uint32_t kEmitQueries = 2, kEmitRows = 4;  // queries per claimed slice; rows of 32 masks loaded at once
constexpr uint32_t kWinDesc = 0, kWinCtl = 256, kWinExcl = 272, kWinCnt = 528, kWinBytes = kWinCnt + kGroupsPerWindow * 32;
static_assert(kWinCnt % 16 == 0 && kWinBytes % 16 == 0, "count rows are stored 16 bytes at a time");
constexpr uint32_t kHelpWindows = 64;              // windows at the end of the scan that warps without a group help with
__device__ __forceinline__ void st_release_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// The hits per query of group g, from the 32 masks its scanning warp still holds (0 in lanes without a record), into the
// group's count row of its window: byte j of sum k counts query 8j + k (at most 32, so no carry into the next byte).  Out of
// line, like build_window_lists: the row loop of k_body keeps its register allocation.
__device__ __noinline__ void store_group_counts(uint8_t* __restrict__ win, unsigned long long g, uint32_t m, int lane) {
  uint32_t c[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) c[k] = __reduce_add_sync(0xffffffffu, (m >> k) & 0x01010101u);
  if (lane == 0) {
    uint4* row = reinterpret_cast<uint4*>(win + (g / kGroupsPerWindow) * kWinBytes + kWinCnt + (g % kGroupsPerWindow) * 32);
    row[0] = make_uint4(c[0], c[1], c[2], c[3]);
    row[1] = make_uint4(c[4], c[5], c[6], c[7]);
  }
}

// Claims query slices of window w's emit until none is left and writes each slice's hits in record order (the window is
// ready).  Every lane keeps the address of the next entry of each query of the slice (the same in all lanes: no shuffles);
// corpus-local record indices are 32-bit.  Queries q0 + j >= nq have no bit in any mask, so nothing is stored for them.
__device__ __forceinline__ void emit_claimed(const uint32_t* __restrict__ hits, uint8_t* __restrict__ win, uint32_t* __restrict__ lists,
                                             unsigned long long stride, unsigned long long n_records, uint32_t nq,
                                             unsigned long long w, int lane) {
  uint8_t* wr = win + w * kWinBytes;
  unsigned int* claim = reinterpret_cast<unsigned int*>(wr + kWinCtl) + 1;
  const unsigned long long* excl = reinterpret_cast<const unsigned long long*>(wr + kWinExcl);
  const unsigned long long r0 = w * kWindow;
  const uint32_t cnt = (uint32_t)((n_records - r0) < kWindow ? (n_records - r0) : kWindow);   // the last window may be short
  const uint32_t* src = hits + r0;
  for (;;) {
    uint32_t b = 0;
    if (lane == 0) b = atomicAdd(claim, 1u);
    b = __shfl_sync(0xffffffffu, b, 0);
    const uint32_t q0 = b * kEmitQueries;
    if (q0 >= nq) break;
    uint32_t* at[kEmitQueries];                                          // where the next hit of query q0 + j goes
#pragma unroll
    for (uint32_t j = 0; j < kEmitQueries; ++j) at[j] = lists + (q0 + j) * stride + __ldcg(excl + q0 + j);
    for (uint32_t i = 0; i < cnt; i += kEmitRows * 32) {
      uint32_t m[kEmitRows];                                              // kEmitRows rows of masks in flight at once
#pragma unroll
      for (uint32_t r = 0; r < kEmitRows; ++r) m[r] = i + r * 32 + lane < cnt ? __ldcg(src + i + r * 32 + lane) : 0u;   // L2: other SMs wrote them
#pragma unroll
      for (uint32_t r = 0; r < kEmitRows; ++r) {
        const uint32_t rec = (uint32_t)r0 + i + r * 32 + lane;
#pragma unroll
        for (uint32_t j = 0; j < kEmitQueries; ++j) at[j] += emit_hits32((m[r] >> (q0 + j)) & 1u, at[j], rec, lane);
      }
    }
  }
}

// Window w's part of the ordered per-query lists, started by the warp that completed the window (out of line, like
// publish_window: the row loop of k_body keeps its register allocation).  Lane q owns query q:
//   1. add up the window's hits from the count rows of its 128 groups (store_group_counts; no mask is read) and publish the
//      sum as the window's aggregate;
//   2. decoupled look-back: add up the aggregates of windows w-1, w-2, ... until one carries an inclusive prefix (or window 0
//      is reached), then publish this window's inclusive prefix, its exclusive one and `ready`; the last window writes totals[q];
//   3. emit query slices of the window until every slice is claimed (emit_claimed).
// Progress: a completer publishes its aggregate before it looks back, and it holds no unfinished group (its own group was
// done when it got here, and it claims the next one only after returning).  Groups are handed out in increasing order and
// only to resident warps, so every window it waits for is either complete -- its completer publishes the aggregate without
// waiting for anything -- or has groups that warps still scanning will finish.
// The time limit only guards against a scan that died: it sets err (reported by finish_timing), and the
// window publishes its prefix anyway so that later windows do not wait on it too.
__device__ __noinline__ void build_window_lists(const uint32_t* __restrict__ hits, uint8_t* __restrict__ win, uint32_t* __restrict__ lists,
                                                unsigned long long stride, unsigned long long* __restrict__ totals,
                                                unsigned long long* __restrict__ err, unsigned long long n_records, uint32_t nq,
                                                unsigned long long w, int lane) {
  __threadfence();                                   // acquire side of the window counter: the other groups' masks and counts are visible now
  const unsigned long long r0 = w * kWindow;
  const uint32_t cnt = (uint32_t)((n_records - r0) < kWindow ? (n_records - r0) : kWindow);
  const bool own = lane < (int)nq;
  uint8_t* wr = win + w * kWinBytes;
  // lane l adds word l & 7 of the rows l >> 3, (l >> 3) + 4, ... (one warp load covers four whole rows): bytes 0 and 2 in lo,
  // 1 and 3 in hi, in 16-bit halves (a window has at most 4096 hits of a query); then the four lanes of each word add theirs
  const uint32_t* rows = reinterpret_cast<const uint32_t*>(wr + kWinCnt);
  uint32_t lo = 0, hi = 0;
#pragma unroll 8
  for (uint32_t r = (uint32_t)lane >> 3; r < kGroupsPerWindow; r += 4) {
    const uint32_t v = __ldcg(rows + r * 8 + (lane & 7));                // L2: other SMs wrote them
    lo += v & 0x00FF00FFu; hi += (v >> 8) & 0x00FF00FFu;
  }
  lo += __shfl_xor_sync(0xffffffffu, lo, 8); hi += __shfl_xor_sync(0xffffffffu, hi, 8);
  lo += __shfl_xor_sync(0xffffffffu, lo, 16); hi += __shfl_xor_sync(0xffffffffu, hi, 16);
  const uint32_t j = (uint32_t)lane >> 3;                                  // lane q holds word q & 7, whose byte q >> 3 counts query q
  const uint32_t agg = ((j & 1u) ? hi : lo) >> (16u * (j >> 1)) & 0xFFFFu;
  unsigned long long* mine = reinterpret_cast<unsigned long long*>(wr + kWinDesc) + lane;
  unsigned long long excl = 0;
  if (w == 0) {
    if (own) st_release_u64(mine, kDescPrefix | agg);
  } else {
    if (own) st_release_u64(mine, kDescAggregate | agg);
    unsigned long long p = w - 1;
    bool done = !own;
    const long long t0 = clock64();
    for (;;) {
      bool moved = false;
      if (!done) {
        const unsigned long long v = ld_acquire_u64(reinterpret_cast<const unsigned long long*>(win + p * kWinBytes + kWinDesc) + lane);
        if (v >> 62) {
          excl += v & kDescCount; moved = true;
          if ((v >> 62) == 2 || p == 0) done = true; else --p;
        }
      }
      if (__all_sync(0xffffffffu, done)) break;
      if (!__any_sync(0xffffffffu, moved)) {
        if (clock64() - t0 > 20000000000ll) { if (lane == 0) atomicExch(err, 1ull); break; }     // ~10 s
        __nanosleep(256);
      }
    }
    if (own) st_release_u64(mine, kDescPrefix | (excl + agg));
  }
  if (own && r0 + cnt == n_records) totals[lane] = excl + agg;
  reinterpret_cast<unsigned long long*>(wr + kWinExcl)[lane] = excl;
  __threadfence();
  __syncwarp();
  if (lane == 0) st_release_u32(reinterpret_cast<unsigned int*>(wr + kWinCtl), 1u);    // offsets published: anyone may emit
  emit_claimed(hits, win, lists, stride, n_records, nq, w, lane);
}

// A warp that finds no group left to scan helps emit the last windows of the scan [0, n_windows): the groups of those
// windows are all handed out, so each becomes ready once its completer has looked back (see build_window_lists); a helper
// holds no group and waits for nothing else.  Windows whose slices are all claimed are skipped.
__device__ __noinline__ void help_tail(const uint32_t* __restrict__ hits, uint8_t* __restrict__ win, uint32_t* __restrict__ lists,
                                       unsigned long long stride, unsigned long long* __restrict__ err,
                                       unsigned long long n_records, uint32_t nq, unsigned long long n_windows, int lane) {
  const unsigned long long w0 = n_windows > kHelpWindows ? n_windows - kHelpWindows : 0;
  const uint32_t slices = (nq + kEmitQueries - 1) / kEmitQueries;
  for (unsigned long long w = w0; w < n_windows; ++w) {
    const unsigned int* ctl = reinterpret_cast<const unsigned int*>(win + w * kWinBytes + kWinCtl);
    if (__ldcg(ctl + 1) >= slices) continue;                     // every slice already taken
    const long long t0 = clock64();
    while (__any_sync(0xffffffffu, ld_acquire_u32(ctl) == 0u)) {
      if (clock64() - t0 > 20000000000ll) { if (lane == 0) atomicExch(err, 1ull); return; }    // ~10 s
      __nanosleep(512);
    }
    emit_claimed(hits, win, lists, stride, n_records, nq, w, lane);
  }
}

// kPush: the multi-GPU instantiation; the single-GPU kernels do not carry the exchange code (it cost 0.5 % of the headline
// when it was compiled into the one kernel: a shuffle and a branch per group, and a different register allocation).
// kLists: k_body, which builds the ordered hit lists window by window when a.lists is set; m is the lane's hit mask
// (0 without a record), whose per-query counts go to the window's state before the group counts as done.
template <bool kPush, bool kLists>
__device__ __forceinline__ void signal_group_done(const BodyArgs& a, unsigned long long g, uint32_t m, int lane) {
  if (!a.win_done) return;
  if (kLists && a.lists) store_group_counts(a.win_state, g, m, lane);
  __threadfence();                                   // this lane's hit mask (and lane 0's count row) is visible device-wide ...
  __syncwarp();
  unsigned int old = 0;
  if (lane == 0) old = atomicAdd(a.win_done + g / kGroupsPerWindow, 1u);   // ... before the group counts as done
  if ((kPush && a.push_n) || (kLists && a.lists)) {
    old = __shfl_sync(0xffffffffu, old, 0);
    if (old + 1u == kGroupsPerWindow) {
      const unsigned long long w = g / kGroupsPerWindow;
      if (kPush && a.push_n) publish_window(a.hits, a.push_peers, a.push_n, a.push_off, a.n_records, w, lane);
      if (kLists && a.lists) build_window_lists(a.hits, a.win_state, a.lists, a.list_stride, a.totals, a.counter + 5, a.n_records, a.nq, w, lane);
    }
  }
}

constexpr int kBodyThreads = 1024;

__device__ __forceinline__ uint32_t shl_clamp(uint32_t v, uint32_t n) {   // PTX shl clamps: n >= 32 -> 0
  uint32_t r;
  asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(v), "r"(n));
  return r;
}

// The size of a table entry as a value ptxas cannot see.  With the immediate 2 it turns column * 2 + trans_s into LEA, an
// ALU-pipe instruction like PRMT, SHF and LOP3; with a register operand the multiply-add stays IMAD on the FMA pipe.
// That is 16 of 93 ALU-pipe instructions per row of k_body<direct, acc64> (DESIGN 5.1).
__constant__ uint32_t c_entry_bytes = 2;

// One DFA step.  kAcc selects how accepting states are recorded (they are numbered 0..n_acc-1):
//   1 / 2 : branch-free, bit k of (a0,a1) = "accepting state k was visited" (n_acc <= 32 / <= 64):
//           no second shared-memory lookup and no divergent branch in the byte loop; the pattern
//           masks out[k] are OR-ed once per record from the visited-state bits;
//   0     : generic: out[] lookup when the new state is accepting.
// Address arithmetic is written so that it lands on the FMA pipe (IMAD) and only the byte extract
// (PRMT) and the accept bits (SHL/LOP3) use the ALU pipe: the loop is ALU-pipe / LDS-wavefront bound.
template <bool kDirect, int kAcc>
struct BodyDfa {
  uint32_t trans_s;            // shared-space address of the transition table
  const uint32_t* out; const uint8_t* cls;
  uint32_t stride2, n_acc;     // stride2 = row stride in bytes
  uint32_t entry_bytes;        // c_entry_bytes in a register
  uint32_t s, a0;
  unsigned long long a64;
  __device__ __forceinline__ void step(uint32_t b) {
    uint32_t col = kDirect ? b : cls[b];
    uint32_t t, addr;
    if (kAcc == 3) asm("mad.lo.u32 %0, %1, 2, %2;" : "=r"(t) : "r"(col), "r"(trans_s));
    else asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(t) : "r"(col), "r"(entry_bytes), "r"(trans_s));   // IMAD (FMA pipe)
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(addr) : "r"(s), "r"(stride2), "r"(t));
    uint16_t nxt;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(nxt) : "r"(addr));
    s = nxt;
    if (kAcc == 1) a0 |= shl_clamp(1u, s);            // s >= 32 shifts out: no bit
    if (kAcc == 2) { unsigned long long bit; asm("shl.b64 %0, %1, %2;" : "=l"(bit) : "l"(1ull), "r"(s)); a64 |= bit; }   // s >= 64: no bit
    if (kAcc == 0) { if (s < n_acc) a0 |= out[s]; }
    // kAcc == 3 ("sticky" single-pattern automaton): nothing to record, the verdict is endout[final state]
  }
  __device__ __forceinline__ void word(uint32_t w) {
    step(__byte_perm(w, 0, 0x4440)); step(__byte_perm(w, 0, 0x4441)); step(__byte_perm(w, 0, 0x4442)); step(__byte_perm(w, 0, 0x4443));
  }
  __device__ __forceinline__ void word_partial(uint32_t w, int nbytes) {
#pragma unroll
    for (int j = 0; j < 4; ++j) if (j < nbytes) step((w >> (8 * j)) & 0xFFu);
  }
  __device__ __forceinline__ void reset(uint32_t start) {
    s = start; a0 = 0; a64 = 0;
    if (kAcc == 0) a0 = start < n_acc ? out[start] : 0u;
    if (kAcc == 1) a0 = shl_clamp(1u, start);
    if (kAcc == 2) a64 = start < 64 ? 1ull << start : 0ull;
  }
  __device__ __forceinline__ uint32_t finish(const uint32_t* endout) const {
    uint32_t acc = endout[s];
    if (kAcc == 3) return acc;
    if (kAcc == 0) return acc | a0;
    unsigned long long m = kAcc == 1 ? (unsigned long long)a0 : a64;
    if (n_acc < 64) m &= (1ull << n_acc) - 1ull;
    while (m) { int k = __ffsll((long long)m) - 1; m &= m - 1; acc |= out[k]; }
    return acc;
  }
};

// Early exit of k_body (kAcc 0 / 1 / 2).  A record's content verdict acc = OR of out[] over the states it visits | endout[final
// state] only ever gains bits, and its hit mask reads no bit of acc but those of the body conditions of its alive queries
// (`need`).  Once every bit of `need` is set by the out[] of a visited state, each of those conditions is decided whatever the
// rest of the record holds (a negated one is false for good), so a lane that stops there writes the hit mask the full scan
// would: finish() sets the same bits of `need`, and the other bits of acc are not read.  Bits that only endout[] sets ($, \Z)
// never enter the running mask, so records that need them are read to the end.
// The check runs between blocks of kDecideRows rows, outside the row loop: a check inside it, even one every 4th row, made
// every row slower on H100 than the skipped lookups saved (DESIGN 5.1).  The
// accepting states visited since the last check are folded into `rem` (the bits of need still unset), each at most once per
// record (`folded`).
constexpr uint32_t kDecideRows = 16;
template <int kAcc>
struct BodyDecide {
  using Bits = typename std::conditional<kAcc == 2, unsigned long long, uint32_t>::type;
  uint32_t rem;                // bits of need not yet set
  Bits folded;                 // accepting states already folded into rem (and the bit positions of non-accepting states)
  __device__ __forceinline__ void reset(uint32_t need, uint32_t n_acc) {
    rem = need;
    if (kAcc == 1) folded = n_acc >= 32 ? 0u : ~0u << n_acc;
    if (kAcc == 2) folded = n_acc >= 64 ? 0ull : ~0ull << n_acc;
  }
  template <bool kDirect>
  __device__ __forceinline__ bool decided(const BodyDfa<kDirect, kAcc>& d) {
    if (kAcc == 0) rem &= ~d.a0;                              // a0 holds the pattern masks already
    if (kAcc == 1 || kAcc == 2) {
      Bits fresh = (kAcc == 1 ? (Bits)d.a0 : (Bits)d.a64) & ~folded;
      if (fresh) {
        folded |= fresh;
        do { rem &= ~d.out[__ffsll((long long)fresh) - 1]; fresh &= fresh - 1; } while (fresh);
      }
    }
    return rem == 0;
  }
};

// The hit mask of a record whose content verdict is acc: of the queries in `alive`, those whose every content condition
// holds (bit `bit` of acc, inverted when negated).  Conditions of the other kinds are already settled in `alive`.
__device__ __forceinline__ uint32_t content_hits(uint32_t acc, uint32_t alive, const fei_prog_query* queries,
                                                 const fei_prog_cond* conds, uint32_t nq) {
  uint32_t hit = 0;
  for (uint32_t q = 0; q < nq; ++q) {
    if (!(alive >> q & 1)) continue;
    bool ok = true;
    for (uint32_t c = queries[q].cond_begin; ok && c < queries[q].cond_end; ++c) {
      const fei_prog_cond& cd = conds[c];
      if (cd.kind == FEI_C_BODY) ok = ((acc >> cd.bit) & 1u) != cd.negate;
    }
    if (ok) hit |= 1u << q;
  }
  return hit;
}

template <bool kDirect, int kAcc, bool kPush>
__global__ void __launch_bounds__(kBodyThreads, 1) k_body(BodyArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  __shared__ uint32_t q_need[33];                  // [q] = content bits the conditions of query q read; [32] = OR over all queries
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const fei_prog_dfa* dd = reinterpret_cast<const fei_prog_dfa*>(a.prog + ph->off_body_dfa);
  const uint32_t table_bytes = dd->table_bytes;
  const fei_prog_cond* conds = reinterpret_cast<const fei_prog_cond*>(a.prog + ph->off_conds);
  const fei_prog_query* queries = reinterpret_cast<const fei_prog_query*>(a.prog + ph->off_queries);
  const uint32_t nq = ph->n_queries;
  // written by warp 0 before stage_table, whose __syncthreads publishes it to the other warps
  if (kAcc != 3 && threadIdx.x < 32) {
    uint32_t bits = 0;
    if (threadIdx.x < nq)
      for (uint32_t c = queries[threadIdx.x].cond_begin; c < queries[threadIdx.x].cond_end; ++c)
        if (conds[c].kind == FEI_C_BODY) bits |= 1u << conds[c].bit;
    q_need[threadIdx.x] = bits;
    bits = __reduce_or_sync(0xffffffffu, bits);
    if (threadIdx.x == 0) q_need[32] = bits;
  }
  stage_table(smem, a.prog + dd->off_trans, table_bytes, &bar);
  const uint32_t* endout = reinterpret_cast<const uint32_t*>(smem + (dd->off_endout - dd->off_trans));
  const uint32_t start = dd->start;
  const uint32_t all_q = nq >= 32 ? 0xFFFFFFFFu : ((1u << nq) - 1u);
  const int lane = threadIdx.x & 31;
  unsigned long long touched = 0;
  uint32_t rows_read = 0;                          // rows of 16 bytes this lane requested
  BodyDfa<kDirect, kAcc> d;
  BodyDecide<kAcc> dec;
  d.trans_s = smem_u32(smem);
  d.out = reinterpret_cast<const uint32_t*>(smem + (dd->off_out - dd->off_trans));
  d.cls = smem + (dd->off_cls - dd->off_trans);
  d.stride2 = dd->row_stride * 2u; d.n_acc = dd->n_acc; d.entry_bytes = c_entry_bytes;
  const uint32_t sticky_state = dd->sticky ? dd->sticky - 1u : 0xFFFFFFFFu;

  for (;;) {
    unsigned long long g = 0;
    if (lane == 0) g = atomicAdd(a.next, 1ull);
    g = __shfl_sync(0xffffffffu, g, 0);
    if (g >= a.n_groups) break;
    const uint32_t rec = a.grp_rec[g * 32 + lane];
    const uint32_t len = a.grp_len[g * 32 + lane];
    const uint32_t units = (len + 15) >> 4;
    uint32_t alive = 0;
    if (rec != kInvalidRec) alive = a.has_alive ? a.hits[rec] : all_q;
    const bool live = alive != 0;
    if (__ballot_sync(0xffffffffu, live) == 0) {              // nobody in this group can still match: skip its bytes
      if (rec != kInvalidRec && !a.has_alive) a.hits[rec] = 0;
      signal_group_done<kPush, true>(a, g, 0u, lane);
      continue;
    }
    const uint8_t* row = a.tiles + a.grp_base[g] * 16;
    const uint32_t maxu = __shfl_sync(0xffffffffu, units, 0);
    // rows below plain_end hold 16 bytes of every one of the 32 records: 512 bytes each, no partial row
    const uint32_t minu = kAcc == 3 ? 0u : __reduce_min_sync(0xffffffffu, units);
    const uint32_t plain_end = minu ? minu - 1u : 0u;
    if (lane == 0) touched += (a.grp_base[g + 1] - a.grp_base[g]) * 16;
    d.reset(start);
    // lim: rows this lane steps through; units, or fewer once its verdicts are decided (0: not live, or decided at the start)
    uint32_t lim = live ? units : 0;
    if (kAcc != 3 && live) {
      uint32_t need = q_need[32];
      if (alive != all_q) {
        need = 0;
        for (uint32_t q = alive; q; q &= q - 1) need |= q_need[__ffs(q) - 1];
      }
      dec.reset(need, d.n_acc);
      if (dec.decided(d)) lim = 0;
    }
    // software pipeline: the next row's 16 bytes are in flight while this row runs through the DFA
    uint4 cur = make_uint4(0, 0, 0, 0);
    if (0 < lim) { cur = ldg_stream16(row + lane * 16); ++rows_read; }
    for (uint32_t k0 = 0; k0 < maxu;) {
      const uint32_t k1 = kAcc == 3 || maxu - k0 <= kDecideRows ? maxu : k0 + kDecideRows;
      bool stop = false;
      // The block's plain rows, without the per-row lane count, 64-bit row step and partial-row test of the loop below.  A lane
      // runs all of them or none: lim is its units, or a block boundary where it was decided.  The test of k against lim inside
      // the loop is always true; it ends the basic block after the load, which ptxas otherwise sinks below the row's tenth
      // lookup, and a load issued that late arrives late (DESIGN 5.1).  The row four ahead is asked into L2 meanwhile.
      if constexpr (kAcc != 3) {
        const uint32_t kp = k1 < plain_end ? k1 : plain_end;
        if (k0 < kp) {
          if (k0 < lim) {
            const uint8_t* p = row + lane * 16;
#pragma unroll 1
            for (uint32_t k = k0; k < kp; ++k) {
              p += 512;
              const uint4 nxt = ldg_stream16(p);
              if (k + 4 < minu) asm volatile("prefetch.global.L2 [%0];" :: "l"(p + 3 * 512));
              if (k < lim) { d.word(cur.x); d.word(cur.y); d.word(cur.z); d.word(cur.w); }
              cur = nxt;
            }
            rows_read += kp - k0;
          }
          row += (uint64_t)(kp - k0) * 512;
          k0 = kp;
        }
      }
      for (uint32_t k = k0; k < k1; ++k) {
        const uint32_t m = __popc(__ballot_sync(0xffffffffu, k < units));
        const uint8_t* next_row = row + (uint64_t)m * 16;
        uint4 nxt = make_uint4(0, 0, 0, 0);
        if (k + 1 < lim) { nxt = ldg_stream16(next_row + lane * 16); ++rows_read; }
        if (k < lim) {
          int nb = (int)len - (int)(k * 16);
          if (nb >= 16) { d.word(cur.x); d.word(cur.y); d.word(cur.z); d.word(cur.w); }
          else { d.word_partial(cur.x, nb); d.word_partial(cur.y, nb - 4); d.word_partial(cur.z, nb - 8); d.word_partial(cur.w, nb - 12); }
        }
        cur = nxt; row = next_row;
        // sticky automaton: stop reading this group as soon as every live lane has either matched or ended
        if (kAcc == 3 && __ballot_sync(0xffffffffu, live && k + 1 < units && d.s != sticky_state) == 0) { stop = true; break; }
      }
      if (stop) break;
      k0 = k1;
      // a decided lane steps no further; row k1, already in flight, is dropped.  The group ends when no lane has rows left.
      if (kAcc != 3 && k1 < lim && dec.decided(d)) lim = k1;
      if (__ballot_sync(0xffffffffu, k1 < lim) == 0) break;
    }
    uint32_t hit = 0;
    if (live) {
      hit = content_hits(d.finish(endout), alive, queries, conds, nq);
      a.hits[rec] = hit;
    } else if (rec != kInvalidRec && !a.has_alive) {
      a.hits[rec] = 0;
    }
    signal_group_done<kPush, true>(a, g, hit, lane);
  }
  if (a.lists && a.win_done)                       // no group left: help write the lists of the scan's last windows
    help_tail(a.hits, a.win_state, a.lists, a.list_stride, a.counter + 5, a.n_records, a.nq,
              a.n_groups / kGroupsPerWindow, lane);
  unsigned long long bytes_read = 16ull * rows_read;
  for (int o = 16; o; o >>= 1) bytes_read += __shfl_down_sync(0xffffffffu, bytes_read, o);
  if (lane == 0 && touched) { atomicAdd(a.counter + 1, touched); atomicAdd(a.counter + 3, bytes_read); }
}

// ---------------------------------------------------------------- single-pattern content scan, small automaton
// k_body_sticky: the kAcc == 3 case of k_body when the whole byte-indexed table sits below shared address 64 Ki.
// The transition entries are rewritten in place, after staging, from "state index" to "shared address of that
// state's row", so one step is PRMT (byte extract) + IMAD (byte * 2 + row address) + LDS.U16: 3 issue slots per
// byte instead of 4, no second multiply on the dependent chain.  Rows that are full for all 32 lanes (all but the
// ragged tail of a group: the records of a group are length-sorted neighbours) run in a predicate-free loop, two
// rows per iteration with the loads for the next two already in flight.
__device__ __forceinline__ uint32_t sticky_step(uint32_t e, uint32_t b) {
  uint32_t addr;
  asm("mad.lo.u32 %0, %1, 2, %2;" : "=r"(addr) : "r"(b), "r"(e));
  uint16_t nxt;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(nxt) : "r"(addr));
  return nxt;
}
__device__ __forceinline__ uint32_t sticky_word(uint32_t e, uint32_t w) {
  e = sticky_step(e, __byte_perm(w, 0, 0x4440)); e = sticky_step(e, __byte_perm(w, 0, 0x4441));
  e = sticky_step(e, __byte_perm(w, 0, 0x4442)); return sticky_step(e, __byte_perm(w, 0, 0x4443));
}
__device__ __forceinline__ uint32_t sticky_row(uint32_t e, const uint4& v) {
  return sticky_word(sticky_word(sticky_word(sticky_word(e, v.x), v.y), v.z), v.w);
}
__device__ __forceinline__ uint32_t sticky_partial(uint32_t e, uint32_t w, int nbytes) {
#pragma unroll
  for (int j = 0; j < 4; ++j) if (j < nbytes) e = sticky_step(e, (w >> (8 * j)) & 0xFFu);
  return e;
}

constexpr int kStages = 2, kChunkRows = 2;        // per warp: 2 stages, each 2 rows (1 KiB) of each of two groups
constexpr uint32_t kChunkBytes = kChunkRows * 512u;
constexpr uint32_t kStageBytes = 2 * kChunkBytes;
constexpr uint32_t kWarpRingBytes = kStages * kStageBytes;
constexpr uint32_t kStickyRingBytes = (kWarpRingBytes + kStages * 8u) * (kBodyThreads / 32);
__device__ __forceinline__ uint4 lds128(uint32_t addr_s) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr_s));
  return r;
}
constexpr unsigned long long kGatherDiv = 16;       // k_body_gather takes over when at most 1 record in 16 is still alive
constexpr uint32_t kStickyAddrLimit = 65535u;
constexpr uint32_t kStickyAddrSlack = 4096u;     // head-room the host leaves for the shared-memory window base

// Rewrite the staged transitions at smem (shared address trans_s) in place from state index to row address
// (trans_s + state * stride2), for k_body_sticky and k_body_gather.
__device__ __forceinline__ void rows_to_addresses(uint8_t* smem, const fei_prog_dfa* dd, uint32_t trans_s, uint32_t stride2) {
  if (trans_s + dd->n_states * stride2 > kStickyAddrLimit) __trap();      // host-side eligibility test left 4 KiB of slack
  uint16_t* t = reinterpret_cast<uint16_t*>(smem);
  const uint32_t n_entries = dd->n_states * dd->row_stride;
  for (uint32_t i = threadIdx.x; i < n_entries; i += kBodyThreads) t[i] = (uint16_t)(trans_s + (uint32_t)t[i] * stride2);
  __syncthreads();
}

template <bool kPush>
__global__ void __launch_bounds__(kBodyThreads, 1) k_body_sticky(BodyArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  if (a.gather_max && a.counter[4] <= a.gather_max) return;    // few live records: k_body_gather has them (uniform for the grid)
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const fei_prog_dfa* dd = reinterpret_cast<const fei_prog_dfa*>(a.prog + ph->off_body_dfa);
  const uint32_t table_bytes = dd->table_bytes;
  stage_table(smem, a.prog + dd->off_trans, table_bytes, &bar);
  const uint32_t trans_s = smem_u32(smem), stride2 = dd->row_stride * 2u;
  // per-warp ring + its mbarriers, behind the table
  const uint32_t warp = threadIdx.x >> 5;
  uint8_t* ring = smem + ((table_bytes + 127u) & ~127u) + warp * kWarpRingBytes;
  const uint32_t ring_s = smem_u32(ring);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ((table_bytes + 127u) & ~127u) + (kBodyThreads / 32) * kWarpRingBytes) + warp * kStages;
  if ((threadIdx.x & 31) < kStages) mbar_init(&bars[threadIdx.x & 31], 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  uint32_t prod = 0, cons = 0;                       // chunks issued / consumed by this warp since kernel start (stage = count % kStages)
  rows_to_addresses(smem, dd, trans_s, stride2);
  const uint32_t* endout = reinterpret_cast<const uint32_t*>(smem + (dd->off_endout - dd->off_trans));
  const uint32_t start_e = trans_s + dd->start * stride2;
  const uint32_t sticky_e = dd->sticky != 0xFFFFFFFFu ? trans_s + (dd->sticky - 1u) * stride2 : 0xFFFFFFFFu;
  const fei_prog_cond* conds = reinterpret_cast<const fei_prog_cond*>(a.prog + ph->off_conds);
  const fei_prog_query* queries = reinterpret_cast<const fei_prog_query*>(a.prog + ph->off_queries);
  const uint32_t nq = ph->n_queries;
  const uint32_t all_q = nq >= 32 ? 0xFFFFFFFFu : ((1u << nq) - 1u);
  const int lane = threadIdx.x & 31;
  unsigned long long touched = 0, bytes_read = 0;

  // One group of 32 records as this warp sees it.
  struct Grp {
    uint32_t rec, len, alive, maxu, full, k, e;
    bool live;
    const uint8_t* row;          // next unread row
  };
  auto open_group = [&](unsigned long long g, Grp& G) {
    G.rec = kInvalidRec; G.len = 0; G.alive = 0; G.maxu = 0; G.full = 0; G.k = 0; G.e = start_e; G.live = false; G.row = a.tiles;
    if (g >= a.n_groups) return;
    G.rec = a.grp_rec[g * 32 + lane];
    G.len = a.grp_len[g * 32 + lane];
    if (G.rec != kInvalidRec) G.alive = a.has_alive ? a.hits[G.rec] : all_q;
    G.live = G.alive != 0;
    const uint32_t live_mask = __ballot_sync(0xffffffffu, G.live);
    if (live_mask == 0) return;                                     // nobody in this group can still match: skip its bytes
    G.row = a.tiles + a.grp_base[g] * 16;
    G.maxu = __shfl_sync(0xffffffffu, (G.len + 15) >> 4, 0);
    // rows that are 16 full bytes for all 32 lanes form one contiguous run of 512-byte rows.  Lanes a header predicate
    // already rejected ride along in the absorbing state (they read zeros, never hold up the early stop, write nothing):
    // a half-alive group keeps the streaming path instead of falling back to the row-by-row loop.
    const uint32_t valid_mask = __ballot_sync(0xffffffffu, G.rec != kInvalidRec);
    G.full = valid_mask == 0xffffffffu ? __reduce_min_sync(0xffffffffu, G.len >> 4) : 0u;
    if (!G.live && sticky_e != 0xFFFFFFFFu) G.e = sticky_e;
    if (lane == 0) touched += (a.grp_base[g + 1] - a.grp_base[g]) * 16;
  };
  // Full rows of ONE group through the ring: kChunkRows rows per bulk copy, kStages copies in flight; a stage is refilled
  // as soon as its rows sit in registers.
  auto stream_single = [&](Grp& G) {
    if (G.k >= G.full) return;
    const uint32_t n_chunks = (G.full - G.k) / kChunkRows;
    if (!n_chunks) return;
    uint32_t issued = 0, c = 0;
    for (; issued < n_chunks && issued < (uint32_t)kStages; ++issued, ++prod)
      if (lane == 0) { mbar_expect_tx(&bars[prod % kStages], kChunkBytes); bulk_g2s(ring + (prod % kStages) * kStageBytes, G.row + (uint64_t)issued * kChunkBytes, kChunkBytes, &bars[prod % kStages]); }
    bool stop = false;
    for (; c < n_chunks && !stop; ++c) {
      const uint32_t st = cons % kStages;
      mbar_wait(&bars[st], (cons / kStages) & 1u);
      ++cons;
      uint4 v[kChunkRows];
#pragma unroll
      for (int r = 0; r < kChunkRows; ++r) v[r] = lds128(ring_s + st * kStageBytes + r * 512u + lane * 16u);
      if (G.e == sticky_e) {                         // matched lanes all look up the same word (a broadcast) from here on
#pragma unroll
        for (int r = 0; r < kChunkRows; ++r) v[r] = make_uint4(0, 0, 0, 0);
      }
      __syncwarp();                                  // every lane holds its rows: the stage may be overwritten
      if (issued < n_chunks) {
        if (lane == 0) { mbar_expect_tx(&bars[st], kChunkBytes); bulk_g2s(ring + st * kStageBytes, G.row + (uint64_t)issued * kChunkBytes, kChunkBytes, &bars[st]); }
        ++issued; ++prod;
      }
#pragma unroll
      for (int r = 0; r < kChunkRows; ++r) G.e = sticky_row(G.e, v[r]);
      stop = __ballot_sync(0xffffffffu, G.e != sticky_e) == 0;      // every lane has matched
    }
    for (; cons < prod; ++cons) mbar_wait(&bars[cons % kStages], (cons / kStages) & 1u);   // early stop: let the copies in flight land
    bytes_read += (unsigned long long)issued * kChunkBytes;
    G.row += (uint64_t)c * kChunkBytes;
    G.k = stop ? G.maxu : G.k + c * kChunkRows;
  };
  // The same for TWO groups in lock step: each lane runs two independent automaton chains, so the shared-memory
  // latency of one lookup is covered by the other chain's (the single chain is LDS-latency bound: 8 warps per scheduler).
  auto stream_pair = [&](Grp& A, Grp& B) {
    const uint32_t n_chunks = (A.full < B.full ? A.full : B.full) / kChunkRows;
    if (!n_chunks) return;
    uint32_t issued = 0, c = 0;
    auto issue = [&](uint32_t st) {
      if (lane == 0) {
        mbar_expect_tx(&bars[st], 2 * kChunkBytes);
        bulk_g2s(ring + st * kStageBytes, A.row + (uint64_t)issued * kChunkBytes, kChunkBytes, &bars[st]);
        bulk_g2s(ring + st * kStageBytes + kChunkBytes, B.row + (uint64_t)issued * kChunkBytes, kChunkBytes, &bars[st]);
      }
      ++issued; ++prod;
    };
    while (issued < n_chunks && issued < (uint32_t)kStages) issue(prod % kStages);
    bool stop_a = false, stop_b = false;
    for (; c < n_chunks && !stop_a && !stop_b; ++c) {
      const uint32_t st = cons % kStages;
      mbar_wait(&bars[st], (cons / kStages) & 1u);
      ++cons;
      uint4 va[kChunkRows], vb[kChunkRows];
#pragma unroll
      for (int r = 0; r < kChunkRows; ++r) {
        va[r] = lds128(ring_s + st * kStageBytes + r * 512u + lane * 16u);
        vb[r] = lds128(ring_s + st * kStageBytes + kChunkBytes + r * 512u + lane * 16u);
      }
      uint32_t ea = A.e, eb = B.e;
      // a lane that has matched stays in the absorbing state whatever it reads: give it zeros, so that all matched
      // lanes look up one and the same word (a broadcast) instead of spreading over the banks of the absorbing row
      if (ea == sticky_e) {
#pragma unroll
        for (int r = 0; r < kChunkRows; ++r) va[r] = make_uint4(0, 0, 0, 0);
      }
      if (eb == sticky_e) {
#pragma unroll
        for (int r = 0; r < kChunkRows; ++r) vb[r] = make_uint4(0, 0, 0, 0);
      }
      __syncwarp();
      if (issued < n_chunks) issue(st);
#pragma unroll
      for (int r = 0; r < kChunkRows; ++r) {
        const uint32_t wa[4] = {va[r].x, va[r].y, va[r].z, va[r].w}, wb[4] = {vb[r].x, vb[r].y, vb[r].z, vb[r].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          ea = sticky_step(ea, __byte_perm(wa[j], 0, 0x4440)); eb = sticky_step(eb, __byte_perm(wb[j], 0, 0x4440));
          ea = sticky_step(ea, __byte_perm(wa[j], 0, 0x4441)); eb = sticky_step(eb, __byte_perm(wb[j], 0, 0x4441));
          ea = sticky_step(ea, __byte_perm(wa[j], 0, 0x4442)); eb = sticky_step(eb, __byte_perm(wb[j], 0, 0x4442));
          ea = sticky_step(ea, __byte_perm(wa[j], 0, 0x4443)); eb = sticky_step(eb, __byte_perm(wb[j], 0, 0x4443));
        }
      }
      A.e = ea; B.e = eb;
      stop_a = __ballot_sync(0xffffffffu, ea != sticky_e) == 0;
      stop_b = __ballot_sync(0xffffffffu, eb != sticky_e) == 0;
    }
    for (; cons < prod; ++cons) mbar_wait(&bars[cons % kStages], (cons / kStages) & 1u);
    bytes_read += 2ull * issued * kChunkBytes;
    A.row += (uint64_t)c * kChunkBytes; B.row += (uint64_t)c * kChunkBytes;
    A.k = stop_a ? A.maxu : c * kChunkRows;
    B.k = stop_b ? B.maxu : c * kChunkRows;
  };
  // Ragged remainder of both groups (and groups with dead lanes), still two chains per lane: row k of a group holds
  // only the lanes that have a unit k (lane count from a ballot), every lane steps through all 16 bytes and keeps
  // the new state only for the bytes its record really has (nb), so there is no divergent branch between the chains.
  auto ragged_pair = [&](Grp& A, Grp& B) {
    const uint32_t rem_a = A.maxu - A.k, rem_b = B.maxu - B.k;       // k <= maxu always
    const uint32_t rounds = rem_a > rem_b ? rem_a : rem_b;
    if (!rounds) return;
    const uint32_t units_a = (A.len + 15) >> 4, units_b = (B.len + 15) >> 4;
    bool act_a = A.live && rem_a, act_b = B.live && rem_b;
    const uint8_t* row_a = A.row; const uint8_t* row_b = B.row;
    uint32_t ea = A.e, eb = B.e;
    uint4 cur_a = make_uint4(0, 0, 0, 0), cur_b = cur_a;
    if (act_a && A.k < units_a) cur_a = ldg_stream16(row_a + lane * 16);
    if (act_b && B.k < units_b) cur_b = ldg_stream16(row_b + lane * 16);
    for (uint32_t i = 0; i < rounds; ++i) {
      const uint32_t ka = A.k + i, kb = B.k + i;
      bytes_read += __popc(__ballot_sync(0xffffffffu, act_a && ka < units_a)) * 16 + __popc(__ballot_sync(0xffffffffu, act_b && kb < units_b)) * 16;
      row_a += (uint64_t)__popc(__ballot_sync(0xffffffffu, ka < units_a)) * 16;
      row_b += (uint64_t)__popc(__ballot_sync(0xffffffffu, kb < units_b)) * 16;
      uint4 nxt_a = make_uint4(0, 0, 0, 0), nxt_b = nxt_a;
      if (act_a && ka + 1 < units_a) nxt_a = ldg_stream16(row_a + lane * 16);
      if (act_b && kb + 1 < units_b) nxt_b = ldg_stream16(row_b + lane * 16);
      int nba = act_a ? (int)A.len - (int)(ka * 16) : 0, nbb = act_b ? (int)B.len - (int)(kb * 16) : 0;   // <= 0: no byte of this row
      const uint32_t wa[4] = {cur_a.x, cur_a.y, cur_a.z, cur_a.w}, wb[4] = {cur_b.x, cur_b.y, cur_b.z, cur_b.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t ta = sticky_step(ea, __byte_perm(wa[j], 0, 0x4440 + q)), tb = sticky_step(eb, __byte_perm(wb[j], 0, 0x4440 + q));
          ea = 4 * j + q < nba ? ta : ea;
          eb = 4 * j + q < nbb ? tb : eb;
        }
      }
      cur_a = nxt_a; cur_b = nxt_b;
      // a group is finished as soon as every live lane has either matched or ended
      if (__ballot_sync(0xffffffffu, act_a && ka + 1 < units_a && ea != sticky_e) == 0) act_a = false;
      if (__ballot_sync(0xffffffffu, act_b && kb + 1 < units_b && eb != sticky_e) == 0) act_b = false;
      if (__ballot_sync(0xffffffffu, act_a || act_b) == 0) break;
    }
    A.e = ea; B.e = eb;
  };
  auto close_group = [&](const Grp& G) {
    if (G.live) {
      a.hits[G.rec] = content_hits(endout[(G.e - trans_s) / stride2], G.alive, queries, conds, nq);
    } else if (G.rec != kInvalidRec && !a.has_alive) {
      a.hits[G.rec] = 0;
    }
  };

  for (;;) {
    unsigned long long g = 0;
    if (lane == 0) g = atomicAdd(a.next, 2ull);
    g = __shfl_sync(0xffffffffu, g, 0);
    if (g >= a.n_groups) break;
    Grp A, B;
    open_group(g, A);
    open_group(g + 1, B);
    stream_pair(A, B);
    stream_single(A);
    stream_single(B);
    ragged_pair(A, B);
    close_group(A);
    close_group(B);
    signal_group_done<kPush, false>(a, g, 0u, lane);
    if (g + 1 < a.n_groups) signal_group_done<kPush, false>(a, g + 1, 0u, lane);
  }
  if (lane == 0 && touched) { atomicAdd(a.counter + 1, touched); atomicAdd(a.counter + 3, bytes_read); }
}

// ---------------------------------------------------------------- single-pattern scan of FEW surviving records
// After selective header predicates a group of 32 has at most a lane or two left alive; k_body_sticky then runs one
// serial automaton chain per group and the SM idles at 64 chains (the latency floor of that shape).  k_live_list compacts the survivors and k_body_gather gives every one its own
// thread: a lane walks its record through the tiles of its group (row k of a group starts 16 * sum_{j<k} m_j after the
// group base, m_j = lanes that still have a unit j, recovered from the group's sorted lengths), so a warp runs 32 chains.
__global__ void __launch_bounds__(256) k_live_list(const uint32_t* __restrict__ alive, uint64_t n, uint32_t* __restrict__ list,
                                                  unsigned long long* __restrict__ count, unsigned long long cap) {
  __shared__ unsigned int cta_count; __shared__ unsigned long long cta_base;
  if (threadIdx.x == 0) cta_count = 0;
  __syncthreads();
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const bool live = i < n && alive[i] != 0;
  const uint32_t bal = __ballot_sync(0xffffffffu, live);
  const int lane = threadIdx.x & 31;
  unsigned int wbase = 0;
  if (lane == 0 && bal) wbase = atomicAdd(&cta_count, (unsigned int)__popc(bal));
  wbase = __shfl_sync(0xffffffffu, wbase, 0);
  __syncthreads();
  if (threadIdx.x == 0 && cta_count) cta_base = atomicAdd(count, (unsigned long long)cta_count);
  __syncthreads();
  if (live) { const unsigned long long at = cta_base + wbase + __popc(bal & ((1u << lane) - 1u)); if (at < cap) list[at] = (uint32_t)i; }
}

__global__ void __launch_bounds__(kBodyThreads, 1) k_body_gather(BodyArgs a, const uint32_t* __restrict__ live, const uint32_t* __restrict__ rec_pos) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  const unsigned long long n_live = a.counter[4];
  if (n_live == 0 || n_live > a.gather_max) return;            // k_body_sticky takes the dense case (uniform for the grid)
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const fei_prog_dfa* dd = reinterpret_cast<const fei_prog_dfa*>(a.prog + ph->off_body_dfa);
  stage_table(smem, a.prog + dd->off_trans, dd->table_bytes, &bar);
  const uint32_t trans_s = smem_u32(smem), stride2 = dd->row_stride * 2u;
  rows_to_addresses(smem, dd, trans_s, stride2);
  const uint32_t* endout = reinterpret_cast<const uint32_t*>(smem + (dd->off_endout - dd->off_trans));
  const uint32_t start_e = trans_s + dd->start * stride2;
  const uint32_t sticky_e = dd->sticky != 0xFFFFFFFFu ? trans_s + (dd->sticky - 1u) * stride2 : 0xFFFFFFFFu;
  const fei_prog_cond* conds = reinterpret_cast<const fei_prog_cond*>(a.prog + ph->off_conds);
  const fei_prog_query* queries = reinterpret_cast<const fei_prog_query*>(a.prog + ph->off_queries);
  const uint32_t nq = ph->n_queries;
  unsigned long long bytes_read = 0;
  for (unsigned long long t = blockIdx.x * (unsigned long long)kBodyThreads + threadIdx.x; t < n_live; t += (unsigned long long)gridDim.x * kBodyThreads) {
    const uint32_t rec = live[t];
    const uint32_t pos = rec_pos[rec];
    const uint64_t g = pos >> 5; const uint32_t l = pos & 31u;
    const uint32_t* gl = a.grp_len + g * 32;
    const uint32_t len = gl[l];
    const uint32_t units = (len + 15) >> 4;
    const uint32_t alive = a.hits[rec];
    uint32_t m = 32;                                             // lanes of the group that have a unit k (lengths are sorted descending)
    uint32_t drop = (gl[31] + 15) >> 4;                          // the first row lane m-1 is missing from
    const uint8_t* p = a.tiles + a.grp_base[g] * 16 + l * 16;
    uint32_t e = start_e;
    for (uint32_t k = 0; k < units; ++k) {
      while (k >= drop) { --m; drop = m > l + 1 ? (gl[m - 1] + 15) >> 4 : 0xFFFFFFFFu; }
      const uint4 v = ldg_stream16(p);
      p += (uint64_t)m * 16;
      const int nb = (int)len - (int)(k * 16);
      if (nb >= 16) e = sticky_row(e, v);
      else { e = sticky_partial(e, v.x, nb); e = sticky_partial(e, v.y, nb - 4); e = sticky_partial(e, v.z, nb - 8); e = sticky_partial(e, v.w, nb - 12); }
      bytes_read += 16;
      if (e == sticky_e) break;                                  // matched: the verdict cannot change any more
    }
    a.hits[rec] = content_hits(endout[(e - trans_s) / stride2], alive, queries, conds, nq);
  }
  for (int o = 16; o; o >>= 1) bytes_read += __shfl_down_sync(0xffffffffu, bytes_read, o);
  if ((threadIdx.x & 31) == 0 && bytes_read) { atomicAdd(a.counter + 3, bytes_read); atomicAdd(a.counter + 1, bytes_read); }
}

// ---------------------------------------------------------------- content position automaton (bit-parallel NFA)
// k_body_nfa: content patterns whose DFA is too large (bounded gaps: `a.{0,60}b`) run as a position automaton
// (feiscan_prog.h fei_prog_nfa): per code point, a W-word bit vector of NFA positions steps through
//     D' = (((D << 1) & SHIFT) | (D & SELF) | OR_g [(D & src_g) && ctx ok] dst_g) & B[class]
// The group loop is k_body's (warps claim 32-record groups, one lane per record, 16-byte rows, groups with no live record
// skipped); each lane undoes the tile byte permutation, decodes UTF-8 and looks the class up (ASCII table, else a binary
// search over the range table).  A program that also has a body DFA (class-indexed, not sticky) steps it on every byte as
// k_body<false, 0> does; its outputs are the content bits below the automaton's first_bit.  The ordered lists are compacted
// after the scan and the multi-GPU hook copies the masks (no window work in the kernel).  kCtr: the automaton has counter
// positions (version-3 programs, feiscan_prog.h fei_prog_nfa_ctr); their positions, bounds and ages take 25 more registers, so
// those instances run 512 threads per CTA (128 registers) at every W.
template <int W, bool kCtr = false> struct NfaThreads { static constexpr int value = W <= 4 && !kCtr ? 1024 : 512; };

// Stage the body DFA's tables (bytes0, may be 0) and the position automaton's behind them with one mbarrier.
__device__ __forceinline__ void stage_two_tables(uint8_t* dst0, const uint8_t* src0, uint32_t bytes0, uint8_t* dst1, const uint8_t* src1,
                                                 uint32_t bytes1, uint64_t* bar) {
  if (threadIdx.x == 0) { mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, bytes0 + bytes1);
    for (uint32_t o = 0; o < bytes0; o += 32768u) bulk_g2s(dst0 + o, src0 + o, bytes0 - o < 32768u ? bytes0 - o : 32768u, bar);
    for (uint32_t o = 0; o < bytes1; o += 32768u) bulk_g2s(dst1 + o, src1 + o, bytes1 - o < 32768u ? bytes1 - o : 32768u, bar);
  }
  mbar_wait(bar, 0);
}

template <int W, bool kHasDfa, bool kCtr>
__global__ void __launch_bounds__(NfaThreads<W, kCtr>::value, 1) k_body_nfa(BodyArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  __shared__ uint32_t q_need[33];                  // as in k_body
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const fei_prog_nfa* nd = reinterpret_cast<const fei_prog_nfa*>(a.prog + ph->off_body_nfa);
  const fei_prog_dfa* dd = reinterpret_cast<const fei_prog_dfa*>(a.prog + ph->off_body_dfa);
  const fei_prog_cond* conds = reinterpret_cast<const fei_prog_cond*>(a.prog + ph->off_conds);
  const fei_prog_query* queries = reinterpret_cast<const fei_prog_query*>(a.prog + ph->off_queries);
  const uint32_t nq = ph->n_queries;
  if (threadIdx.x < 32) {
    uint32_t bits = 0;
    if (threadIdx.x < nq)
      for (uint32_t c = queries[threadIdx.x].cond_begin; c < queries[threadIdx.x].cond_end; ++c)
        if (conds[c].kind == FEI_C_BODY) bits |= 1u << conds[c].bit;
    q_need[threadIdx.x] = bits;
    bits = __reduce_or_sync(0xffffffffu, bits);
    if (threadIdx.x == 0) q_need[32] = bits;
  }
  const uint32_t dfa_bytes = kHasDfa ? dd->table_bytes : 0u;
  uint8_t* nsm = smem + dfa_bytes;                 // both table sizes are multiples of 16
  stage_two_tables(smem, kHasDfa ? a.prog + dd->off_trans : nullptr, dfa_bytes, nsm, a.prog + nd->off_ascii, nd->table_bytes, &bar);
  const NfaTables t(nd, nsm);
  BodyDfa<false, 0> d;
  const uint32_t* endout = nullptr;
  uint32_t dfa_start = 0;
  if constexpr (kHasDfa) {
    d.trans_s = smem_u32(smem);
    d.out = reinterpret_cast<const uint32_t*>(smem + (dd->off_out - dd->off_trans));
    d.cls = smem + (dd->off_cls - dd->off_trans);
    d.stride2 = dd->row_stride * 2u; d.n_acc = dd->n_acc; d.entry_bytes = c_entry_bytes;
    endout = reinterpret_cast<const uint32_t*>(smem + (dd->off_endout - dd->off_trans));
    dfa_start = dd->start;
  }
  Nfa<W, kCtr> nfa;
  if constexpr (kCtr) {                            // check_prog: the descriptor right behind the section, its table staged with it
    const fei_prog_nfa_ctr* cd = reinterpret_cast<const fei_prog_nfa_ctr*>(a.prog + ph->off_body_nfa + sizeof(fei_prog_nfa));
    nfa.load_counters(reinterpret_cast<const uint32_t*>(nsm + (cd->off_counters - nd->off_ascii)), cd->n_counters);
  }
  const uint32_t all_q = nq >= 32 ? 0xFFFFFFFFu : ((1u << nq) - 1u);
  const int lane = threadIdx.x & 31;
  unsigned long long touched = 0;
  uint32_t rows_read = 0;
  for (;;) {
    unsigned long long g = 0;
    if (lane == 0) g = atomicAdd(a.next, 1ull);
    g = __shfl_sync(0xffffffffu, g, 0);
    if (g >= a.n_groups) break;
    const uint32_t rec = a.grp_rec[g * 32 + lane];
    const uint32_t len = a.grp_len[g * 32 + lane];
    const uint32_t units = (len + 15) >> 4;
    uint32_t alive = 0;
    if (rec != kInvalidRec) alive = a.has_alive ? a.hits[rec] : all_q;
    const bool live = alive != 0;
    if (__ballot_sync(0xffffffffu, live) == 0) {              // nobody in this group can still match: skip its bytes
      if (rec != kInvalidRec && !a.has_alive) a.hits[rec] = 0;
      continue;
    }
    const uint8_t* row = a.tiles + a.grp_base[g] * 16;
    const uint32_t maxu = __shfl_sync(0xffffffffu, units, 0);
    if (lane == 0) touched += (a.grp_base[g + 1] - a.grp_base[g]) * 16;
    nfa.reset(t);
    if constexpr (kHasDfa) d.reset(dfa_start);
    // the content bits this lane's alive queries read; the lane stops once the accepts met so far set all of them (bits that
    // only end-only accepts or the DFA's endout[] set keep it reading to the end)
    uint32_t need = 0;
    if (live) {
      need = q_need[32];
      if (alive != all_q) {
        need = 0;
        for (uint32_t q = alive; q; q &= q - 1) need |= q_need[__ffs(q) - 1];
      }
    }
    auto decided = [&]() { return (need & ~(nfa.acc | (kHasDfa ? d.a0 : 0u))) == 0; };
    uint32_t lim = live && !decided() ? units : 0;
    uint4 cur = make_uint4(0, 0, 0, 0);
    if (0 < lim) { cur = ldg_stream16(row + lane * 16); ++rows_read; }
    for (uint32_t k = 0; k < maxu; ++k) {
      const uint32_t m = __popc(__ballot_sync(0xffffffffu, k < units));
      const uint8_t* next_row = row + (uint64_t)m * 16;
      uint4 nxt = make_uint4(0, 0, 0, 0);
      if (k + 1 < lim) { nxt = ldg_stream16(next_row + lane * 16); ++rows_read; }
      if (k < lim) {
        const uint32_t nb = len - k * 16 < 16u ? len - k * 16 : 16u;
        uint4 v = cur;
#pragma unroll 1
        for (uint32_t j = 0; j < nb; ++j) {                    // byte j of the row is the low byte of v.x
          const uint32_t b = v.x & 0xFFu;
          v.x = __funnelshift_r(v.x, v.y, 8); v.y = __funnelshift_r(v.y, v.z, 8); v.z = __funnelshift_r(v.z, v.w, 8); v.w >>= 8;
          if constexpr (kHasDfa) d.step(b);
          nfa.byte(t, tile_byte_unperm((uint8_t)b));
        }
      }
      cur = nxt; row = next_row;
      if (k + 1 < lim && decided()) lim = k + 1;               // row k + 1, already in flight, is dropped
      if (__ballot_sync(0xffffffffu, k + 1 < lim) == 0) break;
    }
    if (live) {
      uint32_t acc = nfa.finish(t);
      if constexpr (kHasDfa) acc |= d.finish(endout);
      a.hits[rec] = content_hits(acc, alive, queries, conds, nq);
    } else if (rec != kInvalidRec && !a.has_alive) {
      a.hits[rec] = 0;
    }
  }
  unsigned long long bytes_read = 16ull * rows_read;
  for (int o = 16; o; o >>= 1) bytes_read += __shfl_down_sync(0xffffffffu, bytes_read, o);
  if (lane == 0 && touched) { atomicAdd(a.counter + 1, touched); atomicAdd(a.counter + 3, bytes_read); }
}

using BodyKernel = void (*)(BodyArgs);
// The k_body_nfa instance for a content automaton of `words` words (check_prog: 1, 2, 4 or 8) and its block size.
struct BodyNfaKernel { BodyKernel k; int threads; };
template <int W, bool kHasDfa, bool kCtr> constexpr BodyNfaKernel body_nfa_of() { return {k_body_nfa<W, kHasDfa, kCtr>, NfaThreads<W, kCtr>::value}; }
static BodyNfaKernel body_nfa_kernel(uint32_t words, bool has_dfa, bool counters) {
  static const BodyNfaKernel of[2][2][4] = {          // [counters][has_dfa][log2 words]
      {{body_nfa_of<1, false, false>(), body_nfa_of<2, false, false>(), body_nfa_of<4, false, false>(), body_nfa_of<8, false, false>()},
       {body_nfa_of<1, true, false>(), body_nfa_of<2, true, false>(), body_nfa_of<4, true, false>(), body_nfa_of<8, true, false>()}},
      {{body_nfa_of<1, false, true>(), body_nfa_of<2, false, true>(), body_nfa_of<4, false, true>(), body_nfa_of<8, false, true>()},
       {body_nfa_of<1, true, true>(), body_nfa_of<2, true, true>(), body_nfa_of<4, true, true>(), body_nfa_of<8, true, true>()}}};
  return of[counters][has_dfa][__builtin_ctz(words)];
}

// The content kernel of one scan: k_body_sticky when the sticky automaton's row addresses fit 16 bits, else the k_body
// instance for the table's column mapping and accumulator mode.
static BodyKernel body_kernel(bool sticky, bool direct, int acc_mode, bool push) {
  static const BodyKernel k_body_of[2][2][4] = {      // [push][direct][acc_mode]
      {{k_body<false, 0, false>, k_body<false, 1, false>, k_body<false, 2, false>, k_body<false, 3, false>},
       {k_body<true, 0, false>, k_body<true, 1, false>, k_body<true, 2, false>, k_body<true, 3, false>}},
      {{k_body<false, 0, true>, k_body<false, 1, true>, k_body<false, 2, true>, k_body<false, 3, true>},
       {k_body<true, 0, true>, k_body<true, 1, true>, k_body<true, 2, true>, k_body<true, 3, true>}}};
  if (sticky) return push ? k_body_sticky<true> : k_body_sticky<false>;
  return k_body_of[push][direct][acc_mode];
}

template <typename Kernel, typename... Args>
static int launch_body(Kernel k, int threads, unsigned grid, size_t smem, cudaStream_t s, Args... args) {
  FEI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k<<<grid, threads, smem, s>>>(args...);
  return FEI_OK;
}

// ---------------------------------------------------------------- compaction
constexpr int kCompactBlock = 256;          // threads
constexpr int kCompactPer = 8;              // records per thread -> 2048 records per block
constexpr uint64_t kCompactRecs = (uint64_t)kCompactBlock * kCompactPer;

// counts[block * nq + q] = records of this block that hit query q
__global__ void __launch_bounds__(kCompactBlock)
k_count(const uint32_t* __restrict__ hits, uint64_t n, uint32_t nq, uint32_t* __restrict__ counts) {
  __shared__ uint32_t sh[32][8];
  const uint64_t blk = blockIdx.x;
  uint64_t base = blk * kCompactRecs;
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t cnt = 0;                        // lane q accumulates query q
  for (int r = 0; r < kCompactPer; ++r) {
    uint64_t i = base + (uint64_t)(warp * kCompactPer + r) * 32 + lane;
    cnt += count_hits32(i < n ? hits[i] : 0u, nq, lane);
  }
  sh[lane][warp] = cnt;
  __syncthreads();
  if (threadIdx.x < 32 && threadIdx.x < nq) {
    uint32_t s = 0;
    for (int w = 0; w < 8; ++w) s += sh[threadIdx.x][w];
    counts[blk * nq + threadIdx.x] = s;
  }
}

// per query: exclusive scan over the blocks [0, nblocks) (one thread block per query), continuing from carry[q] (the hits
// of the segments compacted before this one) and leaving the new running total there
__global__ void k_scan_blocks(const uint32_t* __restrict__ counts, uint64_t nblocks, uint32_t nq,
                              uint64_t* __restrict__ offsets, uint64_t* __restrict__ carry_io) {
  __shared__ uint64_t sh[1024];
  __shared__ uint64_t carry;
  uint32_t q = blockIdx.x;
  if (threadIdx.x == 0) carry = carry_io[q];
  __syncthreads();
  for (uint64_t base = 0; base < nblocks; base += blockDim.x) {
    uint64_t b = base + threadIdx.x;
    uint64_t v = b < nblocks ? counts[b * nq + q] : 0;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < blockDim.x; o <<= 1) {
      uint64_t t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    uint64_t incl = sh[threadIdx.x];
    if (b < nblocks) offsets[b * nq + q] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry += incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) carry_io[q] = carry;
}

// ordered emit: lists[q * stride + rank] = base + i -- corpus-local 32-bit indices (base 0) for a corpus' own lists, 64-bit
// global ones for the lists built from gathered rank segments (comm.cu)
// (a resident scan CTA of k_body holds the whole register file, so these kernels run between scans, not under one)
template <class T>
__global__ void __launch_bounds__(kCompactBlock, 8)
k_emit(const uint32_t* __restrict__ hits, uint64_t n, uint32_t nq, const uint64_t* __restrict__ offsets,
       T base, uint64_t stride, T* __restrict__ lists) {
  __shared__ uint32_t wcnt[8][32];          // [warp][query] hits of this warp's records
  const uint64_t blk = blockIdx.x;
  const uint64_t first = blk * kCompactRecs;
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t m[kCompactPer];
  uint32_t cnt = 0;
  for (int r = 0; r < kCompactPer; ++r) {
    uint64_t i = first + (uint64_t)(warp * kCompactPer + r) * 32 + lane;
    m[r] = i < n ? hits[i] : 0u;
    cnt += count_hits32(m[r], nq, lane);
  }
  wcnt[warp][lane] = cnt;
  __syncthreads();
  for (uint32_t q = 0; q < nq; ++q) {
    uint64_t pos = offsets[blk * nq + q];
    for (int w = 0; w < warp; ++w) pos += wcnt[w][q];
    T* list = lists + q * stride;
    for (int r = 0; r < kCompactPer; ++r)
      pos += emit_hits32<T>((m[r] >> q) & 1u, list + pos, base + (T)(first + (uint64_t)(warp * kCompactPer + r) * 32 + lane), lane);
  }
}

// Ordered lists of the n masks at `masks` (record 0 is index `base`) into lists[q * stride + rank], the ranks continuing
// from sc.totals, which is left holding the running per-query totals.  n > 0.
template <class T>
static void compact_lists(const uint32_t* masks, uint64_t n, uint32_t nq, T base, CompactScratch& sc, uint64_t stride,
                          T* lists, cudaStream_t s) {
  const uint64_t nb = (n + kCompactRecs - 1) / kCompactRecs;
  k_count<<<(unsigned)nb, kCompactBlock, 0, s>>>(masks, n, nq, sc.blk_counts.as<uint32_t>());
  k_scan_blocks<<<nq, 256, 0, s>>>(sc.blk_counts.as<uint32_t>(), nb, nq, sc.blk_offsets.as<uint64_t>(), sc.totals.as<uint64_t>());
  k_emit<T><<<(unsigned)nb, kCompactBlock, 0, s>>>(masks, n, nq, sc.blk_offsets.as<uint64_t>(), base, stride, lists);
}

// dst[i] = base + src[i]: corpus-local list entries as global indices
__global__ void k_widen(const uint32_t* __restrict__ src, uint64_t n, uint64_t base, uint64_t* __restrict__ dst) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) dst[i] = base + src[i];
}

__global__ void k_fill32(uint32_t* __restrict__ p, uint64_t n, uint32_t v) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// Order-sensitive checksum of an index list (entry k is index base + v[k]): sum_k (k + 1) * index_k and sum_k index_k
// (mod 2^64).  Two lists agree on both sums iff (with overwhelming probability) they hold the same indices in the same order;
// the pair (A, S) of the concatenation of two lists follows from the parts: A = A1 + A2 + len1 * S2.
template <class T>
__global__ void __launch_bounds__(256) k_list_checksum(const T* __restrict__ v, uint64_t n, unsigned long long base, unsigned long long* __restrict__ out) {
  unsigned long long a = 0, s = 0;
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long x = base + v[k];
    a += (k + 1) * x; s += x;
  }
  for (int o = 16; o; o >>= 1) { a += __shfl_down_sync(0xffffffffu, a, o); s += __shfl_down_sync(0xffffffffu, s, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(out, a); atomicAdd(out + 1, s); }
}

// ---------------------------------------------------------------- host side
static int check_prog(const uint8_t* prog, uint64_t len) {
  if (!prog || len < sizeof(fei_prog_hdr)) { set_error("program blob too small"); return FEI_E_BADARG; }
  fei_prog_hdr h; memcpy(&h, prog, sizeof(h));
  if (h.magic != FEI_PROG_MAGIC || (h.version != FEI_PROG_VERSION && h.version != FEI_PROG_VERSION_NFA && h.version != FEI_PROG_VERSION_CTR)) { set_error("bad program magic/version"); return FEI_E_BADARG; }
  if (h.total_bytes != len) { set_error("program length mismatch (%u vs %llu)", h.total_bytes, (unsigned long long)len); return FEI_E_BADARG; }
  if (h.n_queries == 0 || h.n_queries > FEI_MAX_QUERIES) { set_error("1..32 queries per program"); return FEI_E_BADARG; }
  if (h.n_slots > FEI_MAX_SLOTS) { set_error("at most %d header slots per program", FEI_MAX_SLOTS); return FEI_E_UNSUPPORTED; }
  if (h.head_bytes > h.total_bytes || (h.head_bytes & 15u)) { set_error("bad head_bytes in program"); return FEI_E_BADARG; }
  auto in = [&](uint64_t off, uint64_t sz) { return off % 16 == 0 && off + sz <= len; };
  if (!in(h.off_conds, (uint64_t)h.n_conds * sizeof(fei_prog_cond)) || !in(h.off_queries, (uint64_t)h.n_queries * sizeof(fei_prog_query)) ||
      !in(h.off_slots, (uint64_t)h.n_slots * sizeof(fei_prog_slot))) { set_error("program section out of bounds"); return FEI_E_BADARG; }
  auto dfa_ok = [&](uint32_t off) {
    if (!off) return true;
    if (!in(off, sizeof(fei_prog_dfa))) return false;
    fei_prog_dfa d; memcpy(&d, prog + off, sizeof(d));
    return in(d.off_trans, d.table_bytes) && d.start < d.n_states && d.n_cols >= 1 && d.n_cols <= 256 &&
           d.off_out >= d.off_trans && d.off_endout >= d.off_trans && d.off_cls >= d.off_trans &&
           d.off_out + 4ull * d.n_states <= (uint64_t)d.off_trans + d.table_bytes &&
           d.off_endout + 4ull * d.n_states <= (uint64_t)d.off_trans + d.table_bytes &&
           d.row_stride >= d.n_cols && 2ull * d.n_states * d.row_stride <= d.trans_bytes && d.n_states <= 65535;
  };
  if (!dfa_ok(h.off_key_dfa) || !dfa_ok(h.off_body_dfa) || !dfa_ok(h.off_flags_dfa) || !dfa_ok(h.off_name_dfa[0]) ||
      !dfa_ok(h.off_name_dfa[1]) || !dfa_ok(h.off_name_dfa[2]) || !dfa_ok(h.off_meta_dfa[0]) || !dfa_ok(h.off_meta_dfa[1])) { set_error("bad DFA descriptor in program"); return FEI_E_BADARG; }
  // A position automaton section (0 = none): every table inside its table_bytes; a head one inside [0, head_bytes) when the head
  // kernels stage the head.  Counters: version 3 if and only if the content automaton has a fei_prog_nfa_ctr right behind its
  // descriptor (the head ones never have one), with its table among the section's; ctr_ok says whether it is well-formed.
  uint32_t n_nfa = 0;
  bool ctr_ok = h.version != FEI_PROG_VERSION_CTR;
  auto nfa_ok = [&](uint32_t off, bool content) {
    if (!off) return true;
    ++n_nfa;
    if (!in(off, sizeof(fei_prog_nfa))) return false;
    fei_prog_nfa a; memcpy(&a, prog + off, sizeof(a));
    const uint64_t W = a.n_words, end = (uint64_t)a.off_ascii + a.table_bytes;
    auto tab = [&](uint64_t o, uint64_t sz) { return o % 16 == 0 && o >= a.off_ascii && o + sz <= end; };
    bool ok = (W == 1 || W == 2 || W == 4 || W == 8) && a.n_pos >= 1 && a.n_pos <= 32 * W && a.n_classes >= 1 &&
              a.n_classes <= FEI_NFA_MAX_CLASSES && a.n_ranges >= 1 && a.n_ranges <= FEI_NFA_MAX_RANGES &&
              a.n_follow <= FEI_NFA_MAX_GROUPS && a.n_accept <= FEI_NFA_MAX_GROUPS && a.first_bit + (uint64_t)a.n_patterns <= 32 &&
              a.table_bytes % 16 == 0 && in(a.off_ascii, a.table_bytes) && tab(a.off_ascii, 2 * 128) &&
              tab(a.off_range_lo, 4ull * a.n_ranges) && tab(a.off_range_ck, 2ull * a.n_ranges) && tab(a.off_cls_b, 4ull * W * a.n_classes) &&
              tab(a.off_masks, 12ull * W) && tab(a.off_follow, 4ull * (2 * W + 1) * a.n_follow) && tab(a.off_accept, 4ull * (W + 2) * a.n_accept) &&
              (content || !h.head_bytes || (off + sizeof(fei_prog_nfa) <= h.head_bytes && end <= h.head_bytes));
    if (ok) {                                      // class ids index cls_b, kinds are 0..4, the range table starts at 0x80
      const uint16_t* asc = reinterpret_cast<const uint16_t*>(prog + a.off_ascii);
      const uint16_t* rck = reinterpret_cast<const uint16_t*>(prog + a.off_range_ck);
      const uint32_t* rlo = reinterpret_cast<const uint32_t*>(prog + a.off_range_lo);
      auto ck_ok = [&](uint16_t v) { return (v & 0xFFu) < a.n_classes && (v >> 8) < 5; };
      for (int c = 0; c < 128 && ok; ++c) ok = ck_ok(asc[c]);
      for (uint32_t r = 0; r < a.n_ranges && ok; ++r) ok = ck_ok(rck[r]) && (r ? rlo[r] > rlo[r - 1] : rlo[0] == 0x80u);
      const uint32_t* acc = reinterpret_cast<const uint32_t*>(prog + a.off_accept);
      for (uint32_t g = 0; g < a.n_accept && ok; ++g) ok = (acc[g * (W + 2) + W + 1] & 0xFFu) < 32;
    }
    if (ok && content && h.version == FEI_PROG_VERSION_CTR) {
      fei_prog_nfa_ctr cd{};
      const uint64_t at = (uint64_t)off + sizeof(a);
      ctr_ok = in(at, sizeof(cd)) && a.off_ascii >= at + sizeof(cd);
      if (ctr_ok) memcpy(&cd, prog + at, sizeof(cd));
      ctr_ok = ctr_ok && cd.n_counters >= 1 && cd.n_counters <= FEI_NFA_MAX_COUNTERS && tab(cd.off_counters, 8ull * cd.n_counters);
      const uint32_t* ct = reinterpret_cast<const uint32_t*>(prog + cd.off_counters);
      const uint32_t* self_loop = reinterpret_cast<const uint32_t*>(prog + a.off_masks) + W;
      for (uint32_t i = 0; i < cd.n_counters && ctr_ok; ++i) {
        const uint32_t pos = ct[2 * i], bound = ct[2 * i + 1];
        ctr_ok = pos >= 1 && pos < a.n_pos && !(self_loop[pos >> 5] >> (pos & 31u) & 1u) && bound >= 1;
      }
    }
    return ok;
  };
  const fei_prog_slot* sl = reinterpret_cast<const fei_prog_slot*>(prog + h.off_slots);
  for (uint32_t s = 0; s < h.n_slots; ++s)
    if ((!sl[s].off_val_dfa && !sl[s].off_val_nfa) || !dfa_ok(sl[s].off_val_dfa) || !nfa_ok(sl[s].off_val_nfa, false)) { set_error("bad slot automaton"); return FEI_E_BADARG; }
  if (h.n_slots && !h.off_key_dfa) { set_error("slots without a key DFA"); return FEI_E_BADARG; }
  if (h.off_head_nfa) {                            // flags and name fields
    fei_prog_head_nfa hn;
    if (!in(h.off_head_nfa, sizeof(hn)) || (h.head_bytes && h.off_head_nfa + sizeof(hn) > h.head_bytes)) { set_error("head position automata out of bounds"); return FEI_E_BADARG; }
    memcpy(&hn, prog + h.off_head_nfa, sizeof(hn));
    bool ok = nfa_ok(hn.off_flags_nfa, false);
    for (int k = 0; k < FEI_NAME_FIELDS && ok; ++k) ok = nfa_ok(hn.off_name_nfa[k], false);
    if (!ok) { set_error("bad flags / name position automaton in program"); return FEI_E_BADARG; }
  }
  if (!nfa_ok(h.off_body_nfa, true)) { set_error("bad content position automaton in program"); return FEI_E_BADARG; }
  if ((h.version != FEI_PROG_VERSION) != (n_nfa != 0)) { set_error("bad program magic/version"); return FEI_E_BADARG; }
  if (!ctr_ok) { set_error("bad counters of the content position automaton in program"); return FEI_E_BADARG; }
  if (h.off_body_nfa) {
    fei_prog_dfa d{};
    if (h.off_body_dfa) memcpy(&d, prog + h.off_body_dfa, sizeof(d));
    if (h.off_body_dfa && (d.n_cols == 256 || d.sticky || d.table_bytes % 16)) { set_error("the body DFA next to a position automaton must be class-indexed"); return FEI_E_BADARG; }
  }
  const fei_prog_query* qs = reinterpret_cast<const fei_prog_query*>(prog + h.off_queries);
  for (uint32_t q = 0; q < h.n_queries; ++q) if (qs[q].cond_begin > qs[q].cond_end || qs[q].cond_end > h.n_conds) { set_error("bad query range"); return FEI_E_BADARG; }
  for (uint32_t c = 0; c < h.n_conds; ++c) {        // folder-set bitmaps: inside the blob, and inside the head the kernels stage
    fei_prog_cond cd; memcpy(&cd, prog + h.off_conds + (uint64_t)c * sizeof(cd), sizeof(cd));
    if (cd.kind != FEI_C_FOLDER_SET || !cd.off_set_words) continue;
    const uint64_t end = cd.off_set_words + 4ull * cd.n_set_words;
    if (!cd.n_set_words || cd.n_set_words > 2048 || !in(cd.off_set_words, 4ull * cd.n_set_words) || (h.head_bytes && end > h.head_bytes)) {
      set_error("bad folder-set bitmap in program"); return FEI_E_BADARG;
    }
  }
  return FEI_OK;
}


enum { kCompactNone = kScanCompactNone, kCompactLists = kScanCompactLists };
constexpr int kWorkCounters = 6;           // work_counter: [0] = BodyArgs::next, [2] = header survivors, the rest see BodyArgs::counter

// key_lut for the program already in c->prog, queued on s: which of the program's fields each distinct header key of the corpus names
static int build_key_lut(fei_corpus* c, cudaStream_t s) {
  FEI_TRY(c->key_lut.ensure(kKeySlots * sizeof(uint32_t)));
  k_key_lut<<<kKeySlots / 128, 128, 0, s>>>(c->prog.as<uint8_t>(), c->hdr.as<uint8_t>(), c->key_tag.as<unsigned long long>(),
                                            c->key_rep.as<unsigned long long>(), c->key_len.as<uint32_t>(), c->key_lut.as<uint32_t>());
  return FEI_OK;
}

// Everything is queued on the context stream; nothing here waits for the GPU.
int run_scan(fei_corpus* c, const uint8_t* prog, uint64_t prog_len, int compact_mode, ScanHook* hook) {
  FEI_TRY(require_loaded(c));
  FEI_TRY(check_prog(prog, prog_len));
  Context& cx = ctx();
  cudaStream_t s = cx.stream;
  fei_prog_hdr h; memcpy(&h, prog, sizeof(h));
  uint64_t n = c->n;
  c->timing = fei_scan_timing{};
  c->last_nq = h.n_queries;
  for (uint32_t q = 0; q < 32; ++q) c->last_counts[q] = 0;
  FEI_TRY(c->prog.ensure(prog_len + 16));
  FEI_TRY(c->hits.ensure((n ? n : 1) * sizeof(uint32_t)));
  FEI_TRY(c->work_counter.ensure(kWorkCounters * sizeof(unsigned long long)));
  FEI_CUDA(cudaEventRecord(c->ev[0], s));
  FEI_CUDA(cudaMemcpyAsync(c->prog.p, prog, prog_len, cudaMemcpyHostToDevice, s));
  FEI_CUDA(cudaMemsetAsync(c->work_counter.p, 0, kWorkCounters * sizeof(unsigned long long), s));
  bool need_head = h.head_mask != 0;
  bool need_body = (h.off_body_dfa != 0 || h.off_body_nfa != 0) && h.body_mask != 0;
  const bool nfa = need_body && h.off_body_nfa != 0;           // k_body_nfa (with the body DFA, if any, stepped alongside)
  // head position automata (check_prog validated them): the kHeadNfa instances of the head kernels run them
  fei_prog_head_nfa hn{};
  if (h.off_head_nfa) memcpy(&hn, prog + h.off_head_nfa, sizeof(hn));
  bool head_nfa = h.off_head_nfa != 0;
  for (uint32_t k = 0; k < h.n_slots; ++k) head_nfa = head_nfa || reinterpret_cast<const fei_prog_slot*>(prog + h.off_slots)[k].off_val_nfa != 0;
  // a folder set held as a bitmap (folder ids of 64 and above): the kFolderBits instances of the head kernels, which are
  // instantiated only next to kHeadNfa (they run programs without head automata too)
  bool folder_bits = false;
  for (uint32_t k = 0; k < h.n_conds; ++k) {
    const fei_prog_cond* cd = reinterpret_cast<const fei_prog_cond*>(prog + h.off_conds) + k;
    folder_bits = folder_bits || (cd->kind == FEI_C_FOLDER_SET && cd->off_set_words != 0);
  }
  if ((h.off_name_dfa[0] || h.off_name_dfa[1] || h.off_name_dfa[2] || hn.off_name_nfa[0] || hn.off_name_nfa[1] || hn.off_name_nfa[2]) && !c->name.p) {
    set_error("program reads filename / id / hostname but the corpus was packed without names"); return FEI_E_STATE;
  }
  const uint32_t nq = h.n_queries;
  const uint64_t nblocks = (n + kCompactRecs - 1) / kCompactRecs;
  if (compact_mode == kCompactLists) {
    FEI_TRY(c->compact.blk_counts.ensure((nblocks ? nblocks : 1) * nq * sizeof(uint32_t)));
    FEI_TRY(c->compact.blk_offsets.ensure((nblocks ? nblocks : 1) * nq * sizeof(uint64_t)));
    FEI_TRY(c->compact.totals.ensure(32 * sizeof(uint64_t)));
    FEI_TRY(c->hit_lists.ensure((n ? n : 1) * nq * sizeof(uint32_t)));
    c->hit_list_stride = n ? n : 1;
    FEI_CUDA(cudaMemsetAsync(c->compact.totals.p, 0, 32 * sizeof(uint64_t), s));
  }
  FEI_CUDA(cudaEventRecord(c->ev[1], s));
  uint32_t launches = 0;
  if (n && need_head) {
    HeadArgs a{c->prog.as<uint8_t>(), c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), c->name.as<uint8_t>(), c->name_off.as<uint64_t>(),
               c->name_spans.as<uint16_t>(), c->wall.as<int64_t>(), c->flags8.as<uint64_t>(), c->fsb.as<uint32_t>(), n, c->hits.as<uint32_t>(),
               c->hdir.as<uint2>(), c->hdir_off.as<uint64_t>(), c->key_lut.as<uint32_t>(), false,
               c->slot_col.as<int8_t>(), c->col_len.as<uint16_t>(), c->col_planes.as<uint8_t>(), c->ts.as<int64_t>(), {}};
    {
      const fei_prog_cond* cds = reinterpret_cast<const fei_prog_cond*>(prog + h.off_conds);
      for (uint32_t k = 0; k < h.n_conds; ++k)
        if (cds[k].kind == FEI_C_RECBITS) {
          const uint32_t x = cds[k].ref;
          if (x >= FEI_MAX_AUX || !c->aux[x].p || c->aux_n[x] != n) { set_error("program reads aux column %u, which is not set for this corpus state (fei_corpus_set_aux)", x); return FEI_E_STATE; }
        }
      for (int x = 0; x < FEI_MAX_AUX; ++x) a.aux[x] = c->aux[x].as<uint8_t>();
    }
    if (h.n_slots) {
      FEI_TRY(build_key_lut(c, s));
      a.key_lut = c->key_lut.as<uint32_t>();
      FEI_TRY(c->slot_col.ensure(FEI_MAX_SLOTS));
      FEI_TRY(c->kid_col.ensure(kKeySlots));
      a.slot_col = c->slot_col.as<int8_t>();
      k_slot_cols<<<1, 32, 0, s>>>(c->prog.as<uint8_t>(), c->key_lut.as<uint32_t>(), c->kid_col.as<int8_t>(), c->n_cols, c->has_text_records ? 1u : 0u, c->slot_col.as<int8_t>());
      launches += 2;
    }
    // selective meta predicates first: stream the meta columns, collect survivors
    FEI_TRY(c->survivors.ensure((n + 32) * sizeof(Survivor)));
    unsigned int* d_count = reinterpret_cast<unsigned int*>(c->work_counter.as<unsigned long long>() + 2);
    const unsigned meta_grid = (unsigned)((n + 256 * kMetaPer - 1) / (256 * kMetaPer));
    // One fused kernel when no meta predicate can thin out the records that need header fields (then every one of them is
    // finished where it was read, no work list); otherwise the meta pass collects the survivors and k_head_parse runs them dense.
    bool fuse = !(getenv("FEI_HEAD_FUSE") && getenv("FEI_HEAD_FUSE")[0] == '0');
    {
      const fei_prog_cond* cds = reinterpret_cast<const fei_prog_cond*>(prog + h.off_conds);
      const fei_prog_query* qs = reinterpret_cast<const fei_prog_query*>(prog + h.off_queries);
      for (uint32_t q = 0; q < h.n_queries && fuse; ++q) {
        if (!((h.slot_mask | h.name_mask) >> q & 1u)) continue;
        for (uint32_t k = qs[q].cond_begin; k < qs[q].cond_end; ++k) {
          const uint8_t kind = cds[k].kind;
          if (kind == FEI_C_SLOT && cds[k].if_missing == 2) { ++k; continue; }      // the fallback field is decided with the header
          if (kind == FEI_C_FLAGS || kind == FEI_C_DATE_CMP || kind == FEI_C_FOLDER_SET || kind == FEI_C_STATUS_SET || kind == FEI_C_RECBITS || kind == FEI_C_TS_CMP) { fuse = false; break; }
        }
      }
    }
    if (fuse) {
      (folder_bits ? k_head_meta<true, true, true> : head_nfa ? k_head_meta<true, true, false> : k_head_meta<true, false, false>)<<<meta_grid, 256, 0, s>>>(a, nullptr, nullptr);
      ++launches;
    } else {
      (folder_bits ? k_head_meta<false, true, true> : head_nfa ? k_head_meta<false, true, false> : k_head_meta<false, false, false>)<<<meta_grid, 256, 0, s>>>(a, c->survivors.as<Survivor>(), d_count);
      ++launches;
      if (h.slot_mask | h.name_mask) {                         // somebody may need header text or name fields
        (folder_bits ? k_head_parse<true, true> : head_nfa ? k_head_parse<true, false> : k_head_parse<false, false>)<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a, c->survivors.as<Survivor>(), d_count);
        ++launches;
      }
    }
  }
  FEI_CUDA(cudaEventRecord(c->ev[2], s));

  // ---- body pass: one launch over all groups
  fei_prog_dfa d; memset(&d, 0, sizeof(d));
  size_t smem = 0;
  int acc_mode = 0; bool direct = false, sticky_kernel = false, gather = false;
  fei_prog_nfa na; memset(&na, 0, sizeof(na));
  if (n && nfa) {
    if (h.off_body_dfa) memcpy(&d, prog + h.off_body_dfa, sizeof(d));
    memcpy(&na, prog + h.off_body_nfa, sizeof(na));
    smem = (size_t)d.table_bytes + na.table_bytes;
    if (smem > 220 * 1024) { set_error("content automata need %zu bytes of shared memory (limit 220 KiB)", smem); return FEI_E_UNSUPPORTED; }
    c->timing.body_kernel = 4u;
    c->timing.body_nfa_words = na.n_words;
    if (h.version == FEI_PROG_VERSION_CTR)
      c->timing.body_nfa_counters = reinterpret_cast<const fei_prog_nfa_ctr*>(prog + h.off_body_nfa + sizeof(fei_prog_nfa))->n_counters;
  } else if (n && need_body) {
    memcpy(&d, prog + h.off_body_dfa, sizeof(d));
    smem = d.table_bytes;
    if (smem > 220 * 1024) { set_error("content automaton needs %zu bytes of shared memory (limit 220 KiB)", smem); return FEI_E_UNSUPPORTED; }
    acc_mode = d.sticky ? 3 : d.n_acc <= 32 ? 1 : d.n_acc <= 64 ? 2 : 0;
    direct = d.n_cols == 256;
    sticky_kernel = direct && acc_mode == 3 && (uint64_t)d.n_states * d.row_stride * 2 + kStickyAddrSlack <= kStickyAddrLimit;
    gather = sticky_kernel && need_head && n >= 65536;         // few survivors of the header pass: one thread per record (device-side choice)
    c->timing.body_kernel = gather ? 2u : sticky_kernel ? 1u : 3u;     // gather: finish_timing settles it from the live count
    c->timing.body_direct = direct ? 1u : 0u;
    c->timing.body_acc_mode = (uint32_t)acc_mode;
  } else if (n && !need_head) {
    // no condition reads the corpus at all (constant queries): every record gets the constant verdict
    // (program.py folds constants into head conditions, so this only happens for empty condition lists)
    uint32_t all_q = nq >= 32 ? 0xFFFFFFFFu : ((1u << nq) - 1u);
    k_fill32<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(c->hits.as<uint32_t>(), n, all_q);
    ++launches;
  }
  const uint64_t n_windows = (n + kWindow - 1) / kWindow;
  // k_body (every multi-pattern scan, and single-pattern ones the sticky kernel cannot take) builds the ordered lists inside the
  // scan; the other scans compact the finished masks with k_count / k_scan_blocks / k_emit after it
  const bool body_lists = n && need_body && !nfa && !sticky_kernel && compact_mode == kCompactLists;
  // multi-GPU: the scan kernel stores every finished window's masks into the peers (k_body_gather and k_body_nfa do not: the
  // hook copies them)
  const bool push = n && need_body && !nfa && !gather && hook && hook->push_peers && hook->push_n;
  BodyArgs a{c->prog.as<uint8_t>(), c->tiles.as<uint8_t>(), c->grp_base.as<uint64_t>(), c->grp_rec.as<uint32_t>(), c->grp_len.as<uint32_t>(),
             c->n_groups, c->hits.as<uint32_t>(), need_head ? 1 : 0, c->work_counter.as<unsigned long long>(), 0ull,
             c->work_counter.as<unsigned long long>(), nullptr};
  a.n_records = n;
  const unsigned grid = (unsigned)cx.sm_count;
  if (n && need_body && gather) {
    a.gather_max = n / kGatherDiv;
    FEI_TRY(c->live_list.ensure((a.gather_max + 1) * sizeof(uint32_t)));
    k_live_list<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(c->hits.as<uint32_t>(), n, c->live_list.as<uint32_t>(), a.counter + 4, a.gather_max);
    FEI_TRY(launch_body(k_body_gather, kBodyThreads, grid, smem, s, a, c->live_list.as<uint32_t>(), c->rec_pos.as<uint32_t>()));
    launches += 2;
  }
  if (body_lists || push) {                                    // window counters (and, for body_lists, descriptors) for the scan
    FEI_TRY(c->win_done.ensure((n_windows + 1) * sizeof(unsigned int)));
    FEI_CUDA(cudaMemsetAsync(c->win_done.p, 0, (n_windows + 1) * sizeof(unsigned int), s));
    a.win_done = c->win_done.as<unsigned int>();
  }
  if (body_lists) {
    FEI_TRY(c->win_state.ensure(n_windows * kWinBytes));
    FEI_CUDA(cudaMemsetAsync(c->win_state.p, 0, n_windows * kWinBytes, s));
    a.win_state = c->win_state.as<uint8_t>();
    a.lists = c->hit_lists.as<uint32_t>(); a.list_stride = c->hit_list_stride;
    a.totals = c->compact.totals.as<unsigned long long>(); a.nq = nq;
  }
  if (push) { a.push_peers = hook->push_peers; a.push_n = hook->push_n; a.push_off = hook->push_off; hook->pushed = true; }
  if (n && nfa) {
    const BodyNfaKernel k = body_nfa_kernel(na.n_words, h.off_body_dfa != 0, c->timing.body_nfa_counters != 0);
    FEI_TRY(launch_body(k.k, k.threads, grid, smem, s, a));
    ++launches;
  } else if (n && need_body) {
    const size_t body_smem = sticky_kernel ? ((smem + 127) & ~(size_t)127) + kStickyRingBytes : smem;   // k_body_sticky: + its rings
    FEI_TRY(launch_body(body_kernel(sticky_kernel, direct, acc_mode, a.push_n != 0), kBodyThreads, grid, body_smem, s, a));
    ++launches;
  }
  FEI_CUDA(cudaEventRecord(c->ev[3], s));
  if (n && compact_mode == kCompactLists && !body_lists) {
    compact_lists<uint32_t>(c->hits.as<uint32_t>(), n, nq, 0u, c->compact, c->hit_list_stride, c->hit_lists.as<uint32_t>(), s);
    launches += 3;
  }
  if (hook) FEI_TRY(hook->after_scan(s));
  if (compact_mode == kCompactLists)
    FEI_CUDA(cudaMemcpyAsync(c->last_counts, c->compact.totals.p, nq * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaEventRecord(c->ev[4], s));
  FEI_CUDA(cudaGetLastError());
  c->timing.kernel_launches = launches;
  return FEI_OK;
}

int finish_timing(fei_corpus* c, bool compacted) {
  cudaStream_t s = ctx().stream;
  FEI_CUDA(cudaEventRecord(c->ev[5], s));
  FEI_CUDA(cudaStreamSynchronize(s));
  float t;
  FEI_CUDA(cudaEventElapsedTime(&t, c->ev[0], c->ev[1])); c->timing.h2d_ms = t;
  FEI_CUDA(cudaEventElapsedTime(&t, c->ev[1], c->ev[2])); c->timing.head_ms = t;
  FEI_CUDA(cudaEventElapsedTime(&t, c->ev[2], c->ev[3])); c->timing.body_ms = t;
  if (compacted) { FEI_CUDA(cudaEventElapsedTime(&t, c->ev[3], c->ev[4])); c->timing.compact_ms = t; }   // what is left after the body kernel
  FEI_CUDA(cudaEventElapsedTime(&t, c->ev[4], c->ev[5])); c->timing.d2h_ms = t;
  FEI_CUDA(cudaEventElapsedTime(&t, c->ev[0], c->ev[5])); c->timing.total_ms = t;
  unsigned long long cnt[kWorkCounters] = {0};
  FEI_CUDA(cudaMemcpy(cnt, c->work_counter.as<unsigned long long>(), sizeof(cnt), cudaMemcpyDeviceToHost));
  c->timing.body_bytes_touched = cnt[1];
  c->timing.body_bytes_read = cnt[3];
  if (c->timing.body_kernel == 2u && cnt[4] > c->n / kGatherDiv) c->timing.body_kernel = 1u;   // k_body_sticky took the dense case
  if (cnt[5]) { set_error("ordered hit lists: a wait in the look-back or for a window's offsets (help_tail) timed out"); return FEI_E_CUDA; }
  return FEI_OK;
}

// Order-preserving compaction of a mask array into per-query lists of global indices (one shot, any stream; used for the
// rank segments of an all-gathered mask array).  counts_out[q] = hits of query q; when `lists` is given,
// lists[q * stride + k] = k-th hit (stride = max count).
int compact_masks(const uint32_t* masks, uint64_t n, uint32_t nq, uint64_t global_base, CompactScratch& sc,
                  uint64_t* counts_out, DevBuf* lists, uint64_t* stride_out, uint32_t* launches, cudaStream_t s) {
  uint64_t nblocks = (n + kCompactRecs - 1) / kCompactRecs;
  for (uint32_t q = 0; q < nq; ++q) counts_out[q] = 0;
  if (stride_out) *stride_out = 1;
  if (n == 0) return FEI_OK;
  FEI_TRY(sc.blk_counts.ensure(nblocks * nq * sizeof(uint32_t)));
  FEI_TRY(sc.blk_offsets.ensure(nblocks * nq * sizeof(uint64_t)));
  FEI_TRY(sc.totals.ensure(32 * sizeof(uint64_t)));
  FEI_CUDA(cudaMemsetAsync(sc.totals.p, 0, 32 * sizeof(uint64_t), s));
  k_count<<<(unsigned)nblocks, kCompactBlock, 0, s>>>(masks, n, nq, sc.blk_counts.as<uint32_t>());
  k_scan_blocks<<<nq, 256, 0, s>>>(sc.blk_counts.as<uint32_t>(), nblocks, nq, sc.blk_offsets.as<uint64_t>(), sc.totals.as<uint64_t>());
  if (launches) *launches += 2;
  FEI_CUDA(cudaMemcpyAsync(counts_out, sc.totals.p, nq * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  if (lists) {
    uint64_t stride = 1;
    for (uint32_t q = 0; q < nq; ++q) if (counts_out[q] > stride) stride = counts_out[q];
    if (stride_out) *stride_out = stride;
    FEI_TRY(lists->ensure(stride * nq * sizeof(uint64_t)));
    k_emit<unsigned long long><<<(unsigned)nblocks, kCompactBlock, 0, s>>>(masks, n, nq, sc.blk_offsets.as<uint64_t>(), global_base, stride,
                                                                         lists->as<unsigned long long>());
    if (launches) *launches += 1;
  }
  FEI_CUDA(cudaGetLastError());
  return FEI_OK;
}

// Global ordered lists from an all-gathered, rank-major mask array: segment r = masks[r * seg_stride .. + seg_n[r]), its
// record 0 is global index seg_base[r].  lists[q * stride + k]; totals_out[q] (host) after a final sync.
int compact_segments(const uint32_t* masks, uint64_t seg_stride, const uint64_t* seg_n, const uint64_t* seg_base, uint32_t n_seg, uint32_t nq,
                     CompactScratch& sc, uint64_t stride, uint64_t* lists, uint64_t* totals_out, cudaStream_t s) {
  uint64_t n_max = 0;
  for (uint32_t r = 0; r < n_seg; ++r) if (seg_n[r] > n_max) n_max = seg_n[r];
  const uint64_t nb_max = (n_max + kCompactRecs - 1) / kCompactRecs;
  FEI_TRY(sc.blk_counts.ensure((nb_max ? nb_max : 1) * nq * sizeof(uint32_t)));
  FEI_TRY(sc.blk_offsets.ensure((nb_max ? nb_max : 1) * nq * sizeof(uint64_t)));
  FEI_TRY(sc.totals.ensure(32 * sizeof(uint64_t)));
  FEI_CUDA(cudaMemsetAsync(sc.totals.p, 0, 32 * sizeof(uint64_t), s));
  for (uint32_t r = 0; r < n_seg; ++r)                         // the totals run on across segments
    if (seg_n[r]) compact_lists<unsigned long long>(masks + (size_t)r * seg_stride, seg_n[r], nq, seg_base[r], sc, stride,
                                                    reinterpret_cast<unsigned long long*>(lists), s);
  if (totals_out) {
    FEI_CUDA(cudaMemcpyAsync(totals_out, sc.totals.p, nq * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaStreamSynchronize(s));
  }
  FEI_CUDA(cudaGetLastError());
  return FEI_OK;
}

// (A, S) checksums of `count` indices base + list[k] (device memory); see k_list_checksum
template <class T>
static int list_checksum_of(const T* list, uint64_t count, uint64_t base, DevBuf& tmp, uint64_t* a_out, uint64_t* s_out, cudaStream_t s) {
  FEI_TRY(tmp.ensure(16));
  FEI_CUDA(cudaMemsetAsync(tmp.p, 0, 16, s));
  if (count) k_list_checksum<T><<<(unsigned)std::min<uint64_t>((count + 255) / 256, 4096), 256, 0, s>>>(list, count, base, tmp.as<unsigned long long>());
  unsigned long long r[2];
  FEI_CUDA(cudaMemcpyAsync(r, tmp.p, 16, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  *a_out = r[0]; *s_out = r[1];
  return FEI_OK;
}
int list_checksum(const uint64_t* list, uint64_t count, DevBuf& tmp, uint64_t* a_out, uint64_t* s_out, cudaStream_t s) {
  return list_checksum_of(list, count, 0, tmp, a_out, s_out, s);
}
int list_checksum(const uint32_t* list, uint64_t count, uint64_t base, DevBuf& tmp, uint64_t* a_out, uint64_t* s_out, cudaStream_t s) {
  return list_checksum_of(list, count, base, tmp, a_out, s_out, s);
}

int widen_list(const uint32_t* src, uint64_t n, uint64_t base, uint64_t* dst, cudaStream_t s) {
  if (n) k_widen<<<(unsigned)std::min<uint64_t>((n + 255) / 256, 4096), 256, 0, s>>>(src, n, base, dst);
  FEI_CUDA(cudaGetLastError());
  return FEI_OK;
}

// Copies (a prefix of) every query's list of the last scan to the host as global indices: each list is widened on the device
// into c->list_stage (one buffer, reused in stream order) and copied from there.  *truncated: some cap[q] was too small.
static int copy_lists_out(fei_corpus* c, uint32_t nq, uint64_t* const* hits, const uint64_t* cap, bool* truncated, cudaStream_t s) {
  uint64_t most = 0;
  for (uint32_t q = 0; q < nq; ++q) {
    const uint64_t take = c->last_counts[q] < cap[q] ? c->last_counts[q] : cap[q];
    if (take < c->last_counts[q]) *truncated = true;
    if (hits[q] && take > most) most = take;
  }
  if (!most) return FEI_OK;
  FEI_TRY(c->list_stage.ensure(most * sizeof(uint64_t)));
  for (uint32_t q = 0; q < nq; ++q) {
    const uint64_t take = c->last_counts[q] < cap[q] ? c->last_counts[q] : cap[q];
    if (!take || !hits[q]) continue;
    FEI_TRY(widen_list(c->hit_lists.as<uint32_t>() + q * c->hit_list_stride, take, c->global_base, c->list_stage.as<uint64_t>(), s));
    FEI_CUDA(cudaMemcpyAsync(hits[q], c->list_stage.p, take * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  }
  return FEI_OK;
}

}  // namespace fei

using namespace fei;

extern "C" int fei_scan_masks(fei_corpus* c, const uint8_t* prog, uint64_t prog_len, uint32_t* masks) {
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(run_scan(c, prog, prog_len, kCompactNone, nullptr));
  if (masks && c->n) FEI_CUDA(cudaMemcpyAsync(masks, c->hits.p, c->n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx().stream));
  return finish_timing(c, false);
}

extern "C" int fei_scan_count(fei_corpus* c, const uint8_t* prog, uint64_t prog_len, uint64_t* nhits) {
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(run_scan(c, prog, prog_len, kCompactLists, nullptr));     // lists stay on the device (fei_comm_allgather_hits, fei_scan_list_checksum)
  FEI_TRY(finish_timing(c, true));
  if (nhits) for (uint32_t q = 0; q < c->last_nq; ++q) nhits[q] = c->last_counts[q];
  return FEI_OK;
}

extern "C" int fei_scan_hits(fei_corpus* c, const uint8_t* prog, uint64_t prog_len,
                             uint64_t* const* hits, const uint64_t* cap, uint64_t* nhits) {
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  if (!hits || !cap || !nhits) { set_error("null argument"); return FEI_E_BADARG; }
  FEI_TRY(run_scan(c, prog, prog_len, kCompactLists, nullptr));
  cudaStream_t s = ctx().stream;
  FEI_CUDA(cudaStreamSynchronize(s));                                  // the counts decide how much of every list is copied
  bool truncated = false;
  for (uint32_t q = 0; q < c->last_nq; ++q) nhits[q] = c->last_counts[q];
  FEI_TRY(copy_lists_out(c, c->last_nq, hits, cap, &truncated, s));
  FEI_TRY(finish_timing(c, true));
  if (truncated) { set_error("hit buffer too small for at least one query (see nhits)"); return FEI_E_CAPACITY; }
  return FEI_OK;
}

/* copies (a prefix of) the ordered lists the last fei_scan_count left on the device: no second scan */
extern "C" int fei_scan_fetch_hits(fei_corpus* c, uint32_t nq, uint64_t* const* hits, const uint64_t* cap) {
  if (!c || !hits || !cap) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  if (nq == 0 || nq != c->last_nq || !c->hit_lists.p) { set_error("no matching scan result with lists on this corpus"); return FEI_E_STATE; }
  cudaStream_t s = ctx().stream;
  bool truncated = false;
  FEI_TRY(copy_lists_out(c, nq, hits, cap, &truncated, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  if (truncated) { set_error("hit buffer too small for at least one query"); return FEI_E_CAPACITY; }
  return FEI_OK;
}

/* (A, S) checksums of the ordered hit lists the last fei_scan_count / fei_scan_hits left on the device */
extern "C" int fei_scan_list_checksum(fei_corpus* c, uint32_t nq, uint64_t* a_out, uint64_t* s_out) {
  if (!c || !a_out || !s_out) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  if (nq == 0 || nq != c->last_nq || !c->hit_lists.p) { set_error("no matching scan result with lists on this corpus"); return FEI_E_STATE; }
  for (uint32_t q = 0; q < nq; ++q)
    FEI_TRY(list_checksum(c->hit_lists.as<uint32_t>() + q * c->hit_list_stride, c->last_counts[q], c->global_base, c->scan_tmp, a_out + q, s_out + q, ctx().stream));
  return FEI_OK;
}

extern "C" int fei_scan_last_timing(const fei_corpus* c, fei_scan_timing* out) {
  if (!c || !out) { set_error("null argument"); return FEI_E_BADARG; }
  *out = c->timing;
  return FEI_OK;
}

// ---------------------------------------------------------------- token histogram of a header field ("next" row 4)
// MemdirFolderManager.get_folder_stats (memdir_tools/folders.py:286-292):
//     if "Tags" in memory["headers"]: for tag in [t.strip() for t in headers["Tags"].split(",")]: stats["tags"][tag] += 1
// One thread per selected record walks the record's header directory for the field (exact key: slot 0 of the program,
// last line wins), splits the value at `sep`, strips every piece with Python's whitespace set and counts it in a device
// hash table (64-bit hash, representative spelling = smallest header offset, every piece verified against it in a
// second pass).  `first` orders the tokens the way the reference's dict does (first record, then position in the value).
namespace fei {
constexpr uint32_t kTokSlots = 1u << 16;
struct TokTable { unsigned long long* tag; unsigned long long* rep; unsigned long long* first; uint32_t* len; uint32_t* count; uint32_t* flag; };

__device__ __forceinline__ unsigned long long tok_hash(const uint8_t* p, uint32_t n) {
  unsigned long long h = 0x9E3779B97F4A7C15ull;
  for (uint32_t i = 0; i < n; ++i) { h ^= p[i]; h *= 0x100000001b3ull; }
  h ^= h >> 31; h *= 0xD6E8FEB86659FD93ull; h ^= h >> 32;
  return h | 1ull;
}

template <int kPass>
__global__ void __launch_bounds__(256) k_tok_hist(const uint8_t* __restrict__ hdr, const uint64_t* __restrict__ hdr_off,
                                                  const uint2* __restrict__ hdir, const uint64_t* __restrict__ hdir_off,
                                                  const uint32_t* __restrict__ key_lut, const uint32_t* __restrict__ alive, uint64_t n,
                                                  uint8_t sep, TokTable t) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n || !(alive[i] & 1u)) return;
  const uint2* ent = hdir + hdir_off[i];
  const uint32_t n_ent = (uint32_t)(hdir_off[i + 1] - hdir_off[i]);
  if (text_record(ent, n_ent)) { atomicOr(t.flag, 4u); return; }                   // header parsed from its text: not handled here
  uint32_t voff, vlen;                                                               // slot 0, exact key: the last line wins
  if (!header_lookup<1>(DirLines{ent, n_ent, key_lut}, [](int) { return 1u; }, &voff, &vlen, no_values)) return;
  const uint8_t* v = hdr + hdr_off[i] + voff;
  uint32_t pos = 0, idx = 0;
  for (;;) {                                                     // str.split(sep): k separators -> k + 1 pieces, empty ones included
    uint32_t end = pos;
    while (end < vlen && v[end] != sep) ++end;
    const uint8_t* a = v + pos; const uint8_t* b = v + end;
    strip_span(a, b);
    const uint32_t len = (uint32_t)(b - a);
    const unsigned long long h = tok_hash(a, len);
    uint32_t s = (uint32_t)(h >> 20) & (kTokSlots - 1);
    bool placed = false;
    for (uint32_t probe = 0; probe < kTokSlots / 2 && !placed; ++probe, s = (s + 1) & (kTokSlots - 1)) {
      unsigned long long cur = t.tag[s];
      if (cur == 0 && kPass == 0) cur = atomicCAS(t.tag + s, 0ull, h), cur = cur == 0 ? h : cur;
      if (cur == h) {
        placed = true;
        if (kPass == 0) {
          atomicAdd(t.count + s, 1u);
          atomicMin(t.rep + s, (unsigned long long)(a - hdr));
          atomicMin(t.first + s, (unsigned long long)i << 20 | (idx < 0xFFFFFu ? idx : 0xFFFFFu));
          t.len[s] = len;
        } else {
          bool same = t.len[s] == len;
          const uint8_t* r = hdr + t.rep[s];
          for (uint32_t k = 0; same && k < len; ++k) same = r[k] == a[k];
          if (!same) atomicOr(t.flag, 2u);                       // two different pieces with one 64-bit hash
        }
      } else if (cur == 0) break;                                // pass 1 only: cannot happen after pass 0
    }
    if (!placed) atomicOr(t.flag, 1u);                           // table over-full
    ++idx;
    if (end >= vlen) break;
    pos = end + 1;
  }
}

__global__ void k_tok_pack(const uint8_t* __restrict__ hdr, const unsigned long long* __restrict__ rep, const uint32_t* __restrict__ len,
                           const uint32_t* __restrict__ slots, const uint64_t* __restrict__ out_off, uint32_t n_tok, uint8_t* __restrict__ out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_tok) return;
  const uint32_t s = slots[k];
  const uint8_t* p = hdr + rep[s];
  for (uint32_t b = 0; b < len[s]; ++b) out[out_off[k] + b] = p[b];
}
}  // namespace fei

extern "C" int fei_corpus_token_histogram(fei_corpus* c, const uint8_t* prog, uint64_t prog_len, uint8_t sep,
                                          uint8_t* tok_blob, uint64_t blob_cap, uint64_t* tok_off, uint64_t* tok_count, uint64_t* tok_first,
                                          uint64_t cap, uint64_t* n_tokens) {
  if (!c || !n_tokens || !tok_off) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  *n_tokens = 0; tok_off[0] = 0;
  FEI_TRY(run_scan(c, prog, prog_len, kCompactNone, nullptr));
  fei_prog_hdr h; memcpy(&h, prog, sizeof(h));
  if (h.n_queries != 1 || h.n_slots < 1) { set_error("token histogram wants one query whose first header field names the column"); return FEI_E_BADARG; }
  if (c->n == 0) return finish_timing(c, false);
  if (c->has_text_records || !c->hdir.p) { set_error("corpus holds records whose header is parsed from its text; the token histogram does not handle them"); return FEI_E_UNSUPPORTED; }
  cudaStream_t s = ctx().stream;
  DevBuf& tb = c->scan_tmp;
  const size_t bytes = (size_t)kTokSlots * (8 + 8 + 8 + 4 + 4) + 16;
  FEI_TRY(tb.ensure(bytes));
  uint8_t* base = tb.as<uint8_t>();
  TokTable t{reinterpret_cast<unsigned long long*>(base), reinterpret_cast<unsigned long long*>(base) + kTokSlots, reinterpret_cast<unsigned long long*>(base) + 2 * kTokSlots,
             reinterpret_cast<uint32_t*>(base + (size_t)kTokSlots * 24), reinterpret_cast<uint32_t*>(base + (size_t)kTokSlots * 28), reinterpret_cast<uint32_t*>(base + (size_t)kTokSlots * 32)};
  FEI_CUDA(cudaMemsetAsync(base, 0, bytes, s));
  FEI_CUDA(cudaMemsetAsync(t.rep, 0xFF, (size_t)kTokSlots * 16, s));           // rep and first: ~0 so that atomicMin works
  const unsigned grid = (unsigned)((c->n + 255) / 256);
  k_tok_hist<0><<<grid, 256, 0, s>>>(c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), c->hdir.as<uint2>(), c->hdir_off.as<uint64_t>(), c->key_lut.as<uint32_t>(),
                                     c->hits.as<uint32_t>(), c->n, sep, t);
  k_tok_hist<1><<<grid, 256, 0, s>>>(c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), c->hdir.as<uint2>(), c->hdir_off.as<uint64_t>(), c->key_lut.as<uint32_t>(),
                                     c->hits.as<uint32_t>(), c->n, sep, t);
  std::vector<unsigned long long> tag(kTokSlots), first(kTokSlots);
  std::vector<uint32_t> len(kTokSlots), count(kTokSlots);
  uint32_t flag = 0;
  FEI_CUDA(cudaMemcpyAsync(tag.data(), t.tag, kTokSlots * 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaMemcpyAsync(first.data(), t.first, kTokSlots * 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaMemcpyAsync(len.data(), t.len, kTokSlots * 4, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaMemcpyAsync(count.data(), t.count, kTokSlots * 4, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaMemcpyAsync(&flag, t.flag, 4, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  FEI_CUDA(cudaGetLastError());
  if (flag & 4u) { set_error("a selected record's header is parsed from its text; the token histogram does not handle it"); return FEI_E_UNSUPPORTED; }
  if (flag) { set_error(flag & 1u ? "more than 32768 distinct tokens" : "64-bit hash collision between two tokens"); return FEI_E_UNSUPPORTED; }
  std::vector<uint32_t> slots;
  for (uint32_t k = 0; k < kTokSlots; ++k) if (tag[k]) slots.push_back(k);
  std::sort(slots.begin(), slots.end(), [&](uint32_t a, uint32_t b) { return first[a] < first[b]; });   // the order a dict filled record by record has
  if (slots.size() > cap) { set_error("token table too small: need %zu entries", slots.size()); return FEI_E_CAPACITY; }
  std::vector<uint64_t> off(slots.size() + 1, 0);
  for (size_t k = 0; k < slots.size(); ++k) off[k + 1] = off[k] + len[slots[k]];
  if (off.back() > blob_cap) { set_error("token buffer too small: need %llu bytes", (unsigned long long)off.back()); return FEI_E_CAPACITY; }
  if (!slots.empty()) {
    DevBuf d_slots, d_off, d_out;
    FEI_TRY(d_slots.ensure(slots.size() * 4)); FEI_TRY(d_off.ensure(off.size() * 8)); FEI_TRY(d_out.ensure(off.back() + 16));
    FEI_CUDA(cudaMemcpyAsync(d_slots.p, slots.data(), slots.size() * 4, cudaMemcpyHostToDevice, s));
    FEI_CUDA(cudaMemcpyAsync(d_off.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice, s));
    k_tok_pack<<<(unsigned)((slots.size() + 127) / 128), 128, 0, s>>>(c->hdr.as<uint8_t>(), t.rep, t.len, d_slots.as<uint32_t>(), d_off.as<uint64_t>(), (uint32_t)slots.size(), d_out.as<uint8_t>());
    if (off.back() && tok_blob) FEI_CUDA(cudaMemcpyAsync(tok_blob, d_out.p, off.back(), cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaStreamSynchronize(s));
    FEI_CUDA(cudaGetLastError());
  }
  for (size_t k = 0; k < slots.size(); ++k) {
    tok_off[k + 1] = off[k + 1];
    if (tok_count) tok_count[k] = count[slots[k]];
    if (tok_first) tok_first[k] = (first[slots[k]] >> 20) + c->global_base;
  }
  *n_tokens = slots.size();
  return finish_timing(c, false);
}


// ---------------------------------------------------------------- header values of one field, record by record
// For conditions only Python can judge value by value (search.py:126-130: Due / Created / Modified / DeletedDate go through
// dateutil.parser.parse per record), the host needs the VALUE the reference would read for every record: slot 0 of the program
// resolved with the reference's dict semantics (mode 0: first key whose lower() equals the field, last line of that exact key;
// mode 1: exact key).  k_slot_spans finds the value's span in the header blob (directory walk, or the text for headers the
// directory cannot address), k_slot_gather packs the values into one blob that goes back to the host.
namespace fei {
__global__ void __launch_bounds__(256) k_slot_spans(HeadArgs a, uint32_t* __restrict__ len_out, uint64_t* __restrict__ src_out) {
  const uint64_t rec = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (rec >= a.n) return;
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const fei_prog_slot* slots = reinterpret_cast<const fei_prog_slot*>(a.prog + ph->off_slots);
  const uint32_t m = slots[0].mode == 0 ? 0u : 1u;              // any other mode: exact key, the last line wins
  auto mode = [m](int) { return m; };
  const uint64_t hoff = a.hdr_off[rec];
  const uint8_t* h = a.hdr + hoff;
  const uint2* ent = a.hdir + a.hdir_off[rec];
  const uint32_t n_ent = (uint32_t)(a.hdir_off[rec + 1] - a.hdir_off[rec]);
  uint32_t voff = 0, vlen = 0;
  const bool have = text_record(ent, n_ent)
      ? header_lookup<1>(TextLines{h, h, a.hdr + a.hdr_off[rec + 1], a.prog, ph->off_key_dfa, false}, mode, &voff, &vlen, no_values)
      : header_lookup<1>(DirLines{ent, n_ent, a.key_lut}, mode, &voff, &vlen, no_values);
  len_out[rec] = have ? vlen : 0u;
  src_out[rec] = have ? hoff + voff : ~0ull;                     // ~0: the record has no such header
}

__global__ void __launch_bounds__(256) k_slot_gather(const uint8_t* __restrict__ hdr, const uint32_t* __restrict__ len, const uint64_t* __restrict__ src,
                                                    const uint64_t* __restrict__ off, uint64_t n, uint8_t* __restrict__ out, uint8_t* __restrict__ present) {
  const uint64_t rec = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (rec >= n) return;
  const bool have = src[rec] != ~0ull;
  present[rec] = have ? 1 : 0;
  if (!have) return;
  const uint8_t* p = hdr + src[rec];
  uint8_t* d = out + off[rec];
  for (uint32_t k = 0; k < len[rec]; ++k) d[k] = p[k];
}
}  // namespace fei

/* prog: any program whose slot 0 names the field (conditions are ignored).  Out: present[n], off[n+1] (value i =
 * blob[off[i] .. off[i+1]), empty for absent headers).  FEI_E_CAPACITY with the needed size in off[n] when blob_cap is too small. */
extern "C" int fei_corpus_slot_values(fei_corpus* c, const uint8_t* prog, uint64_t prog_len, uint8_t* present, uint64_t* off,
                                      uint8_t* blob, uint64_t blob_cap) {
  if (!c || !prog || !present || !off) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_loaded(c));
  FEI_TRY(check_prog(prog, prog_len));
  fei_prog_hdr h; memcpy(&h, prog, sizeof(h));
  if (h.n_slots < 1) { set_error("program has no header field"); return FEI_E_BADARG; }
  const uint64_t n = c->n;
  off[0] = 0;
  if (n == 0) return FEI_OK;
  cudaStream_t s = ctx().stream;
  FEI_TRY(c->prog.ensure(prog_len + 16));
  FEI_CUDA(cudaMemcpyAsync(c->prog.p, prog, prog_len, cudaMemcpyHostToDevice, s));
  FEI_TRY(build_key_lut(c, s));
  HeadArgs a{c->prog.as<uint8_t>(), c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), nullptr, nullptr, nullptr, c->wall.as<int64_t>(), c->flags8.as<uint64_t>(),
             c->fsb.as<uint32_t>(), n, nullptr, c->hdir.as<uint2>(), c->hdir_off.as<uint64_t>(), c->key_lut.as<uint32_t>(), false, nullptr, nullptr, nullptr, c->ts.as<int64_t>(), {}};
  DevBuf d_len, d_src, d_off, d_present, d_out;
  FEI_TRY(d_len.alloc(n * 4)); FEI_TRY(d_src.alloc(n * 8)); FEI_TRY(d_off.alloc((n + 1) * 8)); FEI_TRY(d_present.alloc(n));
  const unsigned grid = (unsigned)((n + 255) / 256);
  k_slot_spans<<<grid, 256, 0, s>>>(a, d_len.as<uint32_t>(), d_src.as<uint64_t>());
  FEI_TRY(queue_offsets(d_len.as<uint32_t>(), n, d_off.as<uint64_t>(), off, true, c->scan_tmp, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  FEI_TRY(d_out.alloc(off[n] + 16));
  k_slot_gather<<<grid, 256, 0, s>>>(c->hdr.as<uint8_t>(), d_len.as<uint32_t>(), d_src.as<uint64_t>(), d_off.as<uint64_t>(), n, d_out.as<uint8_t>(), d_present.as<uint8_t>());
  FEI_CUDA(cudaMemcpyAsync(present, d_present.p, n, cudaMemcpyDeviceToHost, s));
  const bool fits = blob && off[n] <= blob_cap;
  if (fits && off[n]) FEI_CUDA(cudaMemcpyAsync(blob, d_out.p, off[n], cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  FEI_CUDA(cudaGetLastError());
  if (!fits) { set_error("value buffer too small: need %llu bytes", (unsigned long long)off[n]); return FEI_E_CAPACITY; }
  return FEI_OK;
}

/* Aux column k (0 .. FEI_MAX_AUX-1): one verdict byte per record, read by FEI_C_RECBITS conditions of later scans.  n must be the
 * corpus' record count; bytes == NULL drops the column.                                                                         */
extern "C" int fei_corpus_set_aux(fei_corpus* c, uint32_t k, const uint8_t* bytes, uint64_t n) {
  if (!c || k >= FEI_MAX_AUX) { set_error("bad argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_ready());
  if (!bytes) { c->aux[k].release(); c->aux_n[k] = 0; return FEI_OK; }
  if (n != c->n) { set_error("aux column has %llu entries, the corpus %llu records", (unsigned long long)n, (unsigned long long)c->n); return FEI_E_BADARG; }
  cudaStream_t s = ctx().stream;
  FEI_TRY(c->aux[k].ensure(n + 16));
  if (n) FEI_CUDA(cudaMemcpyAsync(c->aux[k].p, bytes, n, cudaMemcpyHostToDevice, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  c->aux_n[k] = n;
  return FEI_OK;
}

// ---------------------------------------------------------------- bulk tag edit (MemdirFolderManager.bulk_tag_folder)
// folders.py:483-587, per record of the selected directories:
//     existing = [t.strip() for t in headers["Tags"].split(",")] if "Tags" in headers else []
//     updated  = existing + [t for t in tags if t not in existing]    (add)
//              | [t for t in existing if t not in tags]              (remove)
//              | tags                                                (replace)
//     affected iff sorted(existing) != sorted(updated); it reports Subject, ", ".join(existing) and ", ".join(updated)
// k_tag_edit_measure decides every selected record (one thread each; Tags = slot 0 and Subject = slot 1 of the program, exact
// keys) and sizes its three strings; two exclusive scans place the affected records and their bytes; k_tag_edit_write writes
// them.  Nothing else of a record leaves the device: the file rewrite is the host's, for the affected records only.
namespace fei {
constexpr uint32_t kTagOpsMax = 64, kTagBytesMax = 4096;
struct TagOps {                                   // the operands, staged in shared memory by every CTA
  uint32_t op, n_tags, n_dist, pad;
  uint32_t off[kTagOpsMax + 1];                   // operand k = bytes[off[k] .. off[k+1])
  uint16_t dist[kTagOpsMax], mult[kTagOpsMax];    // replace: each distinct operand (its first index) and how often it occurs
  uint8_t bytes[kTagBytesMax];
};
static_assert(sizeof(TagOps) % 4 == 0, "TagOps is staged word by word");

struct TagEditArgs {
  const uint8_t* prog; const uint8_t* hdr; const uint64_t* hdr_off; const uint2* hdir; const uint64_t* hdir_off;
  const uint32_t* key_lut; const uint32_t* alive; uint64_t n; const TagOps* ops;
};
struct TagRecord { const uint8_t* tags; const uint8_t* subj; uint32_t tags_len, subj_len; bool has_tags, has_subj; };
// A record's header lines with the key masks shifted by `slot`: header_lookup<1> then reads program slot `slot` (one lookup per
// field keeps the value arrays of header_lookup in registers).
template <class Lines>
struct SlotLines : Lines {
  uint32_t slot;
  __device__ __forceinline__ uint32_t key_mask() const { return Lines::key_mask() >> slot; }
};

__device__ __forceinline__ TagRecord tag_record(const TagEditArgs& a, uint64_t rec) {
  const fei_prog_hdr* ph = reinterpret_cast<const fei_prog_hdr*>(a.prog);
  const uint8_t* h = a.hdr + a.hdr_off[rec];
  const uint2* ent = a.hdir + a.hdir_off[rec];
  const uint32_t n_ent = (uint32_t)(a.hdir_off[rec + 1] - a.hdir_off[rec]);
  const bool text = text_record(ent, n_ent);
  auto mode = [](int) { return 1u; };                           // exact keys, the last line wins
  auto lookup = [&](uint32_t slot, uint32_t* voff, uint32_t* vlen) {
    return text ? header_lookup<1>(SlotLines<TextLines>{{h, h, a.hdr + a.hdr_off[rec + 1], a.prog, ph->off_key_dfa, false}, slot}, mode, voff, vlen, no_values)
                : header_lookup<1>(SlotLines<DirLines>{{ent, n_ent, a.key_lut}, slot}, mode, voff, vlen, no_values);
  };
  uint32_t toff = 0, tlen = 0, soff = 0, slen = 0;
  const bool has_tags = lookup(0, &toff, &tlen) != 0, has_subj = lookup(1, &soff, &slen) != 0;
  return TagRecord{h + toff, h + soff, tlen, slen, has_tags, has_subj};
}

// str.split(",") of a value, every piece strip()ped: f(piece, length) for each until it returns true (then true)
template <class F>
__device__ __forceinline__ bool any_piece(const uint8_t* v, uint32_t len, F f) {
  for (uint32_t pos = 0;;) {
    uint32_t end = pos;
    while (end < len && v[end] != ',') ++end;
    const uint8_t* p = v + pos; const uint8_t* e = v + end;
    strip_span(p, e);
    if (f(p, (uint32_t)(e - p))) return true;
    if (end >= len) return false;
    pos = end + 1;
  }
}
__device__ __forceinline__ bool same_bytes(const uint8_t* p, uint32_t lp, const uint8_t* q, uint32_t lq) {
  if (lp != lq) return false;
  for (uint32_t k = 0; k < lp; ++k) if (p[k] != q[k]) return false;
  return true;
}
__device__ __forceinline__ bool in_existing(const TagRecord& r, const uint8_t* p, uint32_t l) {
  return r.has_tags && any_piece(r.tags, r.tags_len, [&](const uint8_t* q, uint32_t lq) { return same_bytes(p, l, q, lq); });
}
__device__ __forceinline__ bool in_operands(const TagOps& o, const uint8_t* p, uint32_t l) {
  for (uint32_t k = 0; k < o.n_tags; ++k) if (same_bytes(p, l, o.bytes + o.off[k], o.off[k + 1] - o.off[k])) return true;
  return false;
}

// sorted(existing) != sorted(updated)
__device__ __forceinline__ bool tag_edit_changes(const TagOps& o, const TagRecord& r) {
  if (o.op == 0) {                                               // add: some operand is not among the pieces
    for (uint32_t k = 0; k < o.n_tags; ++k) if (!in_existing(r, o.bytes + o.off[k], o.off[k + 1] - o.off[k])) return true;
    return false;
  }
  if (o.op == 1)                                                 // remove: some piece is an operand
    return r.has_tags && any_piece(r.tags, r.tags_len, [&](const uint8_t* p, uint32_t l) { return in_operands(o, p, l); });
  uint32_t pieces = 0;                                           // replace: the multisets differ
  if (r.has_tags) any_piece(r.tags, r.tags_len, [&](const uint8_t*, uint32_t) { ++pieces; return false; });
  if (pieces != o.n_tags) return true;
  for (uint32_t d = 0; d < o.n_dist; ++d) {                      // equal sizes: equal iff every distinct operand occurs as often
    const uint8_t* t = o.bytes + o.off[o.dist[d]];
    const uint32_t lt = o.off[o.dist[d] + 1] - o.off[o.dist[d]];
    uint32_t cnt = 0;
    any_piece(r.tags, r.tags_len, [&](const uint8_t* p, uint32_t l) { cnt += same_bytes(p, l, t, lt) ? 1u : 0u; return false; });
    if (cnt != o.mult[d]) return true;
  }
  return false;
}

template <class Sink>
struct Joiner {                                                  // ", ".join
  Sink& s; bool first = true;
  __device__ void put(const uint8_t* p, uint32_t l) {
    if (!first) { const uint8_t sep[2] = {',', ' '}; s.put(sep, 2); }
    first = false; s.put(p, l);
  }
};
template <class Sink>
__device__ __forceinline__ void emit_old_tags(Sink& s, const TagRecord& r) {
  Joiner<Sink> j{s};
  if (r.has_tags) any_piece(r.tags, r.tags_len, [&](const uint8_t* p, uint32_t l) { j.put(p, l); return false; });
}
template <class Sink>
__device__ __forceinline__ void emit_new_tags(Sink& s, const TagOps& o, const TagRecord& r) {
  Joiner<Sink> j{s};
  if (o.op != 2 && r.has_tags)                                   // add keeps every piece, remove those that are not operands
    any_piece(r.tags, r.tags_len, [&](const uint8_t* p, uint32_t l) { if (o.op == 0 || !in_operands(o, p, l)) j.put(p, l); return false; });
  if (o.op == 1) return;
  for (uint32_t k = 0; k < o.n_tags; ++k) {                      // add: the operands not among the pieces; replace: all of them
    const uint8_t* t = o.bytes + o.off[k];
    const uint32_t lt = o.off[k + 1] - o.off[k];
    if (o.op == 2 || !in_existing(r, t, lt)) j.put(t, lt);
  }
}

__device__ __forceinline__ void stage_tag_ops(const TagOps* g, TagOps& s) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(g);
  uint32_t* dst = reinterpret_cast<uint32_t*>(&s);
  for (uint32_t k = threadIdx.x; k < sizeof(TagOps) / 4; k += blockDim.x) dst[k] = src[k];
  __syncthreads();
}

__global__ void __launch_bounds__(256) k_tag_edit_measure(TagEditArgs a, uint32_t* __restrict__ changed, uint32_t* __restrict__ bytes) {
  __shared__ TagOps ops;
  stage_tag_ops(a.ops, ops);
  const uint64_t rec = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (rec >= a.n) return;
  uint32_t hit = 0, len = 0;
  if (a.alive[rec] & 1u) {
    const TagRecord r = tag_record(a, rec);
    if (tag_edit_changes(ops, r)) {
      CountSink cs;
      emit_old_tags(cs, r);
      emit_new_tags(cs, ops, r);
      hit = 1; len = cs.n + (r.has_subj ? r.subj_len : 0u);
    }
  }
  changed[rec] = hit; bytes[rec] = len;
}

__global__ void __launch_bounds__(256) k_tag_edit_write(TagEditArgs a, const uint32_t* __restrict__ changed, const uint64_t* __restrict__ pos,
                                                        const uint64_t* __restrict__ off, uint64_t global_base, uint64_t* __restrict__ rec_out,
                                                        uint64_t* __restrict__ text_off, uint8_t* __restrict__ has_subject, uint8_t* __restrict__ text) {
  __shared__ TagOps ops;
  stage_tag_ops(a.ops, ops);
  const uint64_t rec = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (rec >= a.n || !changed[rec]) return;
  const TagRecord r = tag_record(a, rec);
  const uint64_t j = pos[rec], o = off[rec];
  WriteSink s{text + o};
  if (r.has_subj) s.put(r.subj, r.subj_len);
  text_off[3 * j] = o;
  text_off[3 * j + 1] = o + (uint64_t)(s.p - (text + o));
  emit_old_tags(s, r);
  text_off[3 * j + 2] = o + (uint64_t)(s.p - (text + o));
  emit_new_tags(s, ops, r);
  rec_out[j] = rec + global_base;
  has_subject[j] = r.has_subj ? 1 : 0;
}
}  // namespace fei

extern "C" int fei_corpus_tag_edit(fei_corpus* c, const uint8_t* prog, uint64_t prog_len, uint32_t op,
                                   const uint8_t* tags, const uint64_t* tags_off, uint32_t n_tags,
                                   uint64_t* rec, uint64_t cap, uint64_t* n_changed,
                                   uint8_t* text, uint64_t text_cap, uint64_t* text_off, uint8_t* has_subject) {
  if (!c || !prog || !n_changed || !text_off || (n_tags && (!tags || !tags_off))) { set_error("null argument"); return FEI_E_BADARG; }
  if (op > 2) { set_error("unknown tag operation %u (0 add, 1 remove, 2 replace)", op); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  *n_changed = 0; text_off[0] = 0;
  const uint64_t op_bytes = n_tags ? tags_off[n_tags] - tags_off[0] : 0;
  if (n_tags > kTagOpsMax || op_bytes > kTagBytesMax) {
    set_error("%u tags of %llu bytes: a tag edit takes at most %u tags of %u bytes in all", n_tags, (unsigned long long)op_bytes, kTagOpsMax, kTagBytesMax);
    return FEI_E_UNSUPPORTED;
  }
  TagOps ops;
  memset(&ops, 0, sizeof(ops));
  ops.op = op; ops.n_tags = n_tags;
  for (uint32_t k = 0; k <= n_tags; ++k) ops.off[k] = n_tags ? (uint32_t)(tags_off[k] - tags_off[0]) : 0u;
  if (op_bytes) memcpy(ops.bytes, tags + tags_off[0], op_bytes);
  for (uint32_t k = 0; k < n_tags; ++k) {                        // the multiset of the operands, for replace
    uint32_t d = 0;
    while (d < ops.n_dist && !(ops.off[ops.dist[d] + 1] - ops.off[ops.dist[d]] == ops.off[k + 1] - ops.off[k] &&
                               !memcmp(ops.bytes + ops.off[ops.dist[d]], ops.bytes + ops.off[k], ops.off[k + 1] - ops.off[k]))) ++d;
    if (d == ops.n_dist) { ops.dist[d] = (uint16_t)k; ops.mult[d] = 0; ++ops.n_dist; }
    ++ops.mult[d];
  }
  FEI_TRY(run_scan(c, prog, prog_len, kCompactNone, nullptr));
  fei_prog_hdr h; memcpy(&h, prog, sizeof(h));
  if (h.n_queries != 1 || h.n_slots < 2) { set_error("a tag edit wants one query whose first two header fields are Tags and Subject"); return FEI_E_BADARG; }
  const uint64_t n = c->n;
  if (n == 0) return finish_timing(c, false);
  cudaStream_t s = ctx().stream;
  DevBuf d_ops, d_changed, d_bytes, d_pos, d_off;
  FEI_TRY(upload(d_ops, &ops, sizeof(ops), 0, s));
  FEI_TRY(d_changed.alloc(n * 4)); FEI_TRY(d_bytes.alloc(n * 4)); FEI_TRY(d_pos.alloc((n + 1) * 8)); FEI_TRY(d_off.alloc((n + 1) * 8));
  const TagEditArgs a{c->prog.as<uint8_t>(), c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), c->hdir.as<uint2>(), c->hdir_off.as<uint64_t>(),
                      c->key_lut.as<uint32_t>(), c->hits.as<uint32_t>(), n, d_ops.as<TagOps>()};
  const unsigned grid = (unsigned)((n + 255) / 256);
  k_tag_edit_measure<<<grid, 256, 0, s>>>(a, d_changed.as<uint32_t>(), d_bytes.as<uint32_t>());
  uint64_t count = 0, total = 0;
  FEI_TRY(queue_offsets(d_changed.as<uint32_t>(), n, d_pos.as<uint64_t>(), &count, false, c->scan_tmp, s));
  FEI_TRY(queue_offsets(d_bytes.as<uint32_t>(), n, d_off.as<uint64_t>(), &total, false, c->scan_tmp, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  if (count > cap || total > text_cap || (count && (!rec || !text || !has_subject))) {
    *n_changed = count; text_off[0] = total;
    set_error("tag edit buffers too small: need %llu records and %llu text bytes", (unsigned long long)count, (unsigned long long)total);
    return FEI_E_CAPACITY;
  }
  if (count) {
    DevBuf d_rec, d_toff, d_has, d_text;
    FEI_TRY(d_rec.alloc(count * 8)); FEI_TRY(d_toff.alloc(3 * count * 8)); FEI_TRY(d_has.alloc(count)); FEI_TRY(d_text.alloc(total + 16));
    k_tag_edit_write<<<grid, 256, 0, s>>>(a, d_changed.as<uint32_t>(), d_pos.as<uint64_t>(), d_off.as<uint64_t>(), c->global_base,
                                          d_rec.as<uint64_t>(), d_toff.as<uint64_t>(), d_has.as<uint8_t>(), d_text.as<uint8_t>());
    FEI_CUDA(cudaMemcpyAsync(rec, d_rec.p, count * 8, cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaMemcpyAsync(text_off, d_toff.p, 3 * count * 8, cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaMemcpyAsync(has_subject, d_has.p, count, cudaMemcpyDeviceToHost, s));
    if (total) FEI_CUDA(cudaMemcpyAsync(text, d_text.p, total, cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaStreamSynchronize(s));
    FEI_CUDA(cudaGetLastError());
  }
  text_off[3 * count] = total;
  *n_changed = count;
  return finish_timing(c, false);
}
