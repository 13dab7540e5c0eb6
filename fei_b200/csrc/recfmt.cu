// Record formatter: the text the Memdir command line prints for a listing (memdir_tools/cli.py, memdir_tools/search.py), written
// byte for byte on the GPU from the packed corpus, so that no per-record dict is built on the host.
//
// The dict every format reads is the one list_memories builds (utils.py:202-253): filename, folder, status, the headers dict of
// parse_memory_content (utils.py:113-118: a repeated key keeps its first position and its last value) and the metadata of
// parse_memory_filename (utils.py:74-95).  Formats (include/feiscan.h FEI_FMT_*):
//   JSON    one element of json.dumps(results, indent=2)           (cli.py:117-121, search.py:533-552)
//   CSV     one row of print_search_results' csv branch            (search.py:554-571)
//   COMPACT one line of its compact branch                          (search.py:573-582)
//   TEXT    print_memory (cli.py:41-67), optionally followed by the separator line the search commands print
// k_recfmt_measure sizes every record with put_record<CountSink>, an exclusive scan places them, k_recfmt_write writes them with
// put_record<WriteSink>: one thread per record, one source for both passes.
#include "corpus.h"
#include "pyws.cuh"
#include "datefmt.cuh"
#include "jsonfmt.cuh"

namespace fei {
using feijson::put_json_fsname;

struct RecFmtArgs {
  const uint64_t* idx; uint64_t m;                 // corpus-local records, in output order
  const uint8_t* hdr; const uint64_t* hdr_off;
  const uint8_t* name; const uint64_t* name_off; const uint16_t* name_spans;
  const int64_t* ts; const int64_t* wall; const uint64_t* flags8; const uint32_t* fsb;
  const uint8_t* body; const uint64_t* body_off;   // bodies of idx[0..m), un-tiled (FEI_FMT_CONTENT only)
  const uint8_t* folders; const uint64_t* folder_off; uint32_t n_folders;   // folder name of each packed folder id
  uint32_t fmt, opts;
};

struct Span { const uint8_t* p; uint32_t n; };

__device__ __forceinline__ bool same_span(const uint8_t* a, const uint8_t* ae, const uint8_t* b, const uint8_t* be) {
  if (ae - a != be - b) return false;
  for (; a < ae; ++a, ++b) if (*a != *b) return false;
  return true;
}

// The headers dict in its iteration order: f(key, value) once per distinct key, at its first line, with its last line's value.
template <class F>
__device__ __forceinline__ void for_each_header(const uint8_t* h, const uint8_t* end, F f) {
  HeaderLine l, e;
  for (const uint8_t* p = h; p < end;) {
    const uint8_t* line = p;
    if (!next_header_line(p, end, l)) continue;
    bool earlier = false;
    for (const uint8_t* q = h; q < line && !earlier;) earlier = next_header_line(q, line, e) && same_span(e.ka, e.kb, l.ka, l.kb);
    if (earlier) continue;
    const uint8_t *va = l.va, *vb = l.vb;
    for (const uint8_t* q = p; q < end;)
      if (next_header_line(q, end, e) && same_span(e.ka, e.kb, l.ka, l.kb)) { va = e.va; vb = e.vb; }
    f(Span{l.ka, (uint32_t)(l.kb - l.ka)}, Span{va, (uint32_t)(vb - va)});
  }
}
// headers.get(key): the value of the last line whose key is exactly `key`
__device__ __forceinline__ bool header_get(const uint8_t* h, const uint8_t* end, const char* key, Span& v) {
  uint32_t kl = 0;
  while (key[kl]) ++kl;
  bool found = false;
  HeaderLine l;
  for (const uint8_t* p = h; p < end;)
    if (next_header_line(p, end, l) && same_span(l.ka, l.kb, reinterpret_cast<const uint8_t*>(key), reinterpret_cast<const uint8_t*>(key) + kl)) {
      v = Span{l.va, (uint32_t)(l.vb - l.va)}; found = true;
    }
  return found;
}

template <class S> __device__ __forceinline__ void put_span(S& o, Span s) { put_bytes(o, s.p, s.n); }
template <class S> __device__ __forceinline__ void put_csv_doubled(S& o, Span s) {      // str.replace('"', '""')
  for (uint32_t k = 0; k < s.n; ++k) { o.put(s.p[k]); if (s.p[k] == '"') o.put('"'); }
}
// date.isoformat(), or date.strftime("%Y-%m-%d")
template <class S> __device__ __forceinline__ void put_datetime(S& o, int64_t wall, bool date_only) {
  civil_text(wall, 'T', date_only, [&](int, uint32_t c) { o.put((uint8_t)c); });
}
// str(int) of the file-name timestamp, most significant digit first (no digit buffer: it would live in local memory)
template <class S> __device__ __forceinline__ void put_decimal(S& o, uint64_t v) {
  uint64_t p = 1;
  while (v / p >= 10) p *= 10;
  for (; p; p /= 10) o.put((uint8_t)('0' + v / p % 10));
}
// memory["folder"] or "Inbox"
template <class S> __device__ __forceinline__ void put_folder_or_inbox(S& o, Span f) { if (f.n) put_span(o, f); else put_lit(o, "Inbox"); }

__device__ __forceinline__ const char* flag_name(uint32_t f) {        // FLAGS (utils.py:25-30)
  switch (f) { case 'S': return "Seen"; case 'R': return "Replied"; case 'F': return "Flagged"; case 'P': return "Priority"; default: return nullptr; }
}

template <class S>
__device__ __forceinline__ void put_record(S& o, const RecFmtArgs& a, uint64_t i) {
  const uint64_t r = a.idx[i];
  const Span name{a.name + a.name_off[r], (uint32_t)(a.name_off[r + 1] - a.name_off[r])};
  const uint16_t* sp = a.name_spans + 4 * r;
  const Span uid{name.p + sp[0], sp[1]}, host{name.p + sp[2], sp[3]};
  const uint32_t fsb = a.fsb[r], fid = fsb & 0xFFFFu, st = (fsb >> 16) & 0xFFu;
  const Span folder = fid < a.n_folders ? Span{a.folders + a.folder_off[fid], (uint32_t)(a.folder_off[fid + 1] - a.folder_off[fid])} : Span{nullptr, 0};
  const char* status = st == 0 ? "cur" : st == 1 ? "new" : "tmp";
  const uint64_t f8 = a.flags8[r];
  const uint32_t n_flags = (uint32_t)(f8 >> 56);
  const int64_t wall = a.wall[r];
  const uint8_t* h = a.hdr + a.hdr_off[r];
  const uint8_t* he = a.hdr + a.hdr_off[r + 1];
  const bool content = (a.opts & FEI_FMT_CONTENT) != 0;
  const Span body = content ? Span{a.body + a.body_off[i], (uint32_t)(a.body_off[i + 1] - a.body_off[i])} : Span{nullptr, 0};

  if (a.fmt == FEI_FMT_JSON) {
    put_lit(o, "  {\n    \"filename\": "); put_json_fsname(o, name.p, name.n);
    put_lit(o, ",\n    \"folder\": "); put_json_fsname(o, folder.p, folder.n);
    put_lit(o, ",\n    \"status\": \""); put_lit(o, status);
    put_lit(o, "\",\n    \"headers\": {");
    bool first = true;
    for_each_header(h, he, [&](Span k, Span v) {
      put_lit(o, first ? "\n      " : ",\n      "); first = false;
      put_json_fsname(o, k.p, k.n); put_lit(o, ": "); put_json_fsname(o, v.p, v.n);
    });
    put_lit(o, first ? "}" : "\n    }");
    put_lit(o, ",\n    \"metadata\": {\n      \"timestamp\": "); put_decimal(o, (uint64_t)a.ts[r]);
    put_lit(o, ",\n      \"unique_id\": "); put_json_fsname(o, uid.p, uid.n);
    put_lit(o, ",\n      \"hostname\": "); put_json_fsname(o, host.p, host.n);
    put_lit(o, ",\n      \"flags\": [");
    for (uint32_t k = 0; k < n_flags; ++k) {
      put_lit(o, k ? ",\n        \"" : "\n        \""); o.put((uint8_t)(f8 >> (8 * k))); o.put('"');
    }
    put_lit(o, n_flags ? "\n      ]" : "]");
    put_lit(o, ",\n      \"date\": \""); put_datetime(o, wall, false); put_lit(o, "\"\n    }");
    if (content) { put_lit(o, ",\n    \"content\": "); put_json_fsname(o, body.p, body.n); }
    put_lit(o, "\n  }");
    return;
  }
  if (a.fmt == FEI_FMT_CSV) {
    Span v{nullptr, 0};
    put_lit(o, "\""); put_span(o, uid);
    put_lit(o, "\",\""); if (header_get(h, he, "Subject", v)) put_csv_doubled(o, v);
    put_lit(o, "\",\""); put_datetime(o, wall, false);
    put_lit(o, "\",\""); put_folder_or_inbox(o, folder);
    put_lit(o, "\",\""); if (header_get(h, he, "Tags", v)) put_csv_doubled(o, v);
    put_lit(o, "\",\""); if (header_get(h, he, "Priority", v)) put_span(o, v);        // not doubled (search.py:567-568)
    put_lit(o, "\",\""); if (header_get(h, he, "Status", v)) put_span(o, v);
    put_lit(o, "\",\""); for (uint32_t k = 0; k < n_flags; ++k) o.put((uint8_t)(f8 >> (8 * k)));
    put_lit(o, "\"\n");
    return;
  }
  if (a.fmt == FEI_FMT_COMPACT) {
    Span v{nullptr, 0};
    put_span(o, uid); put_lit(o, " - "); put_datetime(o, wall, true); put_lit(o, " - ");
    if (header_get(h, he, "Subject", v)) put_span(o, v); else put_lit(o, "No subject");
    put_lit(o, " ("); put_folder_or_inbox(o, folder); put_lit(o, ") ");
    for (uint32_t k = 0; k < n_flags; ++k) o.put((uint8_t)(f8 >> (8 * k)));
    o.put('\n');
    return;
  }
  // FEI_FMT_TEXT: print_memory with COLORS / colorize (cli.py:26-67)
  put_lit(o, "\033[1mMemory ID: "); put_span(o, uid); put_lit(o, "\033[0m\nFile: "); put_span(o, name);
  put_lit(o, "\nDate: "); put_datetime(o, wall, false);
  put_lit(o, "\nFolder: "); put_folder_or_inbox(o, folder);
  put_lit(o, "\nStatus: "); put_lit(o, status);
  put_lit(o, "\nFlags: ");
  if (!n_flags) put_lit(o, "None");
  for (uint32_t k = 0; k < n_flags; ++k) {
    const uint32_t f = (uint32_t)(f8 >> (8 * k)) & 0xFFu;
    if (k) put_lit(o, ", ");
    if (const char* nm = flag_name(f)) put_lit(o, nm); else o.put((uint8_t)f);
  }
  put_lit(o, "\n\033[33m\nHeaders:\033[0m\n");
  for_each_header(h, he, [&](Span k, Span v) { put_lit(o, "  "); put_span(o, k); put_lit(o, ": "); put_span(o, v); o.put('\n'); });
  if (content) { put_lit(o, "\033[32m\nContent:\033[0m\n"); put_span(o, body); o.put('\n'); }
  o.put('\n');
  if (a.opts & FEI_FMT_SEPARATOR) put_lit(o, "----------------------------------\n");
}

__global__ void __launch_bounds__(128) k_recfmt_measure(RecFmtArgs a, uint32_t* __restrict__ len) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= a.m) return;
  CountSink c;
  put_record(c, a, i);
  len[i] = c.n;
}
__global__ void __launch_bounds__(128, 1) k_recfmt_write(RecFmtArgs a, const uint64_t* __restrict__ off, uint8_t* __restrict__ out) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= a.m) return;
  WriteSink w{out + off[i]};
  put_record(w, a, i);
}
}  // namespace fei

using namespace fei;

extern "C" int fei_corpus_format_records(fei_corpus* c, const uint64_t* idx, uint64_t m, uint32_t fmt, uint32_t opts,
                                         const uint8_t* folder_names, const uint64_t* folder_off, uint32_t n_folders,
                                         uint8_t* out, uint64_t out_cap, uint64_t* out_off, float* kernel_ms) {
  if (!c || (m && !idx) || !out_off || (n_folders && (!folder_names || !folder_off))) { set_error("null argument"); return FEI_E_BADARG; }
  if (fmt > FEI_FMT_TEXT || (opts & ~(uint32_t)(FEI_FMT_CONTENT | FEI_FMT_SEPARATOR))) { set_error("unknown format %u / options %#x", fmt, opts); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_loaded(c));
  out_off[0] = 0;
  if (kernel_ms) *kernel_ms = 0.f;
  if (m == 0) return FEI_OK;
  if (!c->name.p) { set_error("the corpus was loaded without file names"); return FEI_E_STATE; }
  FEI_TRY(check_record_indices(c, idx, m));
  cudaStream_t s = ctx().stream;
  DevBuf d_idx, d_fold, d_fold_off, d_boff, d_body, d_len, d_off, d_out;
  FEI_TRY(upload(d_idx, idx, m * 8, 0, s));
  FEI_TRY(upload(d_fold, folder_names, n_folders ? folder_off[n_folders] : 0, 0, s));
  FEI_TRY(upload(d_fold_off, folder_off, n_folders ? (n_folders + 1) * 8 : 0, 0, s));
  struct Events { cudaEvent_t e[2] = {nullptr, nullptr}; ~Events() { for (auto x : e) if (x) cudaEventDestroy(x); } } ev;
  for (auto& e : ev.e) FEI_CUDA(cudaEventCreate(&e));
  FEI_CUDA(cudaEventRecord(ev.e[0], s));
  if (opts & FEI_FMT_CONTENT) {
    uint64_t bytes = 0;
    FEI_TRY(fetch_offsets(c, d_idx.as<uint64_t>(), 0, m, nullptr, d_boff, nullptr, &bytes, false, s));
    FEI_TRY(untile_bodies(c, d_idx.as<uint64_t>(), 0, m, d_boff, bytes, d_body, s));
  }
  const RecFmtArgs a{d_idx.as<uint64_t>(), m, c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), c->name.as<uint8_t>(), c->name_off.as<uint64_t>(),
                     c->name_spans.as<uint16_t>(), c->ts.as<int64_t>(), c->wall.as<int64_t>(), c->flags8.as<uint64_t>(), c->fsb.as<uint32_t>(),
                     d_body.as<uint8_t>(), d_boff.as<uint64_t>(), d_fold.as<uint8_t>(), d_fold_off.as<uint64_t>(), n_folders, fmt, opts};
  FEI_TRY(d_len.alloc(m * 4)); FEI_TRY(d_off.alloc((m + 1) * 8));
  const unsigned grid = (unsigned)((m + 127) / 128);
  k_recfmt_measure<<<grid, 128, 0, s>>>(a, d_len.as<uint32_t>());
  FEI_TRY(queue_offsets(d_len.as<uint32_t>(), m, d_off.as<uint64_t>(), out_off, true, c->scan_tmp, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  FEI_CUDA(cudaGetLastError());
  const uint64_t total = out_off[m];
  if (!out || total > out_cap) { set_error("format buffer too small: need %llu bytes", (unsigned long long)total); return FEI_E_CAPACITY; }
  FEI_TRY(d_out.alloc(total + 16));
  k_recfmt_write<<<grid, 128, 0, s>>>(a, d_off.as<uint64_t>(), d_out.as<uint8_t>());
  FEI_CUDA(cudaEventRecord(ev.e[1], s));
  if (total) FEI_CUDA(cudaMemcpyAsync(out, d_out.p, total, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  FEI_CUDA(cudaGetLastError());
  if (kernel_ms) FEI_CUDA(cudaEventElapsedTime(kernel_ms, ev.e[0], ev.e[1]));
  return FEI_OK;
}
