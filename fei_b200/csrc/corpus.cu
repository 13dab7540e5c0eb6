// Packed corpus: upload / synthetic generation, body tiling ("pack once"), fetch.
// Replaces the per-query directory walk + parse of memdir_tools.utils.list_memories
// (memdir_tools/utils.py:202-253) with a one-time pack; see corpus.h for the layout.
#include "corpus.h"
#include "synth.cuh"
#include <vector>
#include <string.h>

namespace fei {

// ---------------------------------------------------------------- tiler
__global__ void k_units(const uint64_t* __restrict__ off, uint64_t n, uint32_t* __restrict__ len) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) len[i] = (uint32_t)(off[i + 1] - off[i]);
}

// One block per window of kWindow records: bitonic sort by (units desc, index asc), kWindow / kSortThreads keys per thread.
constexpr int kSortThreads = 1024;
__global__ void __launch_bounds__(kSortThreads)
k_window_sort(const uint32_t* __restrict__ len, uint64_t n, uint32_t* __restrict__ grp_rec, uint32_t* __restrict__ grp_len,
              uint32_t* __restrict__ grp_units, uint32_t* __restrict__ rec_pos) {
  __shared__ uint64_t key[kWindow];
  const uint64_t base = (uint64_t)blockIdx.x * kWindow;
  // key: bit 63 = real record, bits 62..32 = units, bits 31..0 = kWindow-1-index.
  // Larger key sorts first: real records, longer bodies, lower index.
  for (uint32_t t = threadIdx.x; t < kWindow; t += kSortThreads) {
    const uint64_t i = base + t;
    const uint32_t l = i < n ? len[i] : 0;
    key[t] = (i < n ? 1ull << 63 : 0ull) | ((uint64_t)((l + 15) >> 4) << 32) | (uint64_t)(kWindow - 1 - t);
  }
  __syncthreads();
  for (uint32_t k = 2; k <= kWindow; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t t = threadIdx.x; t < kWindow; t += kSortThreads) {
        const uint32_t p = t ^ j;
        if (p > t) {
          const uint64_t a = key[t], b = key[p];
          const bool desc = (t & k) == 0;                       // overall descending order
          if (desc ? a < b : a > b) { key[t] = b; key[p] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (uint32_t t = threadIdx.x; t < kWindow; t += kSortThreads) {       // t, t + 1024, ... keep warps on whole groups
    const uint64_t kk = key[t];
    const uint32_t idx = kWindow - 1 - (uint32_t)(kk & 0xFFFFFFFFu);
    const uint64_t rec = base + idx;
    const bool real = (kk >> 63) != 0;
    const uint32_t rl = real ? len[rec] : 0;
    const uint64_t pos = base + t;
    grp_rec[pos] = real ? (uint32_t)rec : kInvalidRec;
    grp_len[pos] = rl;
    if (real) rec_pos[rec] = (uint32_t)pos;
    uint32_t s = (rl + 15) >> 4;
    for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((t & 31) == 0) grp_units[pos >> 5] = s;
  }
}

__device__ __forceinline__ uint32_t mask_bytes(uint32_t w, int keep) {   // keep the low `keep` bytes (0..4)
  return keep >= 4 ? w : keep <= 0 ? 0u : (w & ((1u << (8 * keep)) - 1u));
}

// One warp per group: copy 16-byte units from the canonical blob into the ragged rows.
__global__ void k_tile_copy(const uint8_t* __restrict__ body, const uint64_t* __restrict__ body_off,
                            const uint32_t* __restrict__ grp_rec, const uint32_t* __restrict__ grp_len,
                            const uint64_t* __restrict__ grp_base, uint64_t n_groups, uint8_t* __restrict__ tiles) {
  uint64_t g = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (g >= n_groups) return;
  uint32_t rec = grp_rec[g * 32 + lane];
  uint32_t len = grp_len[g * 32 + lane];
  uint32_t units = (len + 15) >> 4;
  const uint8_t* src = rec != kInvalidRec ? body + body_off[rec] : body;
  uint8_t* row = tiles + grp_base[g] * 16;
  uint32_t maxu = __shfl_sync(0xffffffffu, units, 0);
  for (uint32_t k = 0; k < maxu; ++k) {
    uint32_t m = __popc(__ballot_sync(0xffffffffu, k < units));
    if (k < units) {
      uint4 v = load16(src + (uint64_t)k * 16);
      int rem = (int)len - (int)(k * 16);
      if (rem < 16) { v.x = mask_bytes(v.x, rem); v.y = mask_bytes(v.y, rem - 4); v.z = mask_bytes(v.z, rem - 8); v.w = mask_bytes(v.w, rem - 12); }
      v.x = tile_byte_perm4(v.x); v.y = tile_byte_perm4(v.y); v.z = tile_byte_perm4(v.z); v.w = tile_byte_perm4(v.w);
      *reinterpret_cast<uint4*>(row + lane * 16) = v;
    }
    row += (uint64_t)m * 16;
  }
}

// ---------------------------------------------------------------- fetch: record i of a fetch is idx[i], or first + i when idx is null
__global__ void k_rec_lens(const uint64_t* __restrict__ idx, uint64_t first, uint64_t m, const uint64_t* __restrict__ hdr_off,
                           const uint32_t* __restrict__ rec_pos, const uint32_t* __restrict__ grp_len, uint32_t* __restrict__ hlen,
                           uint32_t* __restrict__ blen) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint64_t r = idx ? idx[i] : first + i;
  hlen[i] = (uint32_t)(hdr_off[r + 1] - hdr_off[r]);
  blen[i] = grp_len[rec_pos[r]];
}
__global__ void k_copy_hdr(const uint64_t* __restrict__ idx, uint64_t m, const uint8_t* __restrict__ hdr, const uint64_t* __restrict__ hdr_off,
                           const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out) {
  const uint64_t i = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;       // a warp per record
  const int lane = threadIdx.x & 31;
  if (i >= m) return;
  const uint64_t r = idx[i];
  const uint8_t* p = hdr + hdr_off[r];
  const uint32_t len = (uint32_t)(hdr_off[r + 1] - hdr_off[r]);
  uint8_t* d = out + out_off[i];
  for (uint32_t k = lane; k < len; k += 32) d[k] = p[k];
}
// Inverse of the tiler: a thread per record copies its units back to a canonical blob.
__global__ void k_untile_idx(const uint8_t* __restrict__ tiles, const uint64_t* __restrict__ grp_base, const uint32_t* __restrict__ grp_len,
                             const uint32_t* __restrict__ rec_pos, const uint64_t* __restrict__ idx, uint64_t first, uint64_t m,
                             const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint32_t pos = rec_pos[idx ? idx[i] : first + i];
  const uint64_t g = pos >> 5; const int lane = pos & 31;
  const uint32_t len = grp_len[pos];
  const uint32_t* gl = grp_len + g * 32;
  uint8_t* dst = out + out_off[i];
  const uint8_t* gb = tiles + grp_base[g] * 16;
  uint32_t units[32];
  for (int l = 0; l < 32; ++l) units[l] = (gl[l] + 15) >> 4;
  for (uint32_t k = 0; k * 16 < len; ++k) {
    uint64_t before = 0;                                      // sum over lanes of min(units, k)
    for (int l = 0; l < 32; ++l) before += units[l] < k ? units[l] : k;
    const uint8_t* p = gb + before * 16 + lane * 16;
    const uint32_t cnt = len - k * 16 < 16 ? len - k * 16 : 16;
    for (uint32_t b = 0; b < cnt; ++b) dst[k * 16 + b] = tile_byte_unperm(p[b]);
  }
}

int fetch_offsets(fei_corpus* c, const uint64_t* d_idx, uint64_t first, uint64_t m, DevBuf* d_hoff, DevBuf& d_boff,
                  uint64_t* hdr_off, uint64_t* body_off, bool whole, cudaStream_t s) {
  DevBuf d_hlen, d_blen;
  FEI_TRY(d_hlen.alloc(m * 4)); FEI_TRY(d_blen.alloc(m * 4)); FEI_TRY(d_boff.alloc((m + 1) * 8));
  k_rec_lens<<<(unsigned)((m + 127) / 128), 128, 0, s>>>(d_idx, first, m, c->hdr_off.as<uint64_t>(), c->rec_pos.as<uint32_t>(), c->grp_len.as<uint32_t>(),
                                                         d_hlen.as<uint32_t>(), d_blen.as<uint32_t>());
  if (d_hoff) {
    FEI_TRY(d_hoff->alloc((m + 1) * 8));
    FEI_TRY(queue_offsets(d_hlen.as<uint32_t>(), m, d_hoff->as<uint64_t>(), hdr_off, whole, c->scan_tmp, s));
  }
  FEI_TRY(queue_offsets(d_blen.as<uint32_t>(), m, d_boff.as<uint64_t>(), body_off, whole, c->scan_tmp, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  return FEI_OK;
}

int untile_bodies(fei_corpus* c, const uint64_t* d_idx, uint64_t first, uint64_t m, const DevBuf& d_boff, uint64_t bytes, DevBuf& d_body,
                  cudaStream_t s) {
  FEI_TRY(d_body.alloc(bytes + 16));
  k_untile_idx<<<(unsigned)((m + 127) / 128), 128, 0, s>>>(c->tiles.as<uint8_t>(), c->grp_base.as<uint64_t>(), c->grp_len.as<uint32_t>(), c->rec_pos.as<uint32_t>(),
                                                           d_idx, first, m, d_boff.as<uint64_t>(), d_body.as<uint8_t>());
  FEI_CUDA(cudaGetLastError());
  return FEI_OK;
}

int corpus_load_events(fei_corpus* c) {
  for (auto& e : c->ev_load) if (!e) FEI_CUDA(cudaEventCreate(&e));
  return FEI_OK;
}
cudaStream_t corpus_load_stream(fei_corpus* c) {
  if (!c->load_stream && cudaStreamCreateWithFlags(&c->load_stream, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); c->load_stream = nullptr; }
  return c->load_stream ? c->load_stream : ctx().copy_stream;
}

static int build_tiles(fei_corpus* c, const uint8_t* d_body, const uint64_t* d_body_off, cudaStream_t s) {
  uint64_t n = c->n;
  uint64_t n_windows = (n + kWindow - 1) / kWindow;
  uint64_t n_groups = n_windows * (kWindow / 32);
  c->n_groups = n_groups;
  uint64_t slots = n_groups * 32;
  DevBuf& len = c->tmp_len; DevBuf& gunits = c->tmp_gunits;
  FEI_TRY(len.ensure((n ? n : 1) * sizeof(uint32_t)));
  FEI_TRY(gunits.ensure((n_groups ? n_groups : 1) * sizeof(uint32_t)));
  FEI_TRY(c->grp_rec.ensure((slots ? slots : 1) * sizeof(uint32_t)));
  FEI_TRY(c->grp_len.ensure((slots ? slots : 1) * sizeof(uint32_t)));
  FEI_TRY(c->rec_pos.ensure((n ? n : 1) * sizeof(uint32_t)));
  FEI_TRY(c->grp_base.ensure((n_groups + 1) * sizeof(uint64_t)));
  if (n == 0) { FEI_CUDA(cudaMemsetAsync(c->grp_base.p, 0, sizeof(uint64_t), s)); c->tile_bytes = 0; return FEI_OK; }
  k_units<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_body_off, n, len.as<uint32_t>());
  k_window_sort<<<(unsigned)n_windows, kSortThreads, 0, s>>>(len.as<uint32_t>(), n, c->grp_rec.as<uint32_t>(), c->grp_len.as<uint32_t>(),
                                                       gunits.as<uint32_t>(), c->rec_pos.as<uint32_t>());
  uint64_t total_units = 0;
  FEI_TRY(queue_offsets(gunits.as<uint32_t>(), n_groups, c->grp_base.as<uint64_t>(), &total_units, false, c->scan_tmp, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  c->tile_bytes = total_units * 16;
  FEI_TRY(c->tiles.ensure(c->tile_bytes + 64));
  unsigned blocks = (unsigned)((n_groups * 32 + 255) / 256);
  k_tile_copy<<<blocks, 256, 0, s>>>(d_body, d_body_off, c->grp_rec.as<uint32_t>(), c->grp_len.as<uint32_t>(),
                                     c->grp_base.as<uint64_t>(), n_groups, c->tiles.as<uint8_t>());
  FEI_CUDA(cudaGetLastError());
  FEI_CUDA(cudaStreamSynchronize(s));
  return FEI_OK;
}

// ---------------------------------------------------------------- synthetic corpus on the GPU
__global__ void k_synth_len(uint64_t seed, uint64_t first, uint64_t n, uint32_t* __restrict__ hlen, uint32_t* __restrict__ blen) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  CountSink ch; feisynth::gen_header(ch, seed, first + i);
  CountSink cb; feisynth::gen_body(cb, seed, first + i);
  hlen[i] = ch.n; blen[i] = cb.n;
}

__global__ void k_synth_write(uint64_t seed, uint64_t first, uint64_t n, const uint64_t* __restrict__ hoff, const uint64_t* __restrict__ boff,
                              uint8_t* __restrict__ hdr, uint8_t* __restrict__ body,
                              int64_t* __restrict__ ts, int64_t* __restrict__ wall, uint64_t* __restrict__ flags8, uint32_t* __restrict__ fsb) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  { WriteSink w{hdr + hoff[i]}; feisynth::gen_header(w, seed, first + i); }
  { WriteSink w{body + boff[i]}; feisynth::gen_body(w, seed, first + i); }
  feisynth::RecMeta m = feisynth::gen_meta(seed, first + i);
  ts[i] = m.ts; wall[i] = m.ts;                              // synthetic corpora live in UTC
  uint64_t f = 0;
  for (int k = 0; k < m.nflags; ++k) f |= (uint64_t)(uint8_t)m.flags[k] << (8 * k);
  flags8[i] = f | ((uint64_t)m.nflags << 56);
  fsb[i] = (uint32_t)m.folder | ((uint32_t)m.status << 16);
}

int check_load(uint64_t n, const fei_corpus_host* h) {
  FEI_TRY(require_ready());
  if (n >= 0xFFFFFFFFull) { set_error("at most 2^32-2 records per shard"); return FEI_E_BADARG; }
  if (h && n && (!h->ts || !h->wall || !h->flags8 || !h->fsb)) { set_error("missing meta array"); return FEI_E_BADARG; }
  return FEI_OK;
}

int require_loaded(const fei_corpus* c) {
  FEI_TRY(require_ready());
  if (!c || !c->loaded) { set_error("corpus not loaded"); return FEI_E_STATE; }
  return FEI_OK;
}

int check_record_indices(const fei_corpus* c, const uint64_t* idx, uint64_t m) {
  for (uint64_t i = 0; i < m; ++i) if (idx[i] >= c->n) { set_error("record index %llu out of range", (unsigned long long)idx[i]); return FEI_E_BADARG; }
  return FEI_OK;
}

int upload_meta(fei_corpus* c, const fei_corpus_host* h, cudaStream_t s) {
  const uint64_t n = h->n;
  FEI_TRY(upload(c->ts, h->ts, n * 8, 0, s)); FEI_TRY(upload(c->wall, h->wall, n * 8, 0, s));
  FEI_TRY(upload(c->flags8, h->flags8, n * 8, 0, s)); FEI_TRY(upload(c->fsb, h->fsb, n * 4, 0, s));
  if (h->name && h->name_off && h->name_spans && n) {
    c->name_bytes = h->name_off[n];
    FEI_TRY(upload(c->name, h->name, c->name_bytes, kBlobSlack, s));
    FEI_TRY(upload(c->name_off, h->name_off, (n + 1) * 8, 0, s));
    FEI_TRY(upload(c->name_spans, h->name_spans, n * 8, 0, s));
  } else { c->name.release(); c->name_off.release(); c->name_spans.release(); c->name_bytes = 0; }
  return FEI_OK;
}

// Once the tiles hold the text, the canonical staging text (body, its offsets and the raw file text of fei_corpus_load_raw) is
// kept for the next load while it is small, so that streamed batches reuse it without a cudaMalloc / cudaFree (a cudaFree
// synchronises the device), and dropped when the caller asks or when it passes 8 GiB, so that HBM holds one copy of a big
// resident corpus' text.  It goes before the header directory, which reads only hdr.
int pack_canonical(fei_corpus* c, DevBuf& body, DevBuf& body_off, cudaStream_t s, bool drop_text, cudaEvent_t packed) {
  FEI_TRY(build_tiles(c, body.as<uint8_t>(), body_off.as<uint64_t>(), s));
  drop_text = drop_text || body.bytes > (8ull << 30);
  if (drop_text) { body.release(); body_off.release(); c->stage_raw.release(); c->staged_text_bytes = ~0ull; }
  FEI_TRY(build_header_dir(c, s));
  if (packed) FEI_CUDA(cudaEventRecord(packed, s));
  if (drop_text) { c->tmp_len.release(); c->tmp_gunits.release(); }
  c->loaded = true;
  return FEI_OK;
}

}  // namespace fei

using namespace fei;

extern "C" int fei_corpus_create(fei_corpus** out) {
  if (!out) { set_error("null out"); return FEI_E_BADARG; }
  FEI_TRY(require_ready());
  fei_corpus* c = new fei_corpus();
  for (auto& e : c->ev) cudaEventCreate(&e);
  *out = c;
  return FEI_OK;
}

extern "C" int fei_corpus_destroy(fei_corpus* c) {
  if (!c) return FEI_OK;
  { std::lock_guard<std::mutex> lock(c->mu); }       // let a scan that another thread still runs on this handle finish
  cudaStreamSynchronize(ctx().stream);
  if (c->load_stream) { cudaStreamSynchronize(c->load_stream); cudaStreamDestroy(c->load_stream); }
  for (auto& e : c->ev_load) if (e) cudaEventDestroy(e);
  for (auto& e : c->ev) if (e) cudaEventDestroy(e);
  delete c;
  return FEI_OK;
}

extern "C" int fei_corpus_load(fei_corpus* c, const fei_corpus_host* h) {
  if (!c || !h) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(check_load(h->n, h));
  if (h->n && (!h->hdr_off || !h->body_off)) { set_error("missing corpus array"); return FEI_E_BADARG; }
  cudaStream_t s = corpus_load_stream(c);            // see fei_corpus_load_raw: loads overlap scans (and loads) of other handles
  uint64_t n = h->n;
  c->n = n; c->global_base = h->global_base; c->loaded = false;
  static const uint64_t zero_off[1] = {0};
  const uint64_t* hoff = n ? h->hdr_off : zero_off;
  const uint64_t* boff = n ? h->body_off : zero_off;
  if (hoff[0] != 0 || boff[0] != 0) { set_error("offset arrays must start at 0"); return FEI_E_BADARG; }
  for (uint64_t i = 0; i < n; ++i)
    if (boff[i + 1] - boff[i] > (32u << 20)) { set_error("record %llu: body larger than 32 MiB is not supported", (unsigned long long)i); return FEI_E_UNSUPPORTED; }
  c->hdr_bytes = hoff[n]; c->body_bytes = boff[n];
  FEI_CUDA(cudaEventRecord(c->ev[0], s));
  FEI_TRY(upload_meta(c, h, s));                     // the small arrays before the text, like fei_corpus_load_raw
  FEI_TRY(upload(c->hdr, h->hdr, c->hdr_bytes, kBlobSlack, s));
  FEI_TRY(upload(c->hdr_off, hoff, (n + 1) * 8, 0, s));
  FEI_TRY(upload(c->stage_body, h->body, c->body_bytes, kBlobSlack, s));
  FEI_TRY(upload(c->stage_body_off, boff, (n + 1) * 8, 0, s));
  FEI_CUDA(cudaEventRecord(c->ev[1], s));
  FEI_TRY(pack_canonical(c, c->stage_body, c->stage_body_off, s, false, nullptr));
  FEI_CUDA(cudaEventElapsedTime(&c->timing.h2d_ms, c->ev[0], c->ev[1]));
  return FEI_OK;
}

extern "C" int fei_corpus_synth(fei_corpus* c, uint64_t seed, uint64_t first, uint64_t n) {
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(check_load(n, nullptr));
  cudaStream_t s = ctx().stream;
  c->n = n; c->global_base = first; c->loaded = false;
  c->name.release(); c->name_off.release(); c->name_spans.release(); c->name_bytes = 0;
  DevBuf hlen, blen, body, body_off;
  uint64_t n1 = n ? n : 1;
  FEI_TRY(hlen.alloc(n1 * 4)); FEI_TRY(blen.alloc(n1 * 4));
  FEI_TRY(c->hdr_off.alloc((n + 1) * 8)); FEI_TRY(body_off.alloc((n + 1) * 8));
  FEI_TRY(c->ts.alloc(n1 * 8)); FEI_TRY(c->wall.alloc(n1 * 8)); FEI_TRY(c->flags8.alloc(n1 * 8)); FEI_TRY(c->fsb.alloc(n1 * 4));
  unsigned g = (unsigned)((n + 127) / 128);
  if (n) k_synth_len<<<g, 128, 0, s>>>(seed, first, n, hlen.as<uint32_t>(), blen.as<uint32_t>());
  uint64_t hb = 0, bb = 0;
  FEI_TRY(queue_offsets(hlen.as<uint32_t>(), n, c->hdr_off.as<uint64_t>(), &hb, false, c->scan_tmp, s));
  FEI_TRY(queue_offsets(blen.as<uint32_t>(), n, body_off.as<uint64_t>(), &bb, false, c->scan_tmp, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  hlen.release(); blen.release();
  c->hdr_bytes = hb; c->body_bytes = bb;
  FEI_TRY(c->hdr.alloc(hb + kBlobSlack)); FEI_TRY(body.alloc(bb + kBlobSlack));
  FEI_CUDA(cudaMemsetAsync((uint8_t*)c->hdr.p + hb, 0, kBlobSlack, s));
  FEI_CUDA(cudaMemsetAsync((uint8_t*)body.p + bb, 0, kBlobSlack, s));
  if (n) k_synth_write<<<g, 128, 0, s>>>(seed, first, n, c->hdr_off.as<uint64_t>(), body_off.as<uint64_t>(), c->hdr.as<uint8_t>(), body.as<uint8_t>(),
                                         c->ts.as<int64_t>(), c->wall.as<int64_t>(), c->flags8.as<uint64_t>(), c->fsb.as<uint32_t>());
  FEI_CUDA(cudaGetLastError());
  return pack_canonical(c, body, body_off, s, true, nullptr);
}

extern "C" int fei_corpus_stats_get(const fei_corpus* c, fei_corpus_stats* out) {
  if (!c || !out) { set_error("null argument"); return FEI_E_BADARG; }
  out->n = c->n; out->global_base = c->global_base;
  out->hdr_bytes = c->hdr_bytes; out->body_bytes = c->body_bytes; out->tile_bytes = c->tile_bytes; out->name_bytes = c->name_bytes;
  out->n_groups = c->n_groups;
  out->device_bytes = c->hdr.bytes + c->hdr_off.bytes + c->name.bytes + c->name_off.bytes + c->ts.bytes + c->wall.bytes + c->flags8.bytes + c->fsb.bytes +
                      c->tiles.bytes + c->grp_base.bytes + c->grp_rec.bytes + c->grp_len.bytes + c->rec_pos.bytes +
                      c->hdir.bytes + c->hdir_off.bytes + c->key_tag.bytes + c->key_rep.bytes + c->key_len.bytes + c->col_len.bytes + c->col_planes.bytes + c->kid_col.bytes;
  return FEI_OK;
}

extern "C" int fei_corpus_fetch(fei_corpus* c, uint64_t first, uint64_t n,
                                uint8_t* hdr, uint64_t hdr_cap, uint64_t* hdr_off,
                                uint8_t* body, uint64_t body_cap, uint64_t* body_off,
                                int64_t* ts, int64_t* wall, uint64_t* flags8, uint32_t* fsb) {
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_loaded(c));
  if (first + n > c->n) { set_error("range out of bounds"); return FEI_E_BADARG; }
  if (n == 0) return FEI_OK;
  cudaStream_t s = ctx().stream;
  uint64_t h0 = 0;
  std::vector<uint64_t> ho, bo;
  DevBuf d_hoff, d_boff, d_body;
  if (hdr || hdr_off || body || body_off) {          // not for the meta columns alone
    ho.resize(n + 1); bo.resize(n + 1);
    FEI_CUDA(cudaMemcpyAsync(&h0, c->hdr_off.as<uint64_t>() + first, 8, cudaMemcpyDeviceToHost, s));
    FEI_TRY(fetch_offsets(c, nullptr, first, n, &d_hoff, d_boff, ho.data(), bo.data(), true, s));
  }
  if (hdr_off) memcpy(hdr_off, ho.data(), (n + 1) * 8);
  if (hdr) {
    if (ho[n] > hdr_cap) { set_error("header buffer too small: need %llu", (unsigned long long)ho[n]); return FEI_E_CAPACITY; }
    FEI_CUDA(cudaMemcpyAsync(hdr, c->hdr.as<uint8_t>() + h0, ho[n], cudaMemcpyDeviceToHost, s));
  }
  if (ts) FEI_CUDA(cudaMemcpyAsync(ts, c->ts.as<int64_t>() + first, n * 8, cudaMemcpyDeviceToHost, s));
  if (wall) FEI_CUDA(cudaMemcpyAsync(wall, c->wall.as<int64_t>() + first, n * 8, cudaMemcpyDeviceToHost, s));
  if (flags8) FEI_CUDA(cudaMemcpyAsync(flags8, c->flags8.as<uint64_t>() + first, n * 8, cudaMemcpyDeviceToHost, s));
  if (fsb) FEI_CUDA(cudaMemcpyAsync(fsb, c->fsb.as<uint32_t>() + first, n * 4, cudaMemcpyDeviceToHost, s));
  if (body_off) memcpy(body_off, bo.data(), (n + 1) * 8);
  if (body) {
    if (bo[n] > body_cap) { set_error("body buffer too small: need %llu", (unsigned long long)bo[n]); return FEI_E_CAPACITY; }
    FEI_TRY(untile_bodies(c, nullptr, first, n, d_boff, bo[n], d_body, s));
    FEI_CUDA(cudaMemcpyAsync(body, d_body.p, bo[n], cudaMemcpyDeviceToHost, s));
  }
  FEI_CUDA(cudaStreamSynchronize(s));
  return FEI_OK;
}

/* Header text and body of the m records idx[0..m) (any order, repeats allowed), for materialising hits: hdr_off / body_off get
 * m + 1 offsets; FEI_E_CAPACITY (needed sizes in hdr_off[m] / body_off[m]) when a blob is too small.  hdr / body may be NULL to
 * only size the buffers.                                                                                                         */
extern "C" int fei_corpus_fetch_records(fei_corpus* c, const uint64_t* idx, uint64_t m, uint8_t* hdr, uint64_t hdr_cap, uint64_t* hdr_off,
                                        uint8_t* body, uint64_t body_cap, uint64_t* body_off) {
  if (!c || (m && !idx) || !hdr_off || !body_off) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_loaded(c));
  hdr_off[0] = 0; body_off[0] = 0;
  if (m == 0) return FEI_OK;
  FEI_TRY(check_record_indices(c, idx, m));
  cudaStream_t s = ctx().stream;
  DevBuf d_idx, d_hoff, d_boff, d_h, d_body;
  FEI_TRY(d_idx.alloc(m * 8));
  FEI_CUDA(cudaMemcpyAsync(d_idx.p, idx, m * 8, cudaMemcpyHostToDevice, s));
  FEI_TRY(fetch_offsets(c, d_idx.as<uint64_t>(), 0, m, &d_hoff, d_boff, hdr_off, body_off, true, s));
  if ((hdr && hdr_off[m] > hdr_cap) || (body && body_off[m] > body_cap)) { set_error("fetch buffers too small: need %llu header and %llu body bytes", (unsigned long long)hdr_off[m], (unsigned long long)body_off[m]); return FEI_E_CAPACITY; }
  if (hdr && hdr_off[m]) {
    FEI_TRY(d_h.alloc(hdr_off[m] + 16));
    k_copy_hdr<<<(unsigned)((m * 32 + 255) / 256), 256, 0, s>>>(d_idx.as<uint64_t>(), m, c->hdr.as<uint8_t>(), c->hdr_off.as<uint64_t>(), d_hoff.as<uint64_t>(), d_h.as<uint8_t>());
    FEI_CUDA(cudaMemcpyAsync(hdr, d_h.p, hdr_off[m], cudaMemcpyDeviceToHost, s));
  }
  if (body && body_off[m]) {
    FEI_TRY(untile_bodies(c, d_idx.as<uint64_t>(), 0, m, d_boff, body_off[m], d_body, s));
    FEI_CUDA(cudaMemcpyAsync(body, d_body.p, body_off[m], cudaMemcpyDeviceToHost, s));
  }
  FEI_CUDA(cudaStreamSynchronize(s));
  FEI_CUDA(cudaGetLastError());
  return FEI_OK;
}
