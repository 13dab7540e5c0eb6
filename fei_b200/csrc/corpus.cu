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

__device__ __forceinline__ uint4 load16_unaligned(const uint8_t* s) {
  // assemble 16 bytes from 4-byte aligned loads (the blob has >= 32 bytes of slack at the end)
  uintptr_t a = reinterpret_cast<uintptr_t>(s);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  uint32_t sh = (uint32_t)(a & 3) * 8;
  uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = sh ? w[4] : 0;
  uint4 r;
  r.x = __funnelshift_r(w0, w1, sh); r.y = __funnelshift_r(w1, w2, sh);
  r.z = __funnelshift_r(w2, w3, sh); r.w = __funnelshift_r(w3, w4, sh);
  return r;
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
      uint4 v = load16_unaligned(src + (uint64_t)k * 16);
      int rem = (int)len - (int)(k * 16);
      if (rem < 16) { v.x = mask_bytes(v.x, rem); v.y = mask_bytes(v.y, rem - 4); v.z = mask_bytes(v.z, rem - 8); v.w = mask_bytes(v.w, rem - 12); }
      v.x = tile_byte_perm4(v.x); v.y = tile_byte_perm4(v.y); v.z = tile_byte_perm4(v.z); v.w = tile_byte_perm4(v.w);
      *reinterpret_cast<uint4*>(row + lane * 16) = v;
    }
    row += (uint64_t)m * 16;
  }
}

// Inverse (fetch / debugging): thread per record copies its units back to a canonical blob.
__global__ void k_untile(const uint8_t* __restrict__ tiles, const uint64_t* __restrict__ grp_base,
                         const uint32_t* __restrict__ grp_len, const uint32_t* __restrict__ rec_pos,
                         uint64_t first, uint64_t n, const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t pos = rec_pos[first + i];
  uint64_t g = pos >> 5; int lane = pos & 31;
  uint32_t len = grp_len[pos];
  const uint32_t* gl = grp_len + g * 32;
  uint8_t* dst = out + out_off[i];
  const uint8_t* gb = tiles + grp_base[g] * 16;
  for (uint32_t k = 0; k * 16 < len; ++k) {
    uint64_t before = 0;                                      // sum over lanes of min(units, k)
    for (int l = 0; l < 32; ++l) { uint32_t u = (gl[l] + 15) >> 4; before += u < k ? u : k; }
    const uint8_t* p = gb + before * 16 + lane * 16;
    uint32_t cnt = len - k * 16 < 16 ? len - k * 16 : 16;
    for (uint32_t b = 0; b < cnt; ++b) { uint8_t t = p[b]; dst[k * 16 + b] = (uint8_t)(t ^ ((t >> 1) & 0x20)); }   // undo the tile byte permutation
  }
}

int corpus_load_events(fei_corpus* c) {
  for (auto& e : c->ev_load) if (!e) FEI_CUDA(cudaEventCreate(&e));
  return FEI_OK;
}
cudaStream_t corpus_load_stream(fei_corpus* c) {
  if (!c->load_stream && cudaStreamCreateWithFlags(&c->load_stream, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); c->load_stream = nullptr; }
  return c->load_stream ? c->load_stream : ctx().copy_stream;
}

int build_tiles(fei_corpus* c, const uint8_t* d_body, const uint64_t* d_body_off, cudaStream_t s) {
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
  FEI_TRY(exclusive_scan_u32_u64(gunits.as<uint32_t>(), n_groups, c->grp_base.as<uint64_t>(), c->scan_tmp, s));
  uint64_t total_units = 0;
  FEI_CUDA(cudaMemcpyAsync(&total_units, c->grp_base.as<uint64_t>() + n_groups, 8, cudaMemcpyDeviceToHost, s));
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
  feisynth::CountSink ch; feisynth::gen_header(ch, seed, first + i);
  feisynth::CountSink cb; feisynth::gen_body(cb, seed, first + i);
  hlen[i] = ch.n; blen[i] = cb.n;
}

__global__ void k_synth_write(uint64_t seed, uint64_t first, uint64_t n, const uint64_t* __restrict__ hoff, const uint64_t* __restrict__ boff,
                              uint8_t* __restrict__ hdr, uint8_t* __restrict__ body,
                              int64_t* __restrict__ ts, int64_t* __restrict__ wall, uint64_t* __restrict__ flags8, uint32_t* __restrict__ fsb) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  { feisynth::WriteSink w(hdr + hoff[i]); feisynth::gen_header(w, seed, first + i); }
  { feisynth::WriteSink w(body + boff[i]); feisynth::gen_body(w, seed, first + i); }
  feisynth::RecMeta m = feisynth::gen_meta(seed, first + i);
  ts[i] = m.ts; wall[i] = m.ts;                              // synthetic corpora live in UTC
  uint64_t f = 0;
  for (int k = 0; k < m.nflags; ++k) f |= (uint64_t)(uint8_t)m.flags[k] << (8 * k);
  flags8[i] = f | ((uint64_t)m.nflags << 56);
  fsb[i] = (uint32_t)m.folder | ((uint32_t)m.status << 16);
}

static int upload(DevBuf& b, const void* src, size_t bytes, size_t slack, cudaStream_t s) {
  FEI_TRY(b.ensure(bytes + slack + 16));
  if (bytes) FEI_CUDA(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, s));
  if (slack) FEI_CUDA(cudaMemsetAsync((uint8_t*)b.p + bytes, 0, slack, s));
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
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_ready());
  if (!c || !h) { set_error("null argument"); return FEI_E_BADARG; }
  if (h->n >= 0xFFFFFFFFull) { set_error("at most 2^32-2 records per shard"); return FEI_E_BADARG; }
  if (h->n && (!h->hdr_off || !h->body_off || !h->ts || !h->wall || !h->flags8 || !h->fsb)) { set_error("missing corpus array"); return FEI_E_BADARG; }
  Context& cx = ctx();
  cudaStream_t s = corpus_load_stream(c);            // see fei_corpus_load_raw: loads overlap scans (and loads) of other handles
  uint64_t n = h->n;
  c->n = n; c->global_base = h->global_base; c->loaded = false;
  static const uint64_t zero_off[1] = {0};
  const uint64_t* hoff = n ? h->hdr_off : zero_off;
  const uint64_t* boff = n ? h->body_off : zero_off;
  if (hoff[0] != 0 || boff[0] != 0) { set_error("offset arrays must start at 0"); return FEI_E_BADARG; }
  c->hdr_bytes = hoff[n]; c->body_bytes = boff[n];
  FEI_CUDA(cudaEventRecord(c->ev[0], s));
  FEI_TRY(upload(c->hdr, h->hdr, c->hdr_bytes, 32, s));
  FEI_TRY(upload(c->hdr_off, hoff, (n + 1) * 8, 0, s));
  FEI_TRY(upload(c->ts, h->ts, n * 8, 0, s));
  FEI_TRY(upload(c->wall, h->wall, n * 8, 0, s));
  FEI_TRY(upload(c->flags8, h->flags8, n * 8, 0, s));
  FEI_TRY(upload(c->fsb, h->fsb, n * 4, 0, s));
  if (h->name && h->name_off && h->name_spans && n) {
    c->name_bytes = h->name_off[n];
    FEI_TRY(upload(c->name, h->name, c->name_bytes, 32, s));
    FEI_TRY(upload(c->name_off, h->name_off, (n + 1) * 8, 0, s));
    FEI_TRY(upload(c->name_spans, h->name_spans, n * 8, 0, s));
  } else { c->name.release(); c->name_off.release(); c->name_spans.release(); c->name_bytes = 0; }
  for (uint64_t i = 0; i < n; ++i)
    if (boff[i + 1] - boff[i] > (32u << 20)) { set_error("record %llu: body larger than 32 MiB is not supported", (unsigned long long)i); return FEI_E_UNSUPPORTED; }
  DevBuf& body = c->stage_body; DevBuf& body_off = c->stage_body_off;
  FEI_TRY(upload(body, h->body, c->body_bytes, 32, s));
  FEI_TRY(upload(body_off, boff, (n + 1) * 8, 0, s));
  FEI_CUDA(cudaEventRecord(c->ev[1], s));
  FEI_TRY(build_tiles(c, body.as<uint8_t>(), body_off.as<uint64_t>(), s));
  FEI_TRY(build_header_dir(c, s));
  // the canonical body is only a staging area: keep it for the next batch when it is small (streaming
  // loads of host batches), drop it for big resident corpora so HBM holds one copy of the text
  if (body.bytes > (8ull << 30)) { body.release(); body_off.release(); c->tmp_len.release(); c->tmp_gunits.release(); }
  FEI_CUDA(cudaEventElapsedTime(&c->timing.h2d_ms, c->ev[0], c->ev[1]));
  c->loaded = true;
  return FEI_OK;
}

extern "C" int fei_corpus_synth(fei_corpus* c, uint64_t seed, uint64_t first, uint64_t n) {
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_ready());
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  if (n >= 0xFFFFFFFFull) { set_error("at most 2^32-2 records per shard"); return FEI_E_BADARG; }
  Context& cx = ctx();
  cudaStream_t s = cx.stream;
  c->n = n; c->global_base = first; c->loaded = false;
  c->name.release(); c->name_off.release(); c->name_spans.release(); c->name_bytes = 0;
  DevBuf hlen, blen, body, body_off;
  uint64_t n1 = n ? n : 1;
  FEI_TRY(hlen.alloc(n1 * 4)); FEI_TRY(blen.alloc(n1 * 4));
  FEI_TRY(c->hdr_off.alloc((n + 1) * 8)); FEI_TRY(body_off.alloc((n + 1) * 8));
  FEI_TRY(c->ts.alloc(n1 * 8)); FEI_TRY(c->wall.alloc(n1 * 8)); FEI_TRY(c->flags8.alloc(n1 * 8)); FEI_TRY(c->fsb.alloc(n1 * 4));
  unsigned g = (unsigned)((n + 127) / 128);
  if (n) k_synth_len<<<g, 128, 0, s>>>(seed, first, n, hlen.as<uint32_t>(), blen.as<uint32_t>());
  FEI_TRY(exclusive_scan_u32_u64(hlen.as<uint32_t>(), n, c->hdr_off.as<uint64_t>(), c->scan_tmp, s));
  FEI_TRY(exclusive_scan_u32_u64(blen.as<uint32_t>(), n, body_off.as<uint64_t>(), c->scan_tmp, s));
  uint64_t hb = 0, bb = 0;
  FEI_CUDA(cudaMemcpyAsync(&hb, c->hdr_off.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaMemcpyAsync(&bb, body_off.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  c->hdr_bytes = hb; c->body_bytes = bb;
  FEI_TRY(c->hdr.alloc(hb + 48)); FEI_TRY(body.alloc(bb + 48));
  FEI_CUDA(cudaMemsetAsync((uint8_t*)c->hdr.p + hb, 0, 48, s));
  FEI_CUDA(cudaMemsetAsync((uint8_t*)body.p + bb, 0, 48, s));
  if (n) k_synth_write<<<g, 128, 0, s>>>(seed, first, n, c->hdr_off.as<uint64_t>(), body_off.as<uint64_t>(), c->hdr.as<uint8_t>(), body.as<uint8_t>(),
                                         c->ts.as<int64_t>(), c->wall.as<int64_t>(), c->flags8.as<uint64_t>(), c->fsb.as<uint32_t>());
  FEI_CUDA(cudaGetLastError());
  FEI_TRY(build_tiles(c, body.as<uint8_t>(), body_off.as<uint64_t>(), s));
  body.release(); body_off.release(); hlen.release(); blen.release();   // the tiles hold the text now; free it before the header directory
  FEI_TRY(build_header_dir(c, s));
  c->loaded = true;
  return FEI_OK;
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
  FEI_TRY(require_ready());
  if (!c || !c->loaded) { set_error("corpus not loaded"); return FEI_E_STATE; }
  if (first + n > c->n) { set_error("range out of bounds"); return FEI_E_BADARG; }
  if (n == 0) return FEI_OK;
  cudaStream_t s = ctx().stream;
  std::vector<uint64_t> ho(n + 1);
  FEI_CUDA(cudaMemcpyAsync(ho.data(), c->hdr_off.as<uint64_t>() + first, (n + 1) * 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  if (hdr_off) for (uint64_t i = 0; i <= n; ++i) hdr_off[i] = ho[i] - ho[0];
  if (hdr) {
    if (ho[n] - ho[0] > hdr_cap) { set_error("header buffer too small: need %llu", (unsigned long long)(ho[n] - ho[0])); return FEI_E_CAPACITY; }
    FEI_CUDA(cudaMemcpyAsync(hdr, c->hdr.as<uint8_t>() + ho[0], ho[n] - ho[0], cudaMemcpyDeviceToHost, s));
  }
  if (ts) FEI_CUDA(cudaMemcpyAsync(ts, c->ts.as<int64_t>() + first, n * 8, cudaMemcpyDeviceToHost, s));
  if (wall) FEI_CUDA(cudaMemcpyAsync(wall, c->wall.as<int64_t>() + first, n * 8, cudaMemcpyDeviceToHost, s));
  if (flags8) FEI_CUDA(cudaMemcpyAsync(flags8, c->flags8.as<uint64_t>() + first, n * 8, cudaMemcpyDeviceToHost, s));
  if (fsb) FEI_CUDA(cudaMemcpyAsync(fsb, c->fsb.as<uint32_t>() + first, n * 4, cudaMemcpyDeviceToHost, s));
  if (body || body_off) {
    // lengths via rec_pos -> grp_len
    std::vector<uint32_t> pos(n), glen(c->n_groups * 32);
    FEI_CUDA(cudaMemcpyAsync(pos.data(), c->rec_pos.as<uint32_t>() + first, n * 4, cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaMemcpyAsync(glen.data(), c->grp_len.p, glen.size() * 4, cudaMemcpyDeviceToHost, s));
    FEI_CUDA(cudaStreamSynchronize(s));
    std::vector<uint64_t> bo(n + 1, 0);
    for (uint64_t i = 0; i < n; ++i) bo[i + 1] = bo[i] + glen[pos[i]];
    if (body_off) memcpy(body_off, bo.data(), (n + 1) * 8);
    if (body) {
      if (bo[n] > body_cap) { set_error("body buffer too small: need %llu", (unsigned long long)bo[n]); return FEI_E_CAPACITY; }
      DevBuf d_off, d_out;
      FEI_TRY(d_off.alloc((n + 1) * 8)); FEI_TRY(d_out.alloc(bo[n] + 16));
      FEI_CUDA(cudaMemcpyAsync(d_off.p, bo.data(), (n + 1) * 8, cudaMemcpyHostToDevice, s));
      k_untile<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(c->tiles.as<uint8_t>(), c->grp_base.as<uint64_t>(), c->grp_len.as<uint32_t>(),
                                                        c->rec_pos.as<uint32_t>(), first, n, d_off.as<uint64_t>(), d_out.as<uint8_t>());
      FEI_CUDA(cudaGetLastError());
      FEI_CUDA(cudaMemcpyAsync(body, d_out.p, bo[n], cudaMemcpyDeviceToHost, s));
      FEI_CUDA(cudaStreamSynchronize(s));
    }
  }
  FEI_CUDA(cudaStreamSynchronize(s));
  return FEI_OK;
}
