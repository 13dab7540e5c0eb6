// Packed-corpus snapshot: the device-resident pack (header blob, meta columns, names, body tiles, header directory, key
// dictionary, value columns) written to / restored from one file, so that a process restart does not re-walk and re-pack the
// Memdir tree (the reference re-reads every file on every query, memdir_tools/utils.py:202-253).  Restoring streams the file
// through a ring of pinned buffers: reader threads pread the next chunks while the copy engine uploads the previous ones.
#include "corpus.h"
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <string.h>
#include <errno.h>
#include <thread>
#include <vector>

namespace fei {
namespace {

constexpr uint64_t kSnapMagic = 0x50414E5349454631ull;   // "1FEISNAP"
constexpr uint32_t kSnapVersion = 2;
constexpr size_t kSlot = 32u << 20;                      // pinned ring slot
constexpr int kSlots = 4;
constexpr int kReaders = 4;

struct SnapHeader {
  uint64_t magic; uint32_t version, n_sections;
  uint64_t n, global_base, hdr_bytes, body_bytes, name_bytes, tile_bytes, n_groups, hdir_entries;
  uint32_t n_cols, has_text_records;
  uint64_t section_bytes[32];
};

struct Ring {
  uint8_t* slot[kSlots] = {nullptr};
  cudaEvent_t ev[kSlots] = {nullptr};
  int init() {
    for (int i = 0; i < kSlots; ++i) { FEI_CUDA(cudaMallocHost(&slot[i], kSlot)); FEI_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming)); }
    return FEI_OK;
  }
  ~Ring() { for (int i = 0; i < kSlots; ++i) { if (slot[i]) cudaFreeHost(slot[i]); if (ev[i]) cudaEventDestroy(ev[i]); } }
};

std::vector<DevBuf*> sections(fei_corpus* c) {
  return {&c->hdr, &c->hdr_off, &c->name, &c->name_off, &c->name_spans, &c->ts, &c->wall, &c->flags8, &c->fsb,
          &c->tiles, &c->grp_base, &c->grp_rec, &c->grp_len, &c->rec_pos, &c->hdir, &c->hdir_off,
          &c->key_tag, &c->key_rep, &c->key_len, &c->kid_col, &c->col_len, &c->col_planes};
}

bool pread_all(int fd, uint8_t* dst, size_t bytes, uint64_t off) {
  size_t done = 0;
  while (done < bytes) {
    ssize_t r = pread(fd, dst + done, bytes - done, (off_t)(off + done));
    if (r < 0) { if (errno == EINTR) continue; return false; }
    if (r == 0) return false;
    done += (size_t)r;
  }
  return true;
}

}  // namespace
}  // namespace fei

using namespace fei;

extern "C" int fei_corpus_save(fei_corpus* c, const char* path) {
  if (!c || !path) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_ready());
  if (!c->loaded) { set_error("corpus not loaded"); return FEI_E_STATE; }
  cudaStream_t s = ctx().copy_stream;
  const int fd = open(path, O_WRONLY | O_CREAT | O_TRUNC, 0644);
  if (fd < 0) { set_error("open(%s): %s", path, strerror(errno)); return FEI_E_BADARG; }
  auto secs = sections(c);
  SnapHeader h; memset(&h, 0, sizeof(h));
  h.magic = kSnapMagic; h.version = kSnapVersion; h.n_sections = (uint32_t)secs.size();
  h.n = c->n; h.global_base = c->global_base; h.hdr_bytes = c->hdr_bytes; h.body_bytes = c->body_bytes; h.name_bytes = c->name_bytes;
  h.tile_bytes = c->tile_bytes; h.n_groups = c->n_groups; h.hdir_entries = c->hdir_entries; h.n_cols = c->n_cols; h.has_text_records = c->has_text_records ? 1 : 0;
  for (size_t k = 0; k < secs.size(); ++k) h.section_bytes[k] = secs[k]->p ? secs[k]->bytes : 0;
  bool ok = write(fd, &h, sizeof(h)) == (ssize_t)sizeof(h);
  Ring ring;
  int rc = ring.init();
  for (size_t k = 0; ok && rc == FEI_OK && k < secs.size(); ++k) {
    const uint64_t total = h.section_bytes[k];
    for (uint64_t o = 0; ok && o < total; o += kSlot) {
      const size_t nb = (size_t)(total - o < kSlot ? total - o : kSlot);
      if (cudaMemcpyAsync(ring.slot[0], (uint8_t*)secs[k]->p + o, nb, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "snapshot D2H", __FILE__, __LINE__); break; }
      size_t done = 0;
      while (done < nb) { ssize_t w = write(fd, ring.slot[0] + done, nb - done); if (w <= 0) { if (errno == EINTR) continue; ok = false; break; } done += (size_t)w; }
    }
  }
  close(fd);
  if (rc != FEI_OK) return rc;
  if (!ok) { set_error("writing snapshot %s: %s", path, strerror(errno)); return FEI_E_BADARG; }
  return FEI_OK;
}

extern "C" int fei_corpus_load_snapshot(fei_corpus* c, const char* path, float* gbs_out) {
  if (!c || !path) { set_error("null argument"); return FEI_E_BADARG; }
  std::lock_guard<std::mutex> lock(c->mu);
  FEI_TRY(require_ready());
  cudaStream_t s = corpus_load_stream(c);
  const int fd = open(path, O_RDONLY);
  if (fd < 0) { set_error("open(%s): %s", path, strerror(errno)); return FEI_E_BADARG; }
  SnapHeader h;
  if (!pread_all(fd, reinterpret_cast<uint8_t*>(&h), sizeof(h), 0) || h.magic != kSnapMagic || h.version != kSnapVersion) { close(fd); set_error("%s is not a feiscan snapshot of this version", path); return FEI_E_BADARG; }
  auto secs = sections(c);
  if (h.n_sections != secs.size()) { close(fd); set_error("snapshot section count mismatch"); return FEI_E_BADARG; }
  c->loaded = false;
  Ring ring;
  int rc = ring.init();
  if (rc != FEI_OK) { close(fd); return rc; }
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0, s);
  uint64_t file_off = sizeof(h), total_bytes = 0;
  // flat list of (device destination, file offset, bytes) chunks over all sections
  struct Chunk { uint8_t* dst; uint64_t off; size_t nb; };
  std::vector<Chunk> chunks;
  for (size_t k = 0; k < secs.size(); ++k) {
    const uint64_t total = h.section_bytes[k];
    if (total) { rc = secs[k]->alloc(total); if (rc != FEI_OK) break; } else secs[k]->release();
    for (uint64_t o = 0; o < total; o += kSlot) chunks.push_back({(uint8_t*)secs[k]->p + o, file_off + o, (size_t)(total - o < kSlot ? total - o : kSlot)});
    file_off += total; total_bytes += total;
  }
  bool io_ok = true;
  if (rc == FEI_OK) {
    // slot j is filled by kReaders threads (each a contiguous quarter), handed to the copy engine, and refilled once its copy is done;
    // the fill of chunk k+1.. overlaps the copies of the chunks before it because filling happens on helper threads
    std::vector<std::thread> fill(kSlots);
    std::vector<char> fill_ok(kSlots, 1);
    auto start_fill = [&](size_t k) {
      const int j = (int)(k % kSlots);
      fill[j] = std::thread([&, k, j]() {
        const Chunk& ck = chunks[k];
        std::vector<std::thread> rd;
        std::vector<char> oks(kReaders, 1);
        const size_t per = (ck.nb + kReaders - 1) / kReaders;
        for (int r = 0; r < kReaders; ++r) {
          const size_t a = (size_t)r * per; if (a >= ck.nb) break;
          const size_t b = a + per < ck.nb ? a + per : ck.nb;
          rd.emplace_back([&, a, b, r]() { oks[r] = pread_all(fd, ring.slot[j] + a, b - a, ck.off + a) ? 1 : 0; });
        }
        for (auto& t : rd) t.join();
        for (char o : oks) if (!o) fill_ok[j] = 0;
      });
    };
    const size_t nchunks = chunks.size();
    for (size_t k = 0; k < nchunks && k < (size_t)kSlots; ++k) start_fill(k);
    for (size_t k = 0; k < nchunks; ++k) {
      const int j = (int)(k % kSlots);
      fill[j].join();
      if (!fill_ok[j]) io_ok = false;
      if (cudaMemcpyAsync(chunks[k].dst, ring.slot[j], chunks[k].nb, cudaMemcpyHostToDevice, s) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "snapshot H2D", __FILE__, __LINE__); break; }
      cudaEventRecord(ring.ev[j], s);
      if (k + kSlots < nchunks) { cudaEventSynchronize(ring.ev[j]); start_fill(k + kSlots); }
    }
    for (auto& t : fill) if (t.joinable()) t.join();
  }
  cudaEventRecord(e1, s);
  if (cudaStreamSynchronize(s) != cudaSuccess && rc == FEI_OK) rc = cuda_fail(cudaGetLastError(), "snapshot sync", __FILE__, __LINE__);
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  close(fd);
  if (rc != FEI_OK) return rc;
  if (!io_ok) { set_error("reading snapshot %s failed (truncated?)", path); return FEI_E_BADARG; }
  c->n = h.n; c->global_base = h.global_base; c->hdr_bytes = h.hdr_bytes; c->body_bytes = h.body_bytes; c->name_bytes = h.name_bytes;
  c->tile_bytes = h.tile_bytes; c->n_groups = h.n_groups; c->hdir_entries = h.hdir_entries; c->n_cols = h.n_cols; c->has_text_records = h.has_text_records != 0;
  for (int x = 0; x < FEI_MAX_AUX; ++x) { c->aux[x].release(); c->aux_n[x] = 0; }
  c->loaded = true;
  if (gbs_out) *gbs_out = ms > 0 ? (float)((double)total_bytes / 1e9 / (ms * 1e-3)) : 0.f;
  return FEI_OK;
}
