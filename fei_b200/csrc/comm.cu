// Multi-GPU plumbing: one process per GPU, NCCL over NVLink 4 / NVSwitch.
//
// The scan shards by contiguous record range (SURVEY.md 8(e)): no data-path collective; the
// only exchange is ONE all-gatherv of the compacted, ordered hit lists at the end (rank-order
// concatenation == global listing order), and an 8-byte min-reduce for a range-sharded chain.
// NCCL has no native gatherv: counts are all-gathered first, then every (rank, query) segment
// is a grouped ncclBroadcast straight into its final position of the gathered list.
//
// libnccl is dlopen()ed at first use so the library also loads on machines without NCCL and
// shares the copy a host process (e.g. torch) may already have mapped.
#include "corpus.h"
#include <dlfcn.h>
#include <vector>
#include <string.h>

namespace fei {
namespace {
void unbind();

typedef struct { char internal[128]; } ncclUniqueId;
typedef void* ncclComm_t;
enum { ncclSuccess = 0 };
enum { ncclUint8 = 1, ncclUint32 = 3, ncclInt64 = 4, ncclUint64 = 5 };
enum { ncclSum = 0, ncclProd = 1, ncclMax = 2, ncclMin = 3 };

struct Nccl {
  void* h = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  ncclComm_t comm = nullptr;
  int nranks = 0, rank = -1;
  DevBuf counts_dev, gathered, gathered_local, scratch, lists;
  CompactScratch compact;
  std::mutex mu;                 // one collective at a time per communicator
  // ---- bound shard set (fei_comm_bind_corpus): record count / first global index of every rank's shard, the rank-major
  // buffer every rank receives the all-gathered hit masks in, and that buffer of every peer mapped into this process
  // (CUDA IPC over NVLink / NVSwitch peer memory) so that the scan kernel can store its finished windows of masks into it
  fei_corpus* bound = nullptr;
  std::vector<uint64_t> shard_n, shard_base;
  uint64_t n_max = 0, n_total = 0;
  DevBuf gathered_masks, totals_dev;
  std::vector<void*> peer_masks;
  DevBuf peer_ptrs;                      // the same pointers as a device array (what the scan kernel stores through)
  bool p2p = false;
  uint64_t* totals_host = nullptr;       // pinned
  // ---- what the last gather left on the device (fei_comm_gathered_checksum / fei_comm_global_lists)
  bool last_pushed = false;              // the last fei_comm_scan_gather moved its masks from inside the scan kernel
  int last_kind = 0;                     // 0 none, 1 dense masks in gathered_masks, 2 sparse lists in `gathered`, 3 dense masks in `gathered` (fei_comm_allgather_hits)
  uint32_t last_nq = 0;
  uint64_t last_tot[32] = {0}, last_qbase[33] = {0};
  uint64_t last_nmax = 0;
  std::vector<uint64_t> last_n, last_base;
  DevBuf global_lists; uint64_t global_stride = 0;
};
Nccl g;

int load_nccl() {
  if (g.h) return FEI_OK;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) { g.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (g.h) break; }
  if (!g.h) { set_error("cannot dlopen libnccl.so.2: %s", dlerror()); return FEI_E_NCCL; }
#define SYM(field, name) *(void**)(&g.field) = dlsym(g.h, name); if (!g.field) { set_error("libnccl lacks %s", name); return FEI_E_NCCL; }
  SYM(GetUniqueId, "ncclGetUniqueId") SYM(CommInitRank, "ncclCommInitRank") SYM(CommDestroy, "ncclCommDestroy")
  SYM(AllGather, "ncclAllGather") SYM(Broadcast, "ncclBroadcast") SYM(AllReduce, "ncclAllReduce")
  SYM(GroupStart, "ncclGroupStart") SYM(GroupEnd, "ncclGroupEnd") SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
  return FEI_OK;
}

int nccl_fail(int rc, const char* what) {
  set_error("NCCL error %d (%s) in %s", rc, g.GetErrorString ? g.GetErrorString(rc) : "?", what);
  return FEI_E_NCCL;
}
#define FEI_NCCL(call) do { int rc__ = (call); if (rc__ != ncclSuccess) return nccl_fail(rc__, #call); } while (0)

void unbind() {
  for (size_t r = 0; r < g.peer_masks.size(); ++r)
    if (g.peer_masks[r] && (int)r != g.rank) cudaIpcCloseMemHandle(g.peer_masks[r]);
  g.peer_masks.clear(); g.bound = nullptr; g.p2p = false;
}

// After the scan, unless the scan kernel stored its masks into the peers itself, this shard's masks go to every rank's
// rank-major buffer:
//   p2p  : one cudaMemcpyAsync per peer into the peer's mapped buffer (copy engines);
//   else : grouped ncclBroadcast, one per rank, straight into the final position (the all-gatherv of the masks).
// Then the per-query totals of all ranks; on the p2p paths this all-reduce is also what tells a rank that every peer's
// stores / copies into its buffer have landed (a rank enters it only after its own, in stream order).
struct GatherHook : ScanHook {
  fei_corpus* c;
  int after_scan(cudaStream_t s) override {
    const int R = g.nranks, me = g.rank;
    if (g.p2p) {                                                       // (only a p2p scan pushes)
      if (!pushed && c->n)
        for (int i = 0; i < R; ++i) {
          const int r = (me + i) % R;                                  // every rank starts with a different peer
          uint32_t* dst = reinterpret_cast<uint32_t*>(g.peer_masks[r]) + (size_t)me * g.n_max;
          FEI_CUDA(cudaMemcpyAsync(dst, c->hits.as<uint32_t>(), c->n * 4, cudaMemcpyDefault, s));
        }
    } else {
      FEI_NCCL(g.GroupStart());
      for (int r = 0; r < R; ++r)
        if (g.shard_n[r])
          FEI_NCCL(g.Broadcast(c->hits.as<uint32_t>(), g.gathered_masks.as<uint32_t>() + (size_t)r * g.n_max, g.shard_n[r], ncclUint32, r, g.comm, s));
      FEI_NCCL(g.GroupEnd());
    }
    FEI_NCCL(g.AllReduce(c->compact.totals.p, g.totals_dev.p, 32, ncclUint64, ncclSum, g.comm, s));
    FEI_CUDA(cudaMemcpyAsync(g.totals_host, g.totals_dev.p, 32 * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    return FEI_OK;
  }
};

}  // namespace
}  // namespace fei

using namespace fei;

// Collective.  Every rank names the shard it will scan; the ranks exchange (record count, first global index), size the
// rank-major mask buffer and map each other's buffer (CUDA IPC).  FEI_COMM_P2P=0 keeps everything on NCCL.
extern "C" int fei_comm_bind_corpus(fei_corpus* c) {
  FEI_TRY(require_ready());
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  if (!g.comm) { set_error("fei_comm_init() has not been called"); return FEI_E_STATE; }
  std::lock_guard<std::mutex> lock(g.mu);
  cudaStream_t s = ctx().stream;
  const int R = g.nranks;
  unbind();
  FEI_TRY(g.counts_dev.ensure((size_t)(R + 1) * 34 * sizeof(uint64_t)));
  uint64_t mine_h[2] = {c->n, c->global_base};
  uint64_t* mine = g.counts_dev.as<uint64_t>() + (size_t)R * 34;
  FEI_CUDA(cudaMemcpyAsync(mine, mine_h, sizeof(mine_h), cudaMemcpyHostToDevice, s));
  FEI_NCCL(g.AllGather(mine, g.counts_dev.p, 2, ncclUint64, g.comm, s));
  std::vector<uint64_t> info((size_t)R * 2);
  FEI_CUDA(cudaMemcpyAsync(info.data(), g.counts_dev.p, info.size() * 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  g.shard_n.assign(R, 0); g.shard_base.assign(R, 0); g.n_max = 0; g.n_total = 0;
  for (int r = 0; r < R; ++r) { g.shard_n[r] = info[2 * r]; g.shard_base[r] = info[2 * r + 1]; g.n_total += g.shard_n[r]; if (g.shard_n[r] > g.n_max) g.n_max = g.shard_n[r]; }
  g.n_max = (g.n_max + 3) & ~3ull;                                // rank segments start 16-byte aligned: the scan kernel stores whole windows with 16-byte stores
  FEI_TRY(g.gathered_masks.alloc(((size_t)R * g.n_max + 1) * sizeof(uint32_t)));     // a fresh allocation: the IPC handle names exactly this buffer
  FEI_TRY(g.totals_dev.ensure(32 * sizeof(uint64_t)));
  if (!g.totals_host) FEI_CUDA(cudaMallocHost(&g.totals_host, 32 * sizeof(uint64_t)));
  g.peer_masks.assign(R, nullptr);
  g.peer_masks[g.rank] = g.gathered_masks.p;
  int ok = 1;
  const char* env = getenv("FEI_COMM_P2P");
  if (env && env[0] == '0') ok = 0;
  cudaIpcMemHandle_t hnd; memset(&hnd, 0, sizeof(hnd));
  if (ok && cudaIpcGetMemHandle(&hnd, g.gathered_masks.p) != cudaSuccess) { cudaGetLastError(); ok = 0; }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  FEI_TRY(g.scratch.ensure((size_t)(R + 1) * 64 + 16));
  uint8_t* hmine = g.scratch.as<uint8_t>() + (size_t)R * 64;
  FEI_CUDA(cudaMemcpyAsync(hmine, &hnd, 64, cudaMemcpyHostToDevice, s));
  FEI_NCCL(g.AllGather(hmine, g.scratch.p, 64, ncclUint8, g.comm, s));
  std::vector<cudaIpcMemHandle_t> all(R);
  FEI_CUDA(cudaMemcpyAsync(all.data(), g.scratch.p, (size_t)R * 64, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  for (int r = 0; ok && r < R; ++r) {
    if (r == g.rank) continue;
    void* p = nullptr;
    if (cudaIpcOpenMemHandle(&p, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0; break; }
    g.peer_masks[r] = p;
  }
  // all ranks or none
  uint64_t flag = ok ? 1 : 0;
  FEI_CUDA(cudaMemcpyAsync(g.totals_dev.p, &flag, 8, cudaMemcpyHostToDevice, s));
  FEI_NCCL(g.AllReduce(g.totals_dev.p, g.totals_dev.p, 1, ncclUint64, ncclMin, g.comm, s));
  FEI_CUDA(cudaMemcpyAsync(&flag, g.totals_dev.p, 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  g.p2p = flag != 0;
  if (g.p2p) {
    FEI_TRY(g.peer_ptrs.ensure((size_t)R * sizeof(void*)));
    FEI_CUDA(cudaMemcpyAsync(g.peer_ptrs.p, g.peer_masks.data(), (size_t)R * sizeof(void*), cudaMemcpyHostToDevice, s));
    FEI_CUDA(cudaStreamSynchronize(s));
  }
  if (!g.p2p) { for (int r = 0; r < R; ++r) if (r != g.rank && g.peer_masks[r]) { cudaIpcCloseMemHandle(g.peer_masks[r]); g.peer_masks[r] = nullptr; } }
  g.bound = c;
  return FEI_OK;
}

extern "C" int fei_comm_is_p2p(void) { return g.p2p ? 1 : 0; }
/* 1 if the last fei_comm_scan_gather exchanged its hit masks with stores from inside the scan kernel (peer memory), 0 if copy
 * engines / NCCL moved them after the scan. */
extern "C" int fei_comm_last_exchange_in_kernel(void) { return g.last_pushed ? 1 : 0; }

// Collective.  Scan + ordered local lists exactly like fei_scan_count; by default the scan kernel stores each finished
// window of masks into every rank's buffer while it scans the next ones.  On return every rank holds the hit masks of ALL
// shards (rank-major = global listing order) on its device and the global per-query totals in nhits_total[nq].
extern "C" int fei_comm_scan_gather(fei_corpus* c, const uint8_t* prog, uint64_t prog_len, uint64_t* nhits_total) {
  FEI_TRY(require_ready());
  if (!c) { set_error("null corpus"); return FEI_E_BADARG; }
  if (!g.comm) { set_error("fei_comm_init() has not been called"); return FEI_E_STATE; }
  std::lock_guard<std::mutex> lock(g.mu);
  std::lock_guard<std::mutex> clock(c->mu);
  if (g.bound != c || g.shard_n[g.rank] != c->n || g.shard_base[g.rank] != c->global_base) { set_error("corpus is not the one bound with fei_comm_bind_corpus (or it was reloaded since)"); return FEI_E_STATE; }
  GatherHook hook; hook.c = c;
  const char* kp = getenv("FEI_COMM_KERNEL_PUSH");
  if (g.p2p && !(kp && kp[0] == '0')) {                            // fused exchange: peer stores from inside the scan kernel
    hook.push_peers = reinterpret_cast<uint32_t* const*>(g.peer_ptrs.p); hook.push_n = (uint32_t)g.nranks; hook.push_off = (uint64_t)g.rank * g.n_max;
  }
  FEI_TRY(run_scan(c, prog, prog_len, kScanCompactLists, &hook));
  g.last_pushed = hook.pushed;
  FEI_TRY(finish_timing(c, true));
  g.last_kind = 1; g.last_nq = c->last_nq; g.last_nmax = g.n_max; g.last_n = g.shard_n; g.last_base = g.shard_base;
  for (uint32_t q = 0; q < 32; ++q) g.last_tot[q] = q < c->last_nq ? g.totals_host[q] : 0;
  if (nhits_total) for (uint32_t q = 0; q < c->last_nq; ++q) nhits_total[q] = g.totals_host[q];
  return FEI_OK;
}

// Order-sensitive checksums (A_q = sum_k (k+1) * list_q[k], S_q = sum_k list_q[k], mod 2^64) and lengths of the GLOBAL ordered
// hit lists the last gather on this rank stands for (dense: compacted from the gathered masks rank by rank; sparse: the
// gathered lists).  An unsharded scan of the same records gives the same numbers through fei_scan_list_checksum.
extern "C" int fei_comm_gathered_checksum(uint32_t nq, uint64_t* totals, uint64_t* a_out, uint64_t* s_out) {
  FEI_TRY(require_ready());
  std::lock_guard<std::mutex> lock(g.mu);
  if (!g.last_kind || nq != g.last_nq || !totals || !a_out || !s_out) { set_error("no matching gather result"); return FEI_E_STATE; }
  cudaStream_t s = ctx().stream;
  for (uint32_t q = 0; q < nq; ++q) { totals[q] = 0; a_out[q] = 0; s_out[q] = 0; }
  if (g.last_kind == 2) {
    for (uint32_t q = 0; q < nq; ++q) {
      totals[q] = g.last_tot[q];
      FEI_TRY(list_checksum(g.gathered.as<uint64_t>() + g.last_qbase[q], g.last_tot[q], g.scratch, a_out + q, s_out + q, s));
    }
    return FEI_OK;
  }
  const uint32_t* masks = g.last_kind == 1 ? g.gathered_masks.as<uint32_t>() : g.gathered.as<uint32_t>();
  for (size_t r = 0; r < g.last_n.size(); ++r) {
    uint64_t cnt[32], stride = 1;
    FEI_TRY(compact_masks(masks + r * g.last_nmax, g.last_n[r], nq, g.last_base[r], g.compact, cnt, &g.lists, &stride, nullptr, s));
    for (uint32_t q = 0; q < nq; ++q) {
      uint64_t a = 0, sum = 0;
      FEI_TRY(list_checksum(g.lists.as<uint64_t>() + (size_t)q * stride, cnt[q], g.scratch, &a, &sum, s));
      a_out[q] += a + totals[q] * sum; s_out[q] += sum; totals[q] += cnt[q];
    }
  }
  return FEI_OK;
}

// The global ordered hit lists themselves, built on this rank's device from the gathered masks (dense result): list q =
// global_lists[q * stride .. + totals[q]).  ms_out = device time of the build.  (The sparse wire format already is the lists.)
extern "C" int fei_comm_global_lists(uint32_t nq, uint64_t* totals, float* ms_out) {
  FEI_TRY(require_ready());
  std::lock_guard<std::mutex> lock(g.mu);
  if ((g.last_kind != 1 && g.last_kind != 3) || nq != g.last_nq) { set_error("no dense gather result"); return FEI_E_STATE; }
  cudaStream_t s = ctx().stream;
  const uint32_t* masks = g.last_kind == 1 ? g.gathered_masks.as<uint32_t>() : g.gathered.as<uint32_t>();
  uint64_t n_total = 0;
  for (uint64_t v : g.last_n) n_total += v;
  g.global_stride = n_total ? n_total : 1;
  FEI_TRY(g.global_lists.ensure(g.global_stride * nq * sizeof(uint64_t)));
  cudaEvent_t e0, e1;
  FEI_CUDA(cudaEventCreate(&e0)); FEI_CUDA(cudaEventCreate(&e1));
  FEI_CUDA(cudaEventRecord(e0, s));
  int rc = compact_segments(masks, g.last_nmax, g.last_n.data(), g.last_base.data(), (uint32_t)g.last_n.size(), nq, g.compact, g.global_stride, g.global_lists.as<uint64_t>(), totals, s);
  cudaEventRecord(e1, s);
  cudaStreamSynchronize(s);
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (ms_out) *ms_out = ms;
  return rc;
}

extern "C" int fei_comm_unique_id(uint8_t* id) {
  if (!id) { set_error("null id"); return FEI_E_BADARG; }
  FEI_TRY(load_nccl());
  ncclUniqueId u;
  FEI_NCCL(g.GetUniqueId(&u));
  memcpy(id, u.internal, FEI_NCCL_ID_BYTES);
  return FEI_OK;
}

extern "C" int fei_comm_init(const uint8_t* id, int nranks, int rank) {
  FEI_TRY(require_ready());
  if (!id || nranks < 1 || rank < 0 || rank >= nranks) { set_error("bad communicator arguments"); return FEI_E_BADARG; }
  FEI_TRY(load_nccl());
  if (g.comm) { g.CommDestroy(g.comm); g.comm = nullptr; }
  ncclUniqueId u; memcpy(u.internal, id, FEI_NCCL_ID_BYTES);
  FEI_NCCL(g.CommInitRank(&g.comm, nranks, u, rank));
  g.nranks = nranks; g.rank = rank;
  return FEI_OK;
}

extern "C" int fei_comm_destroy(void) {
  if (g.comm) { g.CommDestroy(g.comm); g.comm = nullptr; }
  unbind();
  g.counts_dev.release(); g.gathered.release(); g.gathered_local.release(); g.scratch.release(); g.lists.release(); g.gathered_masks.release(); g.totals_dev.release(); g.global_lists.release();
  if (g.totals_host) { cudaFreeHost(g.totals_host); g.totals_host = nullptr; }
  g.last_kind = 0;
  g.compact.blk_counts.release(); g.compact.blk_offsets.release(); g.compact.totals.release();
  g.nranks = 0; g.rank = -1;
  return FEI_OK;
}

// All-gatherv of the scan result of every rank.  Two wire formats, chosen per call from the gathered counts:
//   sparse : the compacted per-query index lists, one grouped ncclBroadcast per (rank, query) segment of the
//            rank's corpus-local 32-bit entries (4 B per hit) straight into its final position, then widened on
//            the receiver with that rank's global_base into the 64-bit global lists;
//   dense  : when the lists would be larger than the per-record hit masks (4 B per record) — typical for
//            many-pattern batches where most records hit — the masks are all-gathered instead (one
//            ncclAllGather) and the global ordered lists are compacted from them on demand.
// Either way rank-order concatenation is the global listing order.
extern "C" int fei_comm_allgather_hits(fei_corpus* c, uint32_t nq, uint64_t* const* hits, const uint64_t* cap,
                                       uint64_t* nhits_total, uint64_t* counts_out) {
  FEI_TRY(require_ready());
  if (!c || nq == 0 || nq > 32 || nq != c->last_nq) { set_error("no matching scan result on this corpus (run fei_scan_count / fei_scan_hits first)"); return FEI_E_STATE; }
  if (!g.comm) { set_error("fei_comm_init() has not been called"); return FEI_E_STATE; }
  std::lock_guard<std::mutex> lock(g.mu);
  std::lock_guard<std::mutex> clock(c->mu);
  cudaStream_t s = ctx().stream;
  const int R = g.nranks;
  const uint32_t W = nq + 2;                                   // per-rank record: counts[nq], n, global_base
  FEI_TRY(g.counts_dev.ensure((size_t)(R + 1) * 34 * sizeof(uint64_t)));
  uint64_t mine_h[34];
  for (uint32_t q = 0; q < nq; ++q) mine_h[q] = c->last_counts[q];
  mine_h[nq] = c->n; mine_h[nq + 1] = c->global_base;
  uint64_t* mine = g.counts_dev.as<uint64_t>() + (size_t)R * 34;
  FEI_CUDA(cudaMemcpyAsync(mine, mine_h, W * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  FEI_NCCL(g.AllGather(mine, g.counts_dev.p, W, ncclUint64, g.comm, s));
  std::vector<uint64_t> info((size_t)R * W);
  FEI_CUDA(cudaMemcpyAsync(info.data(), g.counts_dev.p, info.size() * 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  std::vector<uint64_t> tot(nq, 0);
  uint64_t list_entries = 0, n_total = 0, n_max = 0;
  for (int r = 0; r < R; ++r) {
    for (uint32_t q = 0; q < nq; ++q) { uint64_t v = info[(size_t)r * W + q]; tot[q] += v; list_entries += v; if (counts_out) counts_out[(size_t)r * nq + q] = v; }
    uint64_t nr = info[(size_t)r * W + nq];
    n_total += nr; if (nr > n_max) n_max = nr;
  }
  for (uint32_t q = 0; q < nq; ++q) if (nhits_total) nhits_total[q] = tot[q];
  const bool want_host = hits && cap;
  const bool dense = list_entries * 8 > (uint64_t)R * n_max * 4;
  g.last_kind = dense ? 3 : 2; g.last_nq = nq; g.last_nmax = n_max;
  g.last_n.assign(R, 0); g.last_base.assign(R, 0);
  for (int r = 0; r < R; ++r) { g.last_n[r] = info[(size_t)r * W + nq]; g.last_base[r] = info[(size_t)r * W + nq + 1]; }
  for (uint32_t q = 0; q < 32; ++q) g.last_tot[q] = q < nq ? tot[q] : 0;
  bool truncated = false;
  if (!dense) {
    std::vector<uint64_t> qbase(nq + 1, 0);
    for (uint32_t q = 0; q < nq; ++q) qbase[q + 1] = qbase[q] + tot[q];
    for (uint32_t q = 0; q <= nq; ++q) g.last_qbase[q] = qbase[q];
    FEI_TRY(g.gathered.ensure((qbase[nq] + 1) * sizeof(uint64_t)));
    FEI_TRY(g.gathered_local.ensure((qbase[nq] + 1) * sizeof(uint32_t)));
    FEI_NCCL(g.GroupStart());
    for (uint32_t q = 0; q < nq; ++q) {
      uint64_t pos = qbase[q];
      for (int r = 0; r < R; ++r) {
        uint64_t cnt = info[(size_t)r * W + q];
        if (cnt) {
          const void* src = c->hit_lists.as<uint32_t>() + (size_t)q * c->hit_list_stride;   // only read on the root
          FEI_NCCL(g.Broadcast(src, g.gathered_local.as<uint32_t>() + pos, cnt, ncclUint32, r, g.comm, s));
        }
        pos += cnt;
      }
    }
    FEI_NCCL(g.GroupEnd());
    for (uint32_t q = 0; q < nq; ++q) {
      uint64_t pos = qbase[q];
      for (int r = 0; r < R; ++r) {
        const uint64_t cnt = info[(size_t)r * W + q];
        FEI_TRY(widen_list(g.gathered_local.as<uint32_t>() + pos, cnt, g.last_base[r], g.gathered.as<uint64_t>() + pos, s));
        pos += cnt;
      }
    }
    for (uint32_t q = 0; want_host && q < nq; ++q) {
      if (!hits[q]) continue;
      uint64_t take = tot[q] < cap[q] ? tot[q] : cap[q];
      if (take < tot[q]) truncated = true;
      if (take) FEI_CUDA(cudaMemcpyAsync(hits[q], g.gathered.as<uint64_t>() + qbase[q], take * 8, cudaMemcpyDeviceToHost, s));
    }
  } else {
    // dense: gather the masks (every rank contributes n_max entries; the tail of short shards is ignored)
    if (c->hits.bytes < n_max * sizeof(uint32_t)) {            // shorter shard than the longest one: grow, keep contents
      DevBuf nb;
      FEI_TRY(nb.alloc(n_max * sizeof(uint32_t)));
      FEI_CUDA(cudaMemsetAsync(nb.p, 0, n_max * sizeof(uint32_t), s));
      if (c->n) FEI_CUDA(cudaMemcpyAsync(nb.p, c->hits.p, c->n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
      FEI_CUDA(cudaStreamSynchronize(s));
      void* tp = nb.p; nb.p = c->hits.p; c->hits.p = tp;
      size_t tb = nb.bytes; nb.bytes = c->hits.bytes; c->hits.bytes = tb;
    }
    FEI_TRY(g.gathered.ensure((size_t)R * n_max * sizeof(uint32_t)));
    FEI_NCCL(g.AllGather(c->hits.p, g.gathered.p, n_max, ncclUint32, g.comm, s));
    if (want_host) {
      CompactScratch& sc = g.compact; DevBuf& lists = g.lists;
      std::vector<uint64_t> written(nq, 0);
      for (int r = 0; r < R; ++r) {
        uint64_t nr = info[(size_t)r * W + nq], gb = info[(size_t)r * W + nq + 1];
        uint64_t cnt[32], stride = 1;
        FEI_TRY(compact_masks(g.gathered.as<uint32_t>() + (size_t)r * n_max, nr, nq, gb, sc, cnt, &lists, &stride, nullptr, s));
        for (uint32_t q = 0; q < nq; ++q) {
          if (!hits[q] || !cnt[q]) continue;
          uint64_t room = cap[q] > written[q] ? cap[q] - written[q] : 0;
          uint64_t take = cnt[q] < room ? cnt[q] : room;
          if (take < cnt[q]) truncated = true;
          if (take) FEI_CUDA(cudaMemcpyAsync(hits[q] + written[q], lists.as<uint64_t>() + (size_t)q * stride, take * 8, cudaMemcpyDeviceToHost, s));
          written[q] += take;
        }
        FEI_CUDA(cudaStreamSynchronize(s));
      }
    }
  }
  FEI_CUDA(cudaStreamSynchronize(s));
  if (truncated) { set_error("gathered hit buffer too small for at least one query (see nhits_total)"); return FEI_E_CAPACITY; }
  return FEI_OK;
}

extern "C" int fei_comm_allreduce_first_bad(int64_t* first_bad, int32_t* bad_kind) {
  FEI_TRY(require_ready());
  if (!first_bad || !bad_kind) { set_error("null argument"); return FEI_E_BADARG; }
  if (!g.comm) { set_error("fei_comm_init() has not been called"); return FEI_E_STATE; }
  cudaStream_t s = ctx().stream;
  // key = index*4 + kind, "no failure" = max uint64; min over ranks keeps the reference's first failure
  uint64_t key = *first_bad < 0 ? ~0ull : ((uint64_t)*first_bad << 2 | (uint64_t)(*bad_kind & 3));
  FEI_TRY(g.scratch.ensure(16));
  FEI_CUDA(cudaMemcpyAsync(g.scratch.p, &key, 8, cudaMemcpyHostToDevice, s));
  FEI_NCCL(g.AllReduce(g.scratch.p, g.scratch.p, 1, ncclUint64, ncclMin, g.comm, s));
  FEI_CUDA(cudaMemcpyAsync(&key, g.scratch.p, 8, cudaMemcpyDeviceToHost, s));
  FEI_CUDA(cudaStreamSynchronize(s));
  if (key == ~0ull) { *first_bad = -1; *bad_kind = 0; }
  else { *first_bad = (int64_t)(key >> 2); *bad_kind = (int32_t)(key & 3); }
  return FEI_OK;
}
