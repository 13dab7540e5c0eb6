// Host side of the one-time pack: what utils.list_memories does per directory (memdir_tools/utils.py:202-253) as native,
// multi-threaded code -- readdir + the file-name grammar + stat, the stable newest-first order, and the file reads (pread into one
// contiguous, optionally pinned, buffer that fei_corpus_load_raw uploads).  The text work (decode, newline folding, '---' split,
// strip) stays on the GPU (ingest.cu).  No per-file work is left in Python.
#include "../../include/feiscan.h"
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <string>
#include <thread>
#include <vector>
#include <dirent.h>
#include <sched.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

namespace fei { void set_error(const char* fmt, ...) __attribute__((format(printf, 1, 2))); }
using fei::set_error;

struct fei_dirlist {
  std::string blob;                     // names back to back
  std::vector<uint64_t> name_off;       // n + 1
  std::vector<int64_t> ts, wall, mtime_ns;
  std::vector<uint64_t> ino, size, flags8;
  std::vector<uint16_t> spans;          // 4 per entry: unique_id start, length, hostname start, length (bytes inside the name)
  std::vector<uint8_t> status;          // 1 = a memory file (grammar matched, ASCII fast path); 2 = let Python's re / int() / datetime decide
  std::vector<int64_t> flags_len;       // number of flag letters (> 7 cannot be packed)
};

namespace {

// `\d+\.[a-z0-9]+\.[^:]+:2,[A-Z]*` as a prefix match (utils.py:223, :81).  Python's \d also matches non-ASCII digits: names that
// do not start with an ASCII digit but with a byte >= 0x80 are handed to Python (status 2).
int parse_name(const char* s, size_t len, int64_t* ts, uint16_t* spans, uint64_t* flags8, int64_t* nflags) {
  size_t i = 0;
  if (len && (unsigned char)s[0] >= 0x80) return 2;
  while (i < len && s[i] >= '0' && s[i] <= '9') ++i;
  if (i == 0) return 0;
  if (i < len && (unsigned char)s[i] >= 0x80) return 2;            // could be more (Unicode) digits
  if (i > 18) return 2;                                            // int() is unbounded; int64 is not
  if (i >= len || s[i] != '.') return 0;
  int64_t t = 0;
  for (size_t k = 0; k < i; ++k) t = t * 10 + (s[k] - '0');
  size_t a = ++i;
  while (i < len && ((s[i] >= 'a' && s[i] <= 'z') || (s[i] >= '0' && s[i] <= '9'))) ++i;
  if (i == a || i >= len || s[i] != '.') return 0;
  // `[a-z0-9]+\.` then `[^:]+:2,`: the regex backtracks over where the first group ends only if the remainder fails; since group 2
  // cannot contain '.', its end is the first '.' after at least one character -- no alternative split exists.
  size_t ue = i;
  size_t b = ++i;
  while (i < len && s[i] != ':') ++i;
  if (i == b || i + 2 >= len + 0 || i >= len) return 0;
  if (len - i < 3 || s[i + 1] != '2' || s[i + 2] != ',') return 0;
  size_t he = i;
  i += 3;
  uint64_t f = 0; int64_t nf = 0;
  while (i < len && s[i] >= 'A' && s[i] <= 'Z') { if (nf < 7) f |= (uint64_t)(unsigned char)s[i] << (8 * nf); ++nf; ++i; }
  if (a > 0xFFFF || he > 0xFFFF) return 2;
  *ts = t;
  spans[0] = (uint16_t)a; spans[1] = (uint16_t)(ue - a); spans[2] = (uint16_t)b; spans[3] = (uint16_t)(he - b);
  *flags8 = f | ((uint64_t)(nf < 7 ? nf : 7) << 56);
  *nflags = nf;
  return 1;
}

}  // namespace

// datetime.fromtimestamp(ts) as a naive wall clock, in seconds (timegm of the local broken-down time); false when Python would raise
// (year > 9999).  localtime_r takes glibc's tz lock on every call, which serialises the listing threads, so the UTC offset is
// cached per UTC day: a day whose 25 hourly samples agree has one offset (zone rules change on whole hours at the finest); any
// other day (a DST switch) goes through localtime_r entry by entry.
static bool wall_of_slow(int64_t ts, int64_t* wall) {
  time_t tt = (time_t)ts; struct tm tmv;
  if (!localtime_r(&tt, &tmv) || tmv.tm_year + 1900 > 9999) return false;
  *wall = (int64_t)timegm(&tmv);
  return true;
}
static bool wall_of(int64_t ts, int64_t* wall) {
  struct Slot { int64_t day; int64_t off; int state; };            // state: 0 empty, 1 constant offset, 2 mixed
  static thread_local Slot cache[64];
  if (ts < 0 || ts > 253370764800ll) return wall_of_slow(ts, wall);  // before 1970 / the last weeks of year 9999: no shortcut
  const int64_t day = ts / 86400;
  Slot& sl = cache[day & 63];
  if (sl.state == 0 || sl.day != day) {
    sl.day = day; sl.state = 1; sl.off = 0;
    for (int h = 0; h <= 24; ++h) {
      int64_t w;
      const int64_t t = day * 86400 + h * 3600;
      if (!wall_of_slow(t, &w)) { sl.state = 2; break; }
      if (h == 0) sl.off = w - t; else if (w - t != sl.off) { sl.state = 2; break; }
    }
  }
  if (sl.state == 2) return wall_of_slow(ts, wall);
  *wall = ts + sl.off;
  return true;
}

static int dir_list(const char* path, bool want_stat, fei_dirlist** out) {
  if (!path || !out) { set_error("null argument"); return FEI_E_BADARG; }
  *out = nullptr;
  DIR* d = opendir(path);
  if (!d) {
    if (errno == ENOENT) { *out = new fei_dirlist(); (*out)->name_off.push_back(0); return FEI_OK; }     // os.path.exists(path) false: empty listing
    set_error("opendir(%s): %s", path, strerror(errno)); return FEI_E_BADARG;
  }
  const int dfd = dirfd(d);
  const bool timing = getenv("FEI_LIST_TIMING") != nullptr;
  auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double t0 = now();
  struct Ent { std::string name; int64_t ts, wall, mtime; uint64_t ino, size, f8; uint16_t sp[4]; uint8_t st; int64_t nf; };
  std::vector<Ent> ents;
  while (struct dirent* de = readdir(d)) {
    const char* nm = de->d_name;
    if (nm[0] == '.' && (nm[1] == 0 || (nm[1] == '.' && nm[2] == 0))) continue;
    Ent e; e.ts = 0; e.f8 = 0; e.nf = 0; e.wall = 0; e.ino = 0; e.size = 0; e.mtime = -1; memset(e.sp, 0, sizeof(e.sp));
    const size_t len = strlen(nm);
    const int st = parse_name(nm, len, &e.ts, e.sp, &e.f8, &e.nf);
    if (st == 0) continue;
    e.st = (uint8_t)st; e.name.assign(nm, len); e.ino = (uint64_t)de->d_ino;
    ents.push_back(std::move(e));
  }
  const double t1 = now();
  {
    // stat + local-time conversion of every entry, in parallel (a million fstatat calls are the cold listing's cost)
    const size_t total = ents.size();
    unsigned nt = std::thread::hardware_concurrency();
    if (nt > 32) nt = 32;
    if (nt < 1 || total < 4096) nt = 1;
    std::atomic<size_t> next{0};
    auto work = [&]() {
      for (;;) {
        const size_t i0 = next.fetch_add(512);
        if (i0 >= total) break;
        const size_t i1 = i0 + 512 < total ? i0 + 512 : total;
        for (size_t i = i0; i < i1; ++i) {
          Ent& e = ents[i];
          struct stat sb;
          if (!want_stat) {}                                                             // fei_read_dir_packed fills size / mtime from the open file
          else if (fstatat(dfd, e.name.c_str(), &sb, 0) != 0) { e.st = 2; }              // vanished / unreadable: Python reports it
          else { e.ino = sb.st_ino; e.size = (uint64_t)sb.st_size; e.mtime = (int64_t)sb.st_mtim.tv_sec * 1000000000ll + sb.st_mtim.tv_nsec; }
          if (e.st == 1) {                                           // datetime.fromtimestamp(ts): naive local wall clock (utils.py:94)
            if (!wall_of(e.ts, &e.wall)) e.st = 2;
          }
        }
      }
    };
    std::vector<std::thread> pool;
    for (unsigned t = 1; t < nt; ++t) pool.emplace_back(work);
    work();
    for (auto& t : pool) t.join();
  }
  closedir(d);
  const double t2 = now();
  // newest first, ties in readdir order (utils.py:251: sort(key=timestamp, reverse=True) is stable); entries Python must judge go last
  std::stable_sort(ents.begin(), ents.end(), [](const Ent& a, const Ent& b) { if (a.st != b.st) return a.st < b.st; return a.st == 1 && a.ts > b.ts; });
  const double t3 = now();
  fei_dirlist* l = new fei_dirlist();
  const size_t n = ents.size();
  l->name_off.reserve(n + 1); l->name_off.push_back(0);
  for (const Ent& e : ents) {
    l->blob += e.name; l->name_off.push_back(l->blob.size());
    l->ts.push_back(e.ts); l->wall.push_back(e.wall); l->mtime_ns.push_back(e.mtime); l->ino.push_back(e.ino); l->size.push_back(e.size);
    l->flags8.push_back(e.f8); l->status.push_back(e.st); l->flags_len.push_back(e.nf);
    for (int k = 0; k < 4; ++k) l->spans.push_back(e.sp[k]);
  }
  *out = l;
  if (timing) fprintf(stderr, "[fei_dir_list] %zu entries: readdir+parse %.3f s, stat+localtime %.3f s, sort %.3f s, columns %.3f s\n", n, t1 - t0, t2 - t1, t3 - t2, now() - t3);
  return FEI_OK;
}

extern "C" int fei_dir_list(const char* path, fei_dirlist** out) { return dir_list(path, true, out); }
extern "C" int fei_dir_list_names(const char* path, fei_dirlist** out) { return dir_list(path, false, out); }

extern "C" int fei_dirlist_view_get(const fei_dirlist* l, fei_dirlist_view* v) {
  if (!l || !v) { set_error("null argument"); return FEI_E_BADARG; }
  v->n = l->ts.size();
  v->names = reinterpret_cast<const uint8_t*>(l->blob.data()); v->name_off = l->name_off.data();
  v->ts = l->ts.data(); v->wall = l->wall.data(); v->mtime_ns = l->mtime_ns.data(); v->ino = l->ino.data(); v->size = l->size.data();
  v->flags8 = l->flags8.data(); v->spans = l->spans.data(); v->status = l->status.data(); v->flags_len = l->flags_len.data();
  return FEI_OK;
}

extern "C" void fei_dirlist_free(fei_dirlist* l) { delete l; }

// ---- cold read without a stat pass: open, fstat, read, close per file (a path stat costs more than the other three together where
// system calls are expensive).  Sizes are only known once a file is open, so the bytes go into an ARENA: a worker opens a batch of
// files, reserves the batch's total with one atomic add on *cursor, and reads them there; begin[i] / len[i] say where file i landed.
// The arena is a large NORESERVE mapping (only the touched pages become resident), shared by all directories of a tree.
extern "C" int fei_host_arena_alloc(uint64_t bytes, int huge_pages, void** out) {
  if (!out || !bytes) { set_error("null argument"); return FEI_E_BADARG; }
  void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
  if (p == MAP_FAILED) { set_error("mmap of a %llu-byte arena: %s", (unsigned long long)bytes, strerror(errno)); return FEI_E_CAPACITY; }
#ifdef MADV_HUGEPAGE
  if (huge_pages) madvise(p, bytes, MADV_HUGEPAGE);                      // first touch (and the later unmap) by 2 MiB instead of 4 KiB where THP is "madvise"
#endif
  *out = p;
  return FEI_OK;
}
extern "C" int fei_host_arena_free(void* p, uint64_t bytes) {
  if (p && munmap(p, bytes) != 0) { set_error("munmap: %s", strerror(errno)); return FEI_E_BADARG; }
  return FEI_OK;
}

extern "C" int fei_read_dir_packed(const char* dir, const uint8_t* names, const uint64_t* name_off, uint64_t n, uint8_t* arena, uint64_t arena_cap,
                                   uint64_t* cursor, uint64_t max_file_bytes, int threads, uint64_t* begin, uint64_t* len, uint64_t* ino,
                                   int64_t* mtime_ns, int32_t* err) {
  if (!dir || !cursor || (n && (!names || !name_off || !arena || !begin || !len || !ino || !mtime_ns || !err))) { set_error("null argument"); return FEI_E_BADARG; }
  if (threads < 1) threads = 1;
  if ((uint64_t)threads > n) threads = n ? (int)n : 1;
  const int dfd = open(dir, O_RDONLY | O_DIRECTORY);
  if (dfd < 0) { set_error("open(%s): %s", dir, strerror(errno)); return FEI_E_BADARG; }
  std::atomic<uint64_t> next{0};
  constexpr uint64_t kBatch = 64;
  auto work = [&]() {
    if (!getenv("FEI_SHARED_FDS")) unshare(CLONE_FILES);               // private fd table per worker, see fei_read_files
    std::string nm;
    int fds[kBatch]; uint64_t sz[kBatch];
    for (;;) {
      const uint64_t i0 = next.fetch_add(kBatch);
      if (i0 >= n) break;
      const uint64_t k = i0 + kBatch < n ? kBatch : n - i0;
      uint64_t total = 0;
      for (uint64_t j = 0; j < k; ++j) {
        const uint64_t i = i0 + j;
        begin[i] = 0; len[i] = 0; err[i] = 0; ino[i] = 0; mtime_ns[i] = -1; sz[j] = 0;
        nm.assign(reinterpret_cast<const char*>(names) + name_off[i], name_off[i + 1] - name_off[i]);
        fds[j] = openat(dfd, nm.c_str(), O_RDONLY);
        if (fds[j] < 0) { err[i] = errno; continue; }
        struct stat sb;
        if (fstat(fds[j], &sb) != 0) { err[i] = errno; close(fds[j]); fds[j] = -1; continue; }
        ino[i] = sb.st_ino; mtime_ns[i] = (int64_t)sb.st_mtim.tv_sec * 1000000000ll + sb.st_mtim.tv_nsec;
        if (!S_ISREG(sb.st_mode)) { err[i] = S_ISDIR(sb.st_mode) ? EISDIR : EINVAL; close(fds[j]); fds[j] = -1; continue; }
        if ((uint64_t)sb.st_size > max_file_bytes) { err[i] = EFBIG; len[i] = (uint64_t)sb.st_size; close(fds[j]); fds[j] = -1; continue; }
        sz[j] = (uint64_t)sb.st_size; total += sz[j];
      }
      uint64_t at = __atomic_fetch_add(cursor, total, __ATOMIC_RELAXED);
      const bool fits = at + total <= arena_cap;
      for (uint64_t j = 0; j < k; ++j) {
        const uint64_t i = i0 + j;
        if (fds[j] < 0) continue;
        if (!fits) { err[i] = ENOMEM; close(fds[j]); continue; }
        uint64_t done = 0;
        while (done < sz[j]) {
          const ssize_t r = pread(fds[j], arena + at + done, sz[j] - done, (off_t)done);
          if (r < 0) { if (errno == EINTR) continue; err[i] = errno; break; }
          if (r == 0) break;                                         // shrank since fstat: what is there is the file
          done += (uint64_t)r;
        }
        begin[i] = at; len[i] = done; at += sz[j];
        close(fds[j]);
      }
    }
  };
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t) pool.emplace_back(work);
  for (auto& t : pool) t.join();
  close(dfd);
  return FEI_OK;
}

// Reads n files of one directory into dst at dst_off[i] (capacity dst_off[i+1] - dst_off[i]): `threads` workers, open + pread +
// close each.  got[i] = bytes read (a file that grew since it was listed is cut at the listed size: its new (size, mtime) makes the
// next sync read it again), err[i] = errno or 0.
extern "C" int fei_read_files(const char* dir, const uint8_t* names, const uint64_t* name_off, uint64_t n, uint8_t* dst, const uint64_t* dst_off,
                              int threads, uint64_t* got, int32_t* err) {
  if (!dir || (n && (!names || !name_off || !dst || !dst_off || !got || !err))) { set_error("null argument"); return FEI_E_BADARG; }
  if (threads < 1) threads = 1;
  if ((uint64_t)threads > n) threads = n ? (int)n : 1;
  const int dfd = open(dir, O_RDONLY | O_DIRECTORY);
  if (dfd < 0) { set_error("open(%s): %s", dir, strerror(errno)); return FEI_E_BADARG; }
  std::atomic<uint64_t> next{0};
  auto work = [&](bool own_fd_table) {
    // every open / close takes the process-wide fd-table lock; a worker with a private copy of the table (unshare(CLONE_FILES):
    // dfd stays valid in the copy, the copy dies with the thread) does not contend with the others
    if (own_fd_table && !getenv("FEI_SHARED_FDS")) unshare(CLONE_FILES);
    std::string nm;
    for (;;) {
      const uint64_t i0 = next.fetch_add(64);
      if (i0 >= n) break;
      const uint64_t i1 = i0 + 64 < n ? i0 + 64 : n;
      for (uint64_t i = i0; i < i1; ++i) {
        nm.assign(reinterpret_cast<const char*>(names) + name_off[i], name_off[i + 1] - name_off[i]);
        got[i] = 0; err[i] = 0;
        const int fd = openat(dfd, nm.c_str(), O_RDONLY);
        if (fd < 0) { err[i] = errno; continue; }
        const uint64_t cap = dst_off[i + 1] - dst_off[i];
        uint64_t done = 0;
        while (done < cap) {
          const ssize_t r = pread(fd, dst + dst_off[i] + done, cap - done, (off_t)done);
          if (r < 0) { if (errno == EINTR) continue; err[i] = errno; break; }
          if (r == 0) break;
          done += (uint64_t)r;
        }
        got[i] = done;
        close(fd);
      }
    }
  };
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t) pool.emplace_back(work, true);     // the caller's thread keeps the shared table and only waits
  for (auto& t : pool) t.join();
  close(dfd);
  return FEI_OK;
}

// Test / bench tooling: writes n files (contents blob/off, names names/name_off) into `dir` with `threads` workers.
extern "C" int fei_write_files(const char* dir, const uint8_t* names, const uint64_t* name_off, const uint8_t* blob, const uint64_t* off, uint64_t n, int threads) {
  if (!dir || (n && (!names || !name_off || !blob || !off))) { set_error("null argument"); return FEI_E_BADARG; }
  if (threads < 1) threads = 1;
  const int dfd = open(dir, O_RDONLY | O_DIRECTORY);
  if (dfd < 0) { set_error("open(%s): %s", dir, strerror(errno)); return FEI_E_BADARG; }
  std::atomic<uint64_t> next{0};
  std::atomic<int> bad{0};
  auto work = [&]() {
    std::string nm;
    for (;;) {
      const uint64_t i = next.fetch_add(1);
      if (i >= n) break;
      nm.assign(reinterpret_cast<const char*>(names) + name_off[i], name_off[i + 1] - name_off[i]);
      const int fd = openat(dfd, nm.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
      if (fd < 0) { bad = errno; continue; }
      uint64_t done = 0; const uint64_t len = off[i + 1] - off[i];
      while (done < len) { const ssize_t r = write(fd, blob + off[i] + done, len - done); if (r <= 0) { if (errno == EINTR) continue; bad = errno ? errno : EIO; break; } done += (uint64_t)r; }
      close(fd);
    }
  };
  std::vector<std::thread> pool;
  for (int t = 1; t < threads; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
  close(dfd);
  if (bad) { set_error("writing files into %s: %s", dir, strerror(bad)); return FEI_E_BADARG; }
  return FEI_OK;
}

// ---------------------------------------------------------------- synthetic tree on disk (tests / bench tooling)
#include "synth.cuh"
#include <sys/types.h>

// Writes records [first, first + n) of the deterministic synthetic Memdir (synth.cuh) as Maildir files under `base`
// ("<ts>.<uid>.<hostname>:2,<flags>" in <folder>/<status>/, content = header text + "---\n" + body, utils.py:129-151), `threads`
// workers.  The directories must exist.  Same bytes as fei_b200.synth.write_memdir(record(seed, i)).
extern "C" int fei_synth_write_tree(const char* base, const char* hostname, uint64_t seed, uint64_t first, uint64_t n, int threads) {
  if (!base || !hostname) { set_error("null argument"); return FEI_E_BADARG; }
  static const char* const kFolders[4] = {"", ".Projects/Python", ".Projects/AI", ".ToDoLater/Learning"};
  static const char* const kStatus[3] = {"cur", "new", "tmp"};
  if (threads < 1) threads = 1;
  std::atomic<uint64_t> next{0};
  std::atomic<int> bad{0};
  auto work = [&]() {
    std::vector<uint8_t> buf;
    std::string path;
    for (;;) {
      const uint64_t k0 = next.fetch_add(256);
      if (k0 >= n) break;
      const uint64_t k1 = k0 + 256 < n ? k0 + 256 : n;
      for (uint64_t k = k0; k < k1; ++k) {
        const uint64_t i = first + k;
        fei::CountSink ch; feisynth::gen_header(ch, seed, i);
        fei::CountSink cb; feisynth::gen_body(cb, seed, i);
        buf.resize((size_t)ch.n + 4 + cb.n);
        { fei::WriteSink w{buf.data()}; feisynth::gen_header(w, seed, i); }
        memcpy(buf.data() + ch.n, "---\n", 4);
        { fei::WriteSink w{buf.data() + ch.n + 4}; feisynth::gen_body(w, seed, i); }
        const feisynth::RecMeta m = feisynth::gen_meta(seed, i);
        char name[160];
        snprintf(name, sizeof(name), "%lld.%.8s.%s:2,%.*s", (long long)m.ts, m.uid, hostname, (int)m.nflags, m.flags);
        path.assign(base);
        if (kFolders[m.folder][0]) { path += '/'; path += kFolders[m.folder]; }
        path += '/'; path += kStatus[m.status]; path += '/'; path += name;
        const int fd = open(path.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
        if (fd < 0) { bad = errno; continue; }
        size_t done = 0;
        while (done < buf.size()) { const ssize_t r = write(fd, buf.data() + done, buf.size() - done); if (r <= 0) { if (errno == EINTR) continue; bad = errno ? errno : EIO; break; } done += (size_t)r; }
        close(fd);
      }
    }
  };
  std::vector<std::thread> pool;
  for (int t = 1; t < threads; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
  if (bad) { set_error("writing the synthetic tree under %s: %s", base, strerror(bad)); return FEI_E_BADARG; }
  return FEI_OK;
}
