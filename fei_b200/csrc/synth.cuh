// Deterministic synthetic Memdir / Memorychain generator, usable from host and device.
//
// Record i of a corpus is a pure function of (seed, i): a counter-based RNG
// (splitmix64 keyed on seed and i) drives the same *distributions* as the
// reference's unseeded sample generator (memdir_tools/create_samples.py:82-195,
// :216-239; vocabulary :20-80).  The same source is compiled for the host
// (fixtures for the oracle / reference, CPU baseline samples) and for the GPU
// (10M..100M-entry corpora generated straight into HBM), so both sides see
// byte-identical records.
//
// A record is emitted as two pieces, exactly what the packer would produce from
// the on-disk file  hdr + "---" + "\n" + body :
//   hdr  = header text before the first "---" (parse_memory_content,
//          memdir_tools/utils.py:105-118), newline-terminated lines "Key: value"
//   body = text after the separator, already .strip()ped (utils.py:120)
#pragma once
#include <stdint.h>
#include "sink.cuh"

namespace feisynth {
using fei::put_lit;

struct Word { uint8_t len; char s[55]; };
#define FW(x) { (uint8_t)(sizeof(x) - 1), x }

// Vocabulary lists (values = data of the reference generator's distributions).
#define FEI_TAGS \
  FW("work"), FW("personal"), FW("research"), FW("learning"), FW("project"), FW("idea"), FW("meeting"), \
  FW("conference"), FW("book"), FW("coding"), FW("design"), FW("planning"), FW("review"), FW("tutorial"), \
  FW("howto"), FW("bug"), FW("feature"), FW("documentation"), FW("testing"), FW("production"), \
  FW("development"), FW("performance"), FW("security"), FW("code"), FW("architecture"), FW("database"), \
  FW("frontend"), FW("backend"), FW("devops"), FW("ui"), FW("ux"), FW("mobile"), FW("web"), FW("desktop"), \
  FW("algorithm"), FW("datastructure"), FW("python"), FW("javascript"), FW("rust"), FW("go"), FW("react"), \
  FW("angular"), FW("vue"), FW("node"), FW("django"), FW("flask"), FW("spring"), FW("docker"), FW("kubernetes"), \
  FW("aws"), FW("azure"), FW("gcp"), FW("terraform"), FW("ansible"), FW("git"), FW("cicd"), FW("cloud"), FW("agile")
#define FEI_NTAGS 58
#define FEI_TOPICS \
  FW("Machine Learning"), FW("Data Structures"), FW("Algorithms"), FW("Python"), FW("JavaScript"), \
  FW("Rust"), FW("Go"), FW("Databases"), FW("Cloud Computing"), FW("Web Development"), FW("DevOps"), \
  FW("Security"), FW("Blockchain"), FW("UI/UX Design"), FW("Mobile Development"), FW("Testing"), \
  FW("Big Data"), FW("Microservices"), FW("Docker"), FW("Kubernetes"), FW("React"), FW("Angular"), \
  FW("Vue.js"), FW("Node.js"), FW("Django"), FW("Flask"), FW("Spring Boot"), FW("Natural Language Processing"), \
  FW("Computer Vision"), FW("Reinforcement Learning"), FW("Neural Networks"), FW("Git"), FW("CI/CD")
#define FEI_NTOPICS 33
#define FEI_BOOKS \
  FW("Clean Code"), FW("The Pragmatic Programmer"), FW("Design Patterns"), FW("Refactoring"), \
  FW("Domain-Driven Design"), FW("The Mythical Man-Month"), FW("Soft Skills"), FW("Code Complete"), \
  FW("Working Effectively with Legacy Code"), FW("The Phoenix Project"), FW("Accelerate"), \
  FW("Building Microservices"), FW("Site Reliability Engineering"), FW("The DevOps Handbook"), \
  FW("Continuous Delivery"), FW("Patterns of Enterprise Application Architecture")
#define FEI_NBOOKS 16
#define FEI_PROJECTS \
  FW("Knowledge Management System"), FW("Task Tracker"), FW("Personal Finance App"), \
  FW("Social Network"), FW("E-commerce Platform"), FW("Content Management System"), \
  FW("API Gateway"), FW("Authentication Service"), FW("Data Pipeline"), FW("Analytics Dashboard"), \
  FW("Search Engine"), FW("Chat Application"), FW("Recommendation System"), FW("Mobile Game"), \
  FW("Productivity Tool"), FW("Browser Extension"), FW("Desktop Application")
#define FEI_NPROJECTS 17
#define FEI_EVENTS \
  FW("PyCon 2024"), FW("KubeCon"), FW("AWS Summit"), FW("Google I/O"), FW("Apple WWDC"), \
  FW("GitHub Universe"), FW("Docker Con"), FW("React Conf"), FW("DevOps Days"), FW("Rust Conf"), \
  FW("Node Congress"), FW("JS Conf"), FW("MongoDB World"), FW("PostgreSQL Conference"), \
  FW("Kafka Summit"), FW("TensorFlow Dev Summit"), FW("MLOps Summit")
#define FEI_NEVENTS 17
#define FEI_PEOPLE \
  FW("John Doe"), FW("Jane Smith"), FW("Elon Musk"), FW("Satya Nadella"), FW("Sundar Pichai"), \
  FW("Mark Zuckerberg"), FW("Jensen Huang"), FW("Sam Altman"), FW("Andrew Ng"), FW("Yann LeCun"), \
  FW("Martin Fowler"), FW("Kent Beck"), FW("Robert C. Martin"), FW("Linus Torvalds"), FW("Guido van Rossum")
#define FEI_NPEOPLE 15
#define FEI_SECTIONS \
  FW("Overview"), FW("Details"), FW("Implementation"), FW("Next Steps"), FW("Background"), \
  FW("Summary"), FW("Discussion"), FW("Key Points"), FW("Analysis"), FW("Observations"), \
  FW("Questions"), FW("Decisions"), FW("Action Items"), FW("Resources"), FW("References")
#define FEI_NSECTIONS 15
#define FEI_MISC \
  FW("high"), FW("medium"), FW("low"), /* 0..2 priorities */ \
  FW("active"), FW("pending"), FW("completed"), FW("in-progress"), FW("blocked"), FW("deferred"), /* 3..8 statuses */ \
  FW("Integration"), FW("Export"), FW("Import"), FW("View"), FW("Editor"), FW("Dashboard"), /* 9..14 feature kinds */ \
  FW("Build"), FW("Deploy"), FW("Configure"), FW("Optimize"), FW("Debug"), FW("Test"), FW("Design"), FW("Implement"), /* 15..22 actions */ \
  FW("Pasta"), FW("Pizza"), FW("Salad"), FW("Soup"), FW("Sandwich"), FW("Curry"), FW("Stir-fry") /* 23..29 foods */
#define FEI_NMISC 30

// One flat table; sub-ranges addressed by base index.
enum : int {
  B_TAGS = 0,
  B_TOPICS = B_TAGS + FEI_NTAGS,
  B_BOOKS = B_TOPICS + FEI_NTOPICS,
  B_PROJECTS = B_BOOKS + FEI_NBOOKS,
  B_EVENTS = B_PROJECTS + FEI_NPROJECTS,
  B_PEOPLE = B_EVENTS + FEI_NEVENTS,
  B_SECTIONS = B_PEOPLE + FEI_NPEOPLE,
  B_MISC = B_SECTIONS + FEI_NSECTIONS,
  N_WORDS = B_MISC + FEI_NMISC
};

static const Word h_words[N_WORDS] = { FEI_TAGS, FEI_TOPICS, FEI_BOOKS, FEI_PROJECTS, FEI_EVENTS, FEI_PEOPLE, FEI_SECTIONS, FEI_MISC };
#if defined(__CUDACC__)
__device__ const Word d_words[N_WORDS] = { FEI_TAGS, FEI_TOPICS, FEI_BOOKS, FEI_PROJECTS, FEI_EVENTS, FEI_PEOPLE, FEI_SECTIONS, FEI_MISC };
#endif

FEI_HD const Word& word(int i) {
#if defined(__CUDA_ARCH__)
  return d_words[i];
#else
  return h_words[i];
#endif
}

// ---------------------------------------------------------------- RNG
struct Rng {
  uint64_t s;
  FEI_HD Rng(uint64_t seed, uint64_t idx, uint64_t stream) {
    s = seed * 0x9E3779B97F4A7C15ull ^ (idx + 0x632BE59BD9B4E019ull) * 0xD1342543DE82EF95ull ^ stream * 0xA0761D6478BD642Full;
    next(); next();
  }
  FEI_HD uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  FEI_HD uint32_t below(uint32_t n) { return (uint32_t)(((next() >> 32) * (uint64_t)n) >> 32); }
  FEI_HD uint32_t range(uint32_t lo, uint32_t hi) { return lo + below(hi - lo + 1); }  // inclusive
  FEI_HD bool chance(uint32_t pct) { return below(100) < pct; }
};

// ---------------------------------------------------------------- writers (into a sink.cuh sink)
template <class S> FEI_HD void put_word(S& s, int wi) { const Word& w = word(wi); for (int k = 0; k < w.len; ++k) s.put(w.s[k]); }
template <class S> FEI_HD void put_word_lower(S& s, int wi, bool cap_first) {
  const Word& w = word(wi);
  for (int k = 0; k < w.len; ++k) {
    char c = w.s[k];
    if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
    if (k == 0 && cap_first && c >= 'a' && c <= 'z') c = (char)(c - 32);
    s.put(c);
  }
}
template <class S> FEI_HD void put_uint(S& s, uint32_t v, int width) {  // zero padded decimal
  char tmp[10]; int n = 0;
  do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
  for (int k = n; k < width; ++k) s.put('0');
  while (n) s.put(tmp[--n]);
}

// days since 1970-01-01 -> civil date (proleptic Gregorian)
FEI_HD void civil_from_days(int64_t z, int& y, unsigned& m, unsigned& d) {
  z += 719468;
  const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  const unsigned doe = (unsigned)(z - era * 146097);
  const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  y = (int)yoe + (int)era * 400;
  const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const unsigned mp = (5 * doy + 2) / 153;
  d = doy - (153 * mp + 2) / 5 + 1;
  m = mp < 10 ? mp + 3 : mp - 9;
  y += (m <= 2);
}
template <class S> FEI_HD void put_iso(S& s, int64_t days, uint32_t micros) {
  int y; unsigned m, d; civil_from_days(days, y, m, d);
  put_uint(s, (uint32_t)y, 4); s.put('-'); put_uint(s, m, 2); s.put('-'); put_uint(s, d, 2);
  put_lit(s, "T22:13:20."); put_uint(s, micros, 6);
}

// ---------------------------------------------------------------- record pieces
struct RecMeta {
  int64_t ts;         // filename timestamp (parse_memory_filename, utils.py:90)
  char uid[8];        // 8 lowercase hex
  char flags[4];      // 0..3 distinct of FRSP, sample order
  uint8_t nflags;
  uint8_t status;     // 0 = cur, 1 = new, 2 = tmp
  uint8_t folder;     // 0..3 -> "", ".Projects/Python", ".Projects/AI", ".ToDoLater/Learning"
};

constexpr int64_t kBaseTs = 1700000000;     // 2023-11-14T22:13:20Z
constexpr int64_t kBaseDay = 19675;         // days since epoch of kBaseTs

FEI_HD RecMeta gen_meta(uint64_t seed, uint64_t i) {
  Rng r(seed, i, 1);
  RecMeta m;
  m.ts = kBaseTs + (int64_t)(i >> 2);       // 4 records per second: exercises stable tie order
  uint64_t u = r.next();
  for (int k = 0; k < 8; ++k) { unsigned nib = (unsigned)(u >> (4 * k)) & 15u; m.uid[k] = (char)(nib < 10 ? '0' + nib : 'a' + nib - 10); }
  m.nflags = 0;
  for (int k = 0; k < 4; ++k) m.flags[k] = 0;
  if (r.chance(30)) {                       // create_samples.py:226-231
    const char pool[4] = {'F', 'R', 'S', 'P'};
    unsigned want = r.below(4), used = 0;
    while (m.nflags < want) {
      unsigned c = r.below(4);
      if (used & (1u << c)) continue;
      used |= 1u << c; m.flags[m.nflags++] = pool[c];
    }
  }
  m.status = r.chance(80) ? 0 : 1;          // create_samples.py:238-239
  m.folder = (uint8_t)r.below(4);           // create_samples.py:218-219
  return m;
}

// Subject (create_samples.py:20-28, :138-159).  Written to `s`; identical text is
// needed by header and body, so callers run it twice with the same Rng state.
template <class S> FEI_HD void gen_subject(S& s, Rng r) {
  unsigned t = r.below(20);
  switch (t) {
    case 0: put_lit(s, "Weekly Planning Session"); break;
    case 1: put_lit(s, "Meeting Notes: Product Team"); break;
    case 2: put_lit(s, "Book Review: "); put_word(s, B_BOOKS + r.below(FEI_NBOOKS)); break;
    case 3: put_lit(s, "Research on "); put_word(s, B_TOPICS + r.below(FEI_NTOPICS)); break;
    case 4: put_lit(s, "Project Idea: "); put_word(s, B_PROJECTS + r.below(FEI_NPROJECTS)); break;
    case 5: put_lit(s, "Learning Notes: "); put_word(s, B_TOPICS + r.below(FEI_NTOPICS)); break;
    case 6: put_lit(s, "Conference Notes: "); put_word(s, B_EVENTS + r.below(FEI_NEVENTS)); break;
    case 7: put_lit(s, "Bug Report: Issue #"); put_uint(s, r.range(100, 999), 3); break;
    case 8: put_lit(s, "Feature Request: "); put_word(s, B_PROJECTS + r.below(FEI_NPROJECTS)); s.put(' '); put_word(s, B_MISC + 9 + r.below(6)); break;
    case 9: put_lit(s, "Technical Design: "); put_word(s, B_PROJECTS + r.below(FEI_NPROJECTS)); break;
    case 10: put_lit(s, "Interview with "); put_word(s, B_PEOPLE + r.below(FEI_NPEOPLE)); break;
    case 11: put_lit(s, "Analysis of "); put_word(s, B_TOPICS + r.below(FEI_NTOPICS)); break;
    case 12: put_lit(s, "Quick Thoughts on "); put_word(s, B_TOPICS + r.below(FEI_NTOPICS)); break;
    case 13: put_lit(s, "Tutorial: How to "); put_word(s, B_MISC + 15 + r.below(8)); s.put(' '); put_word(s, B_PROJECTS + r.below(FEI_NPROJECTS)); break;
    case 14: put_lit(s, "Summary of "); put_word(s, B_EVENTS + r.below(FEI_NEVENTS)); break;
    case 15: put_lit(s, "Reflections on "); put_word(s, B_TOPICS + r.below(FEI_NTOPICS)); break;
    case 16: put_lit(s, "Brainstorming Session: "); put_word(s, B_TOPICS + r.below(FEI_NTOPICS)); break;
    case 17: put_lit(s, "Debugging Notes: Issue #"); put_uint(s, r.range(100, 999), 3); break;
    case 18: put_lit(s, "Code Review: "); put_word(s, B_PROJECTS + r.below(FEI_NPROJECTS)); break;
    default: put_lit(s, "Recipe: "); put_word(s, B_MISC + 23 + r.below(7)); break;
  }
}

// Header text: "Key: value\n" lines (create_memory_content, utils.py:129-132, plus the
// "\n" that precedes the "---" separator).  create_samples.py:161-195.
template <class S> FEI_HD void gen_header(S& s, uint64_t seed, uint64_t i) {
  Rng rs(seed, i, 2);                      // subject stream (shared with body)
  Rng r(seed, i, 3);
  put_lit(s, "Subject: "); gen_subject(s, rs); s.put('\n');
  put_lit(s, "Tags: ");
  {
    unsigned ntags = r.range(2, 5);
    uint64_t used = 0;
    for (unsigned k = 0; k < ntags;) {
      unsigned t = r.below(FEI_NTAGS);
      if (used & (1ull << t)) continue;
      used |= 1ull << t;
      if (k) s.put(',');
      put_word(s, B_TAGS + t);
      ++k;
    }
  }
  s.put('\n');
  put_lit(s, "Priority: "); put_word(s, B_MISC + r.below(3)); s.put('\n');
  put_lit(s, "Status: "); put_word(s, B_MISC + 3 + r.below(6)); s.put('\n');
  put_lit(s, "Date: "); { int dd = (int)r.below(61) - 30; uint32_t us = r.below(1000000); put_iso(s, kBaseDay + dd, us); } s.put('\n');
  if (r.chance(30)) { put_lit(s, "Due: "); uint32_t dd = r.range(1, 90); uint32_t us = r.below(1000000); put_iso(s, kBaseDay + dd, us); s.put('\n'); }
  if (r.chance(20)) { put_lit(s, "Author: "); put_word(s, B_PEOPLE + r.below(FEI_NPEOPLE)); s.put('\n'); }
  if (r.chance(10)) { put_lit(s, "Version: "); put_uint(s, r.below(3), 1); s.put('.'); put_uint(s, r.below(10), 1); s.put('.'); put_uint(s, r.below(10), 1); s.put('\n'); }
}

// One sentence: `nw` distinct items of TAGS+TOPICS joined by ' ', str.capitalize()d,
// plus '.' (create_samples.py:94-97).
template <class S> FEI_HD void gen_sentence(S& s, Rng& r, unsigned nw) {
  uint64_t used0 = 0, used1 = 0;
  for (unsigned k = 0; k < nw;) {
    unsigned t = r.below(FEI_NTAGS + FEI_NTOPICS);
    uint64_t bit = 1ull << (t & 63);
    uint64_t& u = (t < 64) ? used0 : used1;
    if (u & bit) continue;
    u |= bit;
    if (k) s.put(' ');
    put_word_lower(s, t, k == 0);          // TAGS and TOPICS are adjacent in the flat table
    ++k;
  }
  s.put('.');
}

// Body, already stripped (create_samples.py:82-133).
template <class S> FEI_HD void gen_body(S& s, uint64_t seed, uint64_t i) {
  Rng rs(seed, i, 2);
  Rng r(seed, i, 4);
  put_lit(s, "# "); gen_subject(s, rs); put_lit(s, "\n\n");
  unsigned nsec = r.range(2, 4);
  unsigned nintro = r.range(2, 4);
  for (unsigned k = 0; k < nintro; ++k) { if (k) s.put(' '); gen_sentence(s, r, r.range(10, 20)); }
  // Separators are emitted *before* each element so the text ends without a
  // trailing newline (the reference joins with "\n" and the parser strips).
  for (unsigned sec = 0; sec < nsec; ++sec) {
    put_lit(s, "\n\n## "); put_word(s, B_SECTIONS + r.below(FEI_NSECTIONS));
    unsigned npar = r.range(1, 3);
    for (unsigned p = 0; p < npar; ++p) {
      put_lit(s, "\n\n");
      unsigned ns = r.range(3, 6);
      for (unsigned k = 0; k < ns; ++k) { if (k) s.put(' '); gen_sentence(s, r, r.range(8, 16)); }
    }
    if (r.chance(50)) {
      put_lit(s, "\n\n");
      unsigned ni = r.range(3, 6);
      for (unsigned k = 0; k < ni; ++k) {
        put_lit(s, "\n- ");
        unsigned pick = r.below(FEI_NTOPICS + FEI_NPROJECTS + FEI_NBOOKS);
        int wi = pick < FEI_NTOPICS ? B_TOPICS + (int)pick
               : pick < FEI_NTOPICS + FEI_NPROJECTS ? B_PROJECTS + (int)(pick - FEI_NTOPICS)
               : B_BOOKS + (int)(pick - FEI_NTOPICS - FEI_NPROJECTS);
        put_word(s, wi);
      }
    }
  }
}

// ---------------------------------------------------------------- chain blocks
// Synthetic Memorychain block i (SURVEY.md 8(d) cfg 4).  Only the fields that
// MemoryBlock.calculate_hash reads (memdir_tools/memorychain.py:117-128).
struct ChainBlockSpec {
  uint64_t index;
  double timestamp;     // 1.7e9 + i + u(0,1), microsecond grid so repr() is short
  char memory_id[8];
  uint8_t task_state;   // index into kTaskStates
  uint8_t difficulty;   // index into kDifficulties
  uint8_t is_task;
};

FEI_HD ChainBlockSpec gen_block(uint64_t seed, uint64_t i) {
  Rng r(seed, i, 7);
  ChainBlockSpec b;
  b.index = i;
  b.timestamp = 1700000000.0 + (double)i + (double)r.below(1000000) * 1e-6;
  uint64_t u = r.next();
  for (int k = 0; k < 8; ++k) { unsigned nib = (unsigned)(u >> (4 * k)) & 15u; b.memory_id[k] = (char)(nib < 10 ? '0' + nib : 'a' + nib - 10); }
  b.is_task = r.chance(10) ? 1 : 0;
  b.task_state = b.is_task ? (uint8_t)r.below(6) : 0;     // 0 = "proposed" (default, memorychain.py:104)
  b.difficulty = b.is_task ? (uint8_t)r.below(5) : 1;     // 1 = "medium"  (default, memorychain.py:102)
  return b;
}

}  // namespace feisynth
