// Host side of the synthetic generators (synth.cuh compiled for the CPU):
//   fei_synth_record_host / fei_synth_block_host  — one record / block, for fixtures
//   fei_chain_synth                                — a linked synthetic Memorychain
// A hash chain is inherently sequential (block i's text contains block i-1's hash), so
// the synthetic chain is built on the host; the small SHA-256 below exists only to
// *construct* that test/bench input and is not reachable from any validate entry point.
#include "common.h"
#include "chain_json.h"
#include "synth.cuh"
#include <string.h>
#include <string>
#include <vector>

namespace {

struct HostSha {
  static uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
  static void digest(const uint8_t* msg, size_t len, uint8_t out[32]) {
    static const uint32_t K[64] = {
        0x428a2f98,0x71374491,0xb5c0fbcf,0xe9b5dba5,0x3956c25b,0x59f111f1,0x923f82a4,0xab1c5ed5,0xd807aa98,0x12835b01,0x243185be,0x550c7dc3,0x72be5d74,0x80deb1fe,0x9bdc06a7,0xc19bf174,
        0xe49b69c1,0xefbe4786,0x0fc19dc6,0x240ca1cc,0x2de92c6f,0x4a7484aa,0x5cb0a9dc,0x76f988da,0x983e5152,0xa831c66d,0xb00327c8,0xbf597fc7,0xc6e00bf3,0xd5a79147,0x06ca6351,0x14292967,
        0x27b70a85,0x2e1b2138,0x4d2c6dfc,0x53380d13,0x650a7354,0x766a0abb,0x81c2c92e,0x92722c85,0xa2bfe8a1,0xa81a664b,0xc24b8b70,0xc76c51a3,0xd192e819,0xd6990624,0xf40e3585,0x106aa070,
        0x19a4c116,0x1e376c08,0x2748774c,0x34b0bcb5,0x391c0cb3,0x4ed8aa4a,0x5b9cca4f,0x682e6ff3,0x748f82ee,0x78a5636f,0x84c87814,0x8cc70208,0x90befffa,0xa4506ceb,0xbef9a3f7,0xc67178f2};
    uint32_t h[8] = {0x6a09e667,0xbb67ae85,0x3c6ef372,0xa54ff53a,0x510e527f,0x9b05688c,0x1f83d9ab,0x5be0cd19};
    size_t total = ((len + 9 + 63) / 64) * 64;
    std::vector<uint8_t> buf(total, 0);
    memcpy(buf.data(), msg, len);
    buf[len] = 0x80;
    uint64_t bits = (uint64_t)len * 8;
    for (int k = 0; k < 8; ++k) buf[total - 1 - k] = (uint8_t)(bits >> (8 * k));
    for (size_t off = 0; off < total; off += 64) {
      uint32_t w[64];
      for (int t = 0; t < 16; ++t) w[t] = (uint32_t)buf[off + 4 * t] << 24 | (uint32_t)buf[off + 4 * t + 1] << 16 | (uint32_t)buf[off + 4 * t + 2] << 8 | buf[off + 4 * t + 3];
      for (int t = 16; t < 64; ++t) {
        uint32_t s0 = rotr(w[t - 15], 7) ^ rotr(w[t - 15], 18) ^ (w[t - 15] >> 3);
        uint32_t s1 = rotr(w[t - 2], 17) ^ rotr(w[t - 2], 19) ^ (w[t - 2] >> 10);
        w[t] = w[t - 16] + s0 + w[t - 7] + s1;
      }
      uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
      for (int t = 0; t < 64; ++t) {
        uint32_t t1 = hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K[t] + w[t];
        uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
      }
      h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
    }
    for (int k = 0; k < 8; ++k) { out[4 * k] = (uint8_t)(h[k] >> 24); out[4 * k + 1] = (uint8_t)(h[k] >> 16); out[4 * k + 2] = (uint8_t)(h[k] >> 8); out[4 * k + 3] = (uint8_t)h[k]; }
  }
};

const char* const kTaskStates[6] = {"proposed", "accepted", "in_progress", "solution_proposed", "completed", "rejected"};
const char* const kDifficulties[5] = {"easy", "medium", "hard", "very_hard", "extreme"};
const char kResponsible[] = "3f0c9a52-7d41-4e8b-9c1d-5a6b7c8d9e0f";
const char kProposer[] = "b7e1d2c3-4a5f-4b6c-8d7e-0f1a2b3c4d5e";

}  // namespace

extern "C" int fei_synth_record_host(uint64_t seed, uint64_t i,
                                     uint8_t* hdr, uint32_t hdr_cap, uint32_t* hdr_len,
                                     uint8_t* body, uint32_t body_cap, uint32_t* body_len,
                                     int64_t* ts, char* uid8, char* flags4, uint8_t* nflags, uint8_t* status, uint8_t* folder) {
  using namespace feisynth;
  fei::CountSink ch; gen_header(ch, seed, i);
  fei::CountSink cb; gen_body(cb, seed, i);
  if (hdr_len) *hdr_len = ch.n;
  if (body_len) *body_len = cb.n;
  if ((hdr && ch.n > hdr_cap) || (body && cb.n > body_cap)) { fei::set_error("record %llu needs %u header / %u body bytes", (unsigned long long)i, ch.n, cb.n); return FEI_E_CAPACITY; }
  if (hdr) { fei::WriteSink w{hdr}; gen_header(w, seed, i); }
  if (body) { fei::WriteSink w{body}; gen_body(w, seed, i); }
  RecMeta m = gen_meta(seed, i);
  if (ts) *ts = m.ts;
  if (uid8) memcpy(uid8, m.uid, 8);
  if (flags4) memcpy(flags4, m.flags, 4);
  if (nflags) *nflags = m.nflags;
  if (status) *status = m.status;
  if (folder) *folder = m.folder;
  return FEI_OK;
}

extern "C" int fei_synth_block_host(uint64_t seed, uint64_t i, double* timestamp, char* memory_id8,
                                    uint8_t* task_state, uint8_t* difficulty, uint8_t* is_task) {
  feisynth::ChainBlockSpec b = feisynth::gen_block(seed, i);
  if (timestamp) *timestamp = b.timestamp;
  if (memory_id8) memcpy(memory_id8, b.memory_id, 8);
  if (task_state) *task_state = b.task_state;
  if (difficulty) *difficulty = b.difficulty;
  if (is_task) *is_task = b.is_task;
  return FEI_OK;
}

// Builds blocks [0, first+n) sequentially (needed for the links), keeps [first, first+n)
// plus the one-block halo before it when first > 0 (position 0 of a resident chain is
// never checked, exactly like the genesis block).
extern "C" int fei_chain_synth(fei_chain* ch, uint64_t seed, uint64_t first, uint64_t n, int64_t corrupt_at) {
  if (!ch) { fei::set_error("null chain"); return FEI_E_BADARG; }
  uint64_t keep_from = first > 0 ? first - 1 : 0;
  uint64_t end = first + n;
  std::vector<uint8_t> msgs, hashes, prevs;
  std::vector<uint64_t> moff{0}, hoff{0}, poff{0};
  msgs.reserve((end - keep_from) * 368);
  std::string prev_hash = "0";                       // genesis previous_hash (memorychain.py:546)
  fei::ByteVec one; std::vector<uint64_t> one_off;
  static const char hx[] = "0123456789abcdef";
  for (uint64_t i = 0; i < end; ++i) {
    feisynth::ChainBlockSpec b = feisynth::gen_block(seed, i);
    const char* diff = kDifficulties[b.difficulty];
    const char* tstate = kTaskStates[b.task_state];
    uint64_t idx = i, nonce = 0, tsbits; memcpy(&tsbits, &b.timestamp, 8);
    uint64_t o_diff[2] = {0, strlen(diff)}, o_mid[2] = {0, 8}, o_prev[2] = {0, prev_hash.size()}, o_prop[2] = {0, sizeof(kProposer) - 1},
             o_resp[2] = {0, sizeof(kResponsible) - 1}, o_ts[2] = {0, strlen(tstate)};
    fei_json_col cols[FEI_CHAIN_NCOLS] = {
        {nullptr, FEI_J_STR, nullptr, (const uint8_t*)diff, o_diff},
        {nullptr, FEI_J_INT, &idx, nullptr, nullptr},
        {nullptr, FEI_J_STR, nullptr, (const uint8_t*)b.memory_id, o_mid},
        {nullptr, FEI_J_INT, &nonce, nullptr, nullptr},
        {nullptr, FEI_J_STR, nullptr, (const uint8_t*)prev_hash.data(), o_prev},
        {nullptr, FEI_J_STR, nullptr, (const uint8_t*)kProposer, o_prop},
        {nullptr, FEI_J_STR, nullptr, (const uint8_t*)kResponsible, o_resp},
        {nullptr, FEI_J_NULL, nullptr, nullptr, nullptr},
        {nullptr, FEI_J_STR, nullptr, (const uint8_t*)tstate, o_ts},
        {nullptr, FEI_J_FLOAT, &tsbits, nullptr, nullptr}};
    int rc = fei::serialize_chain_cols(cols, 1, one, one_off);
    if (rc != FEI_OK) return rc;
    uint8_t dg[32];
    HostSha::digest(one.data(), one.size(), dg);
    char hex[64];
    for (int k = 0; k < 32; ++k) { hex[2 * k] = hx[dg[k] >> 4]; hex[2 * k + 1] = hx[dg[k] & 15]; }
    if (i >= keep_from) {
      msgs.insert(msgs.end(), one.begin(), one.end()); moff.push_back(msgs.size());
      prevs.insert(prevs.end(), prev_hash.begin(), prev_hash.end()); poff.push_back(prevs.size());
      size_t at = hashes.size();
      hashes.insert(hashes.end(), hex, hex + 64); hoff.push_back(hashes.size());
      if (corrupt_at >= 0 && (uint64_t)corrupt_at == i) hashes[at + 5] = hashes[at + 5] == 'a' ? 'b' : 'a';
    }
    prev_hash.assign(hex, 64);
  }
  return fei_chain_load_msgs(ch, msgs.data(), moff.data(), hashes.data(), hoff.data(), prevs.data(), poff.data(), end - keep_from, keep_from);
}
