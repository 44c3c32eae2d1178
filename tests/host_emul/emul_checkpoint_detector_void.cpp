// TEST-ONLY host build of the checkpoint format with the detector void (checkpoint.cpp, format version 4): a file of a
// given fingerprint is written to memory and read back, so the version choice, the counter section's length, the round
// trip and the named refusal can be checked without a GPU; never linked into libpumitally.so.
#include <cstring>
#include <string>
#include <vector>

#include "checkpoint.hpp"

using namespace ptb::ckpt;

namespace {
Fingerprint fp(int32_t det_void) {
  Fingerprint f;
  f.nelems = 10;
  f.nverts = 8;
  f.batch_stats = 1;
  f.det_xyz = {0.5, 1.5, -2.0, 100.0, 0.0, 3.0};  // the second detector outside the mesh
  f.det_r0 = {0.0, 0.25};
  f.sigma_crc = 0x1234abcdu;
  f.det_void = uint32_t(det_void);
  return f;
}
}  // namespace

extern "C" {
// A file with an open batch of 4 doubles, statistics of 4, det_len 6 and the detector counters (the values i + 0.5 in
// every double section, i + 1 in the counters).  Returns its size; out[cap].
int64_t ptb_ckpt_void_write(int32_t det_void, uint8_t *out, int64_t cap) {
  std::vector<uint8_t> b;
  Writer w([&](const void *p, size_t n) { b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n); return true; },
           [&](uint64_t off, const void *p, size_t n) { std::memcpy(b.data() + off, p, n); return true; });
  Header h;
  h.batches = 2;
  h.open = 1;
  h.open_len = 4;
  h.stats_len = 4;
  h.det_len = 6;
  h.det_words = uint32_t(det_void ? kDetCountWordsVoid : kDetCountWords);
  if (!w.begin(h, fp(det_void))) return -1;
  for (const auto &s : sections_of(h)) {
    std::vector<uint64_t> v(s.second / 8);
    for (size_t i = 0; i < v.size(); ++i) {
      const double x = double(i) + 0.5;
      if (s.first == kDetCounts) v[i] = i + 1;
      else std::memcpy(&v[i], &x, 8);
    }
    if (!w.section(s.first, s.second, 64, [&](size_t, uint64_t off, size_t) { return (const void *)((const uint8_t *)v.data() + off); }))
      return -1;
  }
  if (int64_t(b.size()) > cap) return -1;
  std::memcpy(out, b.data(), b.size());
  return int64_t(b.size());
}

// Reads the file against an engine fingerprint with the void det_void: 0 with the format version in *version and the
// counters in counts[*nwords]; 1 with the mismatch named in err; 2 with the reader's error.
int32_t ptb_ckpt_void_read(const uint8_t *in, int64_t n, int32_t det_void, uint32_t *version, uint64_t *counts,
                           int32_t *nwords, char *err, int64_t cap) {
  size_t pos = 0;
  Reader r([&](void *p, size_t k) { std::memcpy(p, in + pos, k); pos += k; return true; }, uint64_t(n));
  Header h;
  Fingerprint f;
  std::memcpy(version, in + 8, 4);
  auto put_err = [&](const std::string &s) { std::strncpy(err, s.c_str(), size_t(cap) - 1); err[cap - 1] = 0; };
  if (!r.begin(&h, &f)) { put_err(r.error()); return 2; }
  if (const char *field = fingerprint_mismatch(fp(det_void), f, false)) { put_err(field); return 1; }
  *nwords = int32_t(h.det_words);
  for (const auto &s : sections_of(h)) {
    std::vector<uint8_t> buf(s.second);
    if (!r.section(s.first, s.second, 64, [&](size_t) -> void * { return buf.data(); },
                   [&](size_t, uint64_t off, const void *p, size_t k) {
                     if (s.first == kDetCounts) std::memcpy((uint8_t *)counts + off, p, k);
                     return true;
                   })) {
      put_err(r.error());
      return 2;
    }
  }
  if (!r.at_end()) { put_err("data after the last section"); return 2; }
  return 0;
}
}
