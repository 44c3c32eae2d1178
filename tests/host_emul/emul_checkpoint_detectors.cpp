// TEST-ONLY host build of the checkpoint format with point detectors (checkpoint.cpp, format version 3): a file of a
// given fingerprint is written to memory and read back, so the version choice, the round trip and the named refusals
// can be checked without a GPU; never linked into libpumitally.so.
#include <cstring>
#include <string>
#include <vector>

#include "checkpoint.hpp"

using namespace ptb::ckpt;

namespace {
Fingerprint fp(int32_t ndet, const double *xyz, const double *r0, uint32_t crc, int32_t nmu) {
  Fingerprint f;
  f.nelems = 10;
  f.nverts = 8;
  f.batch_stats = 1;
  if (nmu > 0)
    for (int32_t j = 0; j <= nmu; ++j) f.mu_edges.push_back(double(j) / nmu);
  f.det_xyz.assign(xyz, xyz + 3 * ndet);
  f.det_r0.assign(r0, r0 + ndet);
  f.sigma_crc = crc;
  return f;
}
}  // namespace

extern "C" {
// A file with an open batch of 4 doubles, statistics of 4 and, with detectors, det_len doubles per detector section
// (the values i + 0.5 in every section).  Returns its size; out[cap].
int64_t ptb_ckpt_det_write(int32_t ndet, const double *xyz, const double *r0, uint32_t crc, int64_t det_len, int32_t nmu,
                           uint8_t *out, int64_t cap) {
  std::vector<uint8_t> b;
  Writer w([&](const void *p, size_t n) { b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n); return true; },
           [&](uint64_t off, const void *p, size_t n) { std::memcpy(b.data() + off, p, n); return true; });
  Header h;
  h.batches = 2;
  h.open = 1;
  h.open_len = 4;
  h.stats_len = 4;
  h.det_len = ndet > 0 ? uint64_t(det_len) : 0;
  if (!w.begin(h, fp(ndet, xyz, r0, crc, nmu))) return -1;
  for (const auto &s : sections_of(h)) {
    std::vector<double> v(s.second / 8);
    for (size_t i = 0; i < v.size(); ++i) v[i] = double(i) + 0.5;
    if (!w.section(s.first, s.second, 64, [&](size_t, uint64_t off, size_t) { return (const void *)((const uint8_t *)v.data() + off); }))
      return -1;
  }
  if (int64_t(b.size()) > cap) return -1;
  std::memcpy(out, b.data(), b.size());
  return int64_t(b.size());
}

// Reads the file against an engine fingerprint: 0 and det_len[0] = the declared length, the section ids in ids[]
// (count in *nids); 1 with the mismatch named in err; 2 with the reader's error.
int32_t ptb_ckpt_det_read(const uint8_t *in, int64_t n, int32_t ndet, const double *xyz, const double *r0, uint32_t crc,
                          int32_t nmu, int64_t *det_len, uint32_t *ids, int32_t *nids, char *err, int64_t cap) {
  size_t pos = 0;
  Reader r([&](void *p, size_t k) { std::memcpy(p, in + pos, k); pos += k; return true; }, uint64_t(n));
  Header h;
  Fingerprint f;
  auto put_err = [&](const std::string &s) { std::strncpy(err, s.c_str(), size_t(cap) - 1); err[cap - 1] = 0; };
  if (!r.begin(&h, &f)) {
    put_err(r.error());
    return 2;
  }
  if (const char *m = fingerprint_mismatch(fp(ndet, xyz, r0, crc, nmu), f, false)) {
    put_err(m);
    return 1;
  }
  *det_len = int64_t(h.det_len);
  *nids = 0;
  for (const auto &s : sections_of(h)) {
    std::vector<uint8_t> buf(s.second + 64);
    if (!r.section(s.first, s.second, 64, [&](size_t k) { return (void *)(buf.data() + 64 * k); },
                   [](size_t, uint64_t, const void *, size_t) { return true; })) {
      put_err(r.error());
      return 2;
    }
    ids[(*nids)++] = s.first;
  }
  return r.at_end() ? 0 : 2;
}
}
