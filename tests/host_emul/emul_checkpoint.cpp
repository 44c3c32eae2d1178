// TEST-ONLY host build of the checkpoint format (checkpoint.cpp) and of welford_merge (batch_stats.cuh), the update
// merge_checkpoint's kernel runs.  Compiled by g++ so that both can be checked on a machine without a GPU; never linked
// into libpumitally.so.  The sections go through the same chunked callbacks the engine uses, here backed by memory.
#include <cstdint>
#include <cstring>
#include <vector>

#include "batch_stats.cuh"
#include "checkpoint.hpp"

namespace {

// The test fingerprint: fixed values except the element count, scores and time-bin edges.
ptb::ckpt::Fingerprint test_fingerprint(int64_t nelems, int32_t nscores, const double *edges, int32_t nedges) {
  ptb::ckpt::Fingerprint f;
  f.nelems = nelems;
  f.nverts = 2 * nelems + 3;
  f.mesh_hash = 0x1234;
  f.order_hash = 0x5678;
  f.nbins = 2;
  f.nscores = nscores;
  f.stride = nscores + 1;
  f.collision = 1;
  f.batch_stats = 1;
  f.nregions = 3;
  f.region_hash = 0x9abc;
  f.norm_mode = 2;
  f.norm_value = 37.0;
  f.edges.assign(edges, edges + nedges);
  return f;
}

void set_err(const std::string &s, char *err, int64_t cap) {
  if (cap <= 0) return;
  std::strncpy(err, s.c_str(), size_t(cap - 1));
  err[cap - 1] = '\0';
}

}  // namespace

extern "C" {

// (mean[i], m2[i]) <- welford_merge(mean_b[i], m2_b[i], na, nb) for i < n
void ptb_welford_merge(const double *mean_b, const double *m2_b, double na, double nb, double *mean, double *m2,
                       int64_t n) {
  for (int64_t i = 0; i < n; ++i) ptb::welford_merge(mean_b[i], m2_b[i], na, nb, mean[i], m2[i]);
}

// x[b * n + i] for b < B folded in order into (mean[i], m2[i]) of nb0 earlier batches
void ptb_welford_fold_all(const double *x, int64_t B, int64_t n, double nb0, double *mean, double *m2) {
  for (int64_t b = 0; b < B; ++b)
    for (int64_t i = 0; i < n; ++i) ptb::welford_fold(x[b * n + i], nb0 + double(b + 1), mean[i], m2[i]);
}

uint64_t ptb_hash64(const void *p, int64_t n, uint64_t seed) { return ptb::ckpt::hash64(p, size_t(n), seed); }

// Writes a checkpoint into out[cap] through chunk-sized callbacks.  hdr = {batches, open, open_len, stats_len,
// region_len}; scalars: 13 words (only read with open).  Returns the bytes written, -1 on failure.
int64_t ptb_ckpt_write(const int64_t *hdr, const double *open_tally, const uint64_t *scalars, const double *mean,
                       const double *m2, const double *rmean, const double *rm2, int64_t nelems, int32_t nscores,
                       const double *edges, int32_t nedges, int64_t chunk, uint8_t *out, int64_t cap) {
  namespace ck = ptb::ckpt;
  ck::Header h;
  h.batches = hdr[0];
  h.open = uint32_t(hdr[1]);
  h.open_len = uint64_t(hdr[2]);
  h.stats_len = uint64_t(hdr[3]);
  h.region_len = uint64_t(hdr[4]);
  std::vector<uint8_t> file;
  ck::Writer w([&](const void *p, size_t n) {
                 file.insert(file.end(), static_cast<const uint8_t *>(p), static_cast<const uint8_t *>(p) + n);
                 return true;
               },
               [&](uint64_t off, const void *p, size_t n) {
                 if (off + n > file.size()) return false;
                 std::memcpy(file.data() + off, p, n);
                 return true;
               });
  if (!w.begin(h, test_fingerprint(nelems, nscores, edges, nedges))) return -1;
  std::vector<uint8_t> bounce(static_cast<size_t>(chunk));  // each chunk is handed over from a buffer, as from a pinned one
  auto data = [&](uint32_t id, const void *src, uint64_t bytes) {
    return w.section(id, bytes, size_t(chunk), [&](size_t, uint64_t off, size_t len) -> const void * {
      std::memcpy(bounce.data(), static_cast<const uint8_t *>(src) + off, len);
      return bounce.data();
    });
  };
  for (const auto &s : ck::sections_of(h)) {
    const void *src = s.first == ck::kOpenTally     ? static_cast<const void *>(open_tally)
                      : s.first == ck::kMean        ? static_cast<const void *>(mean)
                      : s.first == ck::kM2          ? static_cast<const void *>(m2)
                      : s.first == ck::kRegionMean  ? static_cast<const void *>(rmean)
                      : s.first == ck::kRegionM2    ? static_cast<const void *>(rm2)
                                                    : nullptr;
    std::vector<uint8_t> packed;
    if (s.first == ck::kOpenScalars) {
      ck::OpenScalars o;
      std::memcpy(&o.initial_weight, &scalars[0], 8);
      o.initial_weight_pending = scalars[1];
      for (int i = 0; i < 3; ++i) o.coll_counts[i] = scalars[2 + i];
      o.segments = scalars[5];
      o.tracks = scalars[6];
      o.relocations = scalars[7];
      o.lost = scalars[8];
      o.fallbacks = scalars[9];
      o.moves = scalars[10];
      o.scored_moves = scalars[11];
      packed = ck::pack_open_scalars(o);
      src = packed.data();
    }
    if (!data(s.first, src, s.second)) return -1;
  }
  if (int64_t(file.size()) > cap) return -1;
  std::memcpy(out, file.data(), file.size());
  return int64_t(file.size());
}

// Reads the checkpoint in[n] against the test fingerprint of (nelems, nscores, edges).  Returns 0 on success, 2 when
// the header or fingerprint is refused (nothing read past them), 3 when a section is refused.  hdr_out as hdr above;
// the arrays receive the sections present (caller-sized); *max_request: the largest single read asked of the source.
int32_t ptb_ckpt_read(const uint8_t *in, int64_t n, int64_t nelems, int32_t nscores, const double *edges,
                      int32_t nedges, int64_t chunk, int64_t *hdr_out, double *open_tally, uint64_t *scalars,
                      double *mean, double *m2, double *rmean, double *rm2, int64_t *max_request, char *err,
                      int64_t errcap) {
  namespace ck = ptb::ckpt;
  uint64_t pos = 0;
  *max_request = 0;
  ck::Reader r([&](void *p, size_t k) {
                 *max_request = std::max<int64_t>(*max_request, int64_t(k));
                 if (pos + k > uint64_t(n)) return false;
                 std::memcpy(p, in + pos, k);
                 pos += k;
                 return true;
               },
               uint64_t(n));
  ck::Header h;
  ck::Fingerprint f;
  if (!r.begin(&h, &f)) {
    set_err(r.error(), err, errcap);
    return 2;
  }
  if (const char *field = ck::fingerprint_mismatch(test_fingerprint(nelems, nscores, edges, nedges), f, false)) {
    set_err(std::string("fingerprint: ") + field, err, errcap);
    return 2;
  }
  hdr_out[0] = h.batches;
  hdr_out[1] = h.open;
  hdr_out[2] = int64_t(h.open_len);
  hdr_out[3] = int64_t(h.stats_len);
  hdr_out[4] = int64_t(h.region_len);
  std::vector<uint8_t> bounce(static_cast<size_t>(chunk));
  for (const auto &s : ck::sections_of(h)) {
    std::vector<uint8_t> got(s.second);
    const bool ok = r.section(s.first, s.second, size_t(chunk), [&](size_t) -> void * { return bounce.data(); },
                              [&](size_t, uint64_t off, const void *p, size_t len) {
                                std::memcpy(got.data() + off, p, len);
                                return true;
                              });
    if (!ok) {
      set_err(r.error(), err, errcap);
      return 3;
    }
    void *dst = s.first == ck::kOpenTally     ? static_cast<void *>(open_tally)
                : s.first == ck::kMean        ? static_cast<void *>(mean)
                : s.first == ck::kM2          ? static_cast<void *>(m2)
                : s.first == ck::kRegionMean  ? static_cast<void *>(rmean)
                : s.first == ck::kRegionM2    ? static_cast<void *>(rm2)
                                              : nullptr;
    if (s.first == ck::kOpenScalars) {
      ck::OpenScalars o;
      if (!ck::unpack_open_scalars(got.data(), got.size(), &o)) {
        set_err("corrupt open-batch counters", err, errcap);
        return 3;
      }
      const uint64_t w[12] = {0, o.initial_weight_pending, o.coll_counts[0], o.coll_counts[1], o.coll_counts[2],
                              o.segments, o.tracks, o.relocations, o.lost, o.fallbacks, o.moves, o.scored_moves};
      std::memcpy(scalars, w, sizeof(w));
      std::memcpy(&scalars[0], &o.initial_weight, 8);
    } else {
      std::memcpy(dst, got.data(), got.size());
    }
  }
  if (!r.at_end()) {
    set_err("data after the last section", err, errcap);
    return 3;
  }
  return 0;
}
}
