// Checkpoint file format (checkpoint.hpp).
#include "checkpoint.hpp"

#include <zlib.h>

#include <algorithm>
#include <cstring>

namespace ptb {
namespace ckpt {
namespace {

constexpr char kMagic[8] = {'P', 'T', 'B', 'C', 'K', 'P', 'T', '\0'};
constexpr uint32_t kEndianMarker = 0x01020304u;
constexpr uint32_t kMaxEdges = 1025;          // kMaxTimeBins + 1 (walk_core.cuh)
constexpr uint32_t kMaxMuEdges = 65;          // kMaxCosineBins + 1 (walk_core.cuh)
constexpr uint32_t kMaxDetectors = 256;       // kMaxDetectors (walk_core.cuh)
constexpr uint64_t kMaxLen = uint64_t(1) << 56;  // doubles: beyond any device memory, and no overflow below
constexpr size_t kSectionHead = 16;           // id (u32), byte length (u64), CRC-32 (u32)

void put_le(std::vector<uint8_t> &b, uint64_t v, int n) {
  for (int i = 0; i < n; ++i) b.push_back(uint8_t(v >> (8 * i)));
}
uint64_t get_le(const uint8_t *p, int n) {
  uint64_t v = 0;
  for (int i = 0; i < n; ++i) v |= uint64_t(p[i]) << (8 * i);
  return v;
}
uint64_t bits_of(double d) {
  uint64_t u;
  std::memcpy(&u, &d, 8);
  return u;
}
double double_of(uint64_t u) {
  double d;
  std::memcpy(&d, &u, 8);
  return d;
}

// header and fingerprint, without the prefix (magic, version, marker) and the CRC
constexpr size_t kHeaderBytes = 8 + 4 + 4 + 8 + 8 + 8;
constexpr size_t kFingerprintFixed = 8 + 8 + 8 + 8 + 8 * 4 + 8 + 8 + 4 + 4 + 8 + 4;  // up to the edge count

void put_header(std::vector<uint8_t> &b, const Header &h, const Fingerprint &f) {
  put_le(b, uint64_t(h.batches), 8);
  put_le(b, h.open, 4);
  put_le(b, 0, 4);
  put_le(b, h.open_len, 8);
  put_le(b, h.stats_len, 8);
  put_le(b, h.region_len, 8);
  put_le(b, uint64_t(f.nelems), 8);
  put_le(b, uint64_t(f.nverts), 8);
  put_le(b, f.mesh_hash, 8);
  put_le(b, f.order_hash, 8);
  for (int32_t v : {f.nbins, f.nscores, f.stride, f.moments, f.collision, f.batch_stats, f.nregions, f.norm_mode})
    put_le(b, uint32_t(v), 4);
  put_le(b, f.region_hash, 8);
  put_le(b, bits_of(f.norm_value), 8);
  put_le(b, uint32_t(f.rank), 4);
  put_le(b, uint32_t(f.nranks), 4);
  put_le(b, f.share, 8);
  put_le(b, uint32_t(f.edges.size()), 4);
  for (double e : f.edges) put_le(b, bits_of(e), 8);
  if (!f.mu_edges.empty() || !f.det_r0.empty()) {  // versions 2 and 3
    put_le(b, uint32_t(f.mu_edges.size()), 4);
    for (double e : f.mu_edges) put_le(b, bits_of(e), 8);
  }
  if (!f.det_r0.empty()) {  // version 3 only
    put_le(b, uint32_t(f.det_r0.size()), 4);
    for (double e : f.det_xyz) put_le(b, bits_of(e), 8);
    for (double e : f.det_r0) put_le(b, bits_of(e), 8);
    put_le(b, f.sigma_crc, 4);
    put_le(b, h.det_len, 8);
  }
}

void get_header(const uint8_t *p, Header *h, Fingerprint *f, bool cosines, bool detectors) {
  h->batches = int64_t(get_le(p, 8));
  h->open = uint32_t(get_le(p + 8, 4));
  h->open_len = get_le(p + 16, 8);
  h->stats_len = get_le(p + 24, 8);
  h->region_len = get_le(p + 32, 8);
  p += kHeaderBytes;
  f->nelems = int64_t(get_le(p, 8));
  f->nverts = int64_t(get_le(p + 8, 8));
  f->mesh_hash = get_le(p + 16, 8);
  f->order_hash = get_le(p + 24, 8);
  p += 32;
  int32_t *ints[] = {&f->nbins, &f->nscores, &f->stride, &f->moments, &f->collision, &f->batch_stats, &f->nregions,
                     &f->norm_mode};
  for (int32_t *v : ints) {
    *v = int32_t(uint32_t(get_le(p, 4)));
    p += 4;
  }
  f->region_hash = get_le(p, 8);
  f->norm_value = double_of(get_le(p + 8, 8));
  f->rank = int32_t(uint32_t(get_le(p + 16, 4)));
  f->nranks = int32_t(uint32_t(get_le(p + 20, 4)));
  f->share = get_le(p + 24, 8);
  const uint32_t ne = uint32_t(get_le(p + 32, 4));
  p += 36;
  f->edges.resize(ne);
  for (uint32_t j = 0; j < ne; ++j) f->edges[j] = double_of(get_le(p + 8 * j, 8));
  f->mu_edges.clear();
  f->det_xyz.clear();
  f->det_r0.clear();
  f->sigma_crc = 0;
  h->det_len = 0;
  if (cosines || detectors) {
    p += 8 * size_t(ne);
    const uint32_t nm = uint32_t(get_le(p, 4));
    f->mu_edges.resize(nm);
    for (uint32_t j = 0; j < nm; ++j) f->mu_edges[j] = double_of(get_le(p + 4 + 8 * j, 8));
    p += 4 + 8 * size_t(nm);
  }
  if (detectors) {
    const uint32_t nd = uint32_t(get_le(p, 4));
    p += 4;
    f->det_xyz.resize(3 * size_t(nd));
    f->det_r0.resize(nd);
    for (size_t j = 0; j < 3 * size_t(nd); ++j) f->det_xyz[j] = double_of(get_le(p + 8 * j, 8));
    p += 24 * size_t(nd);
    for (size_t j = 0; j < nd; ++j) f->det_r0[j] = double_of(get_le(p + 8 * j, 8));
    p += 8 * size_t(nd);
    f->sigma_crc = uint32_t(get_le(p, 4));
    h->det_len = get_le(p + 4, 8);
  }
}

uint64_t rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

}  // namespace

uint64_t hash64(const void *data, size_t bytes, uint64_t seed) {
  const uint8_t *p = static_cast<const uint8_t *>(data);
  uint64_t h = seed ^ (uint64_t(bytes) * 0x9e3779b97f4a7c15ull);
  auto step = [&](uint64_t w) {
    w *= 0x87c37b91114253d5ull;
    w = rotl(w, 31) * 0x4cf5ad432745937full;
    h = rotl(h ^ w, 27) * 5 + 0x52dce729u;
  };
  size_t i = 0;
  for (; i + 8 <= bytes; i += 8) step(get_le(p + i, 8));
  if (i < bytes) step(get_le(p + i, int(bytes - i)) ^ (uint64_t(bytes - i) << 59));
  h ^= h >> 33;  // splitmix64 / murmur3 finaliser
  h *= 0xff51afd7ed558ccdull;
  h ^= h >> 33;
  h *= 0xc4ceb9fe1a85ec53ull;
  return h ^ (h >> 33);
}

uint32_t crc32(const void *data, size_t bytes, uint32_t crc) {
  const Bytef *p = static_cast<const Bytef *>(data);
  uLong c = crc;
  while (bytes > 0) {  // zlib takes uInt lengths
    const size_t n = bytes < (size_t(1) << 30) ? bytes : (size_t(1) << 30);
    c = ::crc32(c, p, uInt(n));
    p += n;
    bytes -= n;
  }
  return uint32_t(c);
}

const char *fingerprint_mismatch(const Fingerprint &a, const Fingerprint &b, bool ignore_norm_value) {
  if (a.nelems != b.nelems) return "number of elements";
  if (a.nverts != b.nverts) return "number of vertices";
  if (a.mesh_hash != b.mesh_hash) return "mesh (hash of coordinates and t2v)";
  if (a.order_hash != b.order_hash) return "internal element order (hash of orig_of_internal)";
  if (a.nbins != b.nbins) return "score bins";
  if (a.nscores != b.nscores) return "scores";
  if (a.stride != b.stride) return "record stride";
  if (a.edges.size() != b.edges.size()) return "number of time bins";
  for (size_t j = 0; j < a.edges.size(); ++j)
    if (bits_of(a.edges[j]) != bits_of(b.edges[j])) return "time-bin edges";
  if (a.mu_edges.size() != b.mu_edges.size()) return "number of current cosine bins (set_current_cosine_bins)";
  for (size_t j = 0; j < a.mu_edges.size(); ++j)
    if (bits_of(a.mu_edges[j]) != bits_of(b.mu_edges[j])) return "current cosine-bin edges (set_current_cosine_bins)";
  if (a.moments != b.moments) return "moment order";
  if (a.collision != b.collision) return "collision estimator";
  if (a.batch_stats != b.batch_stats) return "batch statistics on/off";
  if (a.nregions != b.nregions) return "number of regions";
  if (a.region_hash != b.region_hash) return "region map";
  if (a.norm_mode != b.norm_mode) return "source-normalisation mode";
  if (a.norm_mode == 2 && !ignore_norm_value && bits_of(a.norm_value) != bits_of(b.norm_value))
    return "source-normalisation value";
  if (a.rank != b.rank) return "rank";
  if (a.nranks != b.nranks) return "number of ranks";
  if (a.share != b.share) return "rank share";
  if (a.det_r0.size() != b.det_r0.size()) return "number of point detectors (set_point_detectors)";
  for (size_t j = 0; j < a.det_xyz.size(); ++j)
    if (bits_of(a.det_xyz[j]) != bits_of(b.det_xyz[j])) return "point-detector positions (set_point_detectors)";
  for (size_t j = 0; j < a.det_r0.size(); ++j)
    if (bits_of(a.det_r0[j]) != bits_of(b.det_r0[j])) return "point-detector exclusion radii (set_point_detectors)";
  if (a.sigma_crc != b.sigma_crc) return "detector cross-section table (set_detector_cross_sections)";
  if (a.det_void != b.det_void) return "detector void (set_detector_void)";
  return nullptr;
}

std::vector<uint8_t> pack_open_scalars(const OpenScalars &s) {
  std::vector<uint8_t> b;
  const uint64_t w[kOpenScalarWords] = {bits_of(s.initial_weight), s.initial_weight_pending, s.coll_counts[0],
                                        s.coll_counts[1], s.coll_counts[2], s.segments, s.tracks, s.relocations,
                                        s.lost, s.fallbacks, s.moves, s.scored_moves, 0};
  for (uint64_t v : w) put_le(b, v, 8);
  return b;
}

bool unpack_open_scalars(const void *bytes, size_t n, OpenScalars *s) {
  if (n != 8 * kOpenScalarWords) return false;
  const uint8_t *p = static_cast<const uint8_t *>(bytes);
  uint64_t w[kOpenScalarWords];
  for (size_t i = 0; i < kOpenScalarWords; ++i) w[i] = get_le(p + 8 * i, 8);
  if (w[1] > 1 || w[12] != 0) return false;
  s->initial_weight = double_of(w[0]);
  s->initial_weight_pending = w[1];
  for (int i = 0; i < 3; ++i) s->coll_counts[i] = w[2 + i];
  s->segments = w[5];
  s->tracks = w[6];
  s->relocations = w[7];
  s->lost = w[8];
  s->fallbacks = w[9];
  s->moves = w[10];
  s->scored_moves = w[11];
  return true;
}

std::vector<std::pair<uint32_t, uint64_t>> sections_of(const Header &h) {
  std::vector<std::pair<uint32_t, uint64_t>> s;
  if (h.open) {
    s.emplace_back(kOpenTally, 8 * h.open_len);
    s.emplace_back(kOpenScalars, 8 * kOpenScalarWords);
  }
  if (h.stats_len) {
    s.emplace_back(kMean, 8 * h.stats_len);
    s.emplace_back(kM2, 8 * h.stats_len);
  }
  if (h.region_len) {
    s.emplace_back(kRegionMean, 8 * h.region_len);
    s.emplace_back(kRegionM2, 8 * h.region_len);
  }
  if (h.det_len && h.open) {
    s.emplace_back(kDetOpen, 8 * h.det_len);
    s.emplace_back(kDetCounts, 8 * uint64_t(h.det_words));
  }
  if (h.det_len && h.stats_len) {
    s.emplace_back(kDetMean, 8 * h.det_len);
    s.emplace_back(kDetM2, 8 * h.det_len);
  }
  return s;
}

// ---------------------------------------------------------------- Writer

bool Writer::put(const void *p, size_t n) {
  if (!write_(p, n)) {
    err_ = "write failed";
    return false;
  }
  pos_ += n;
  return true;
}

bool Writer::begin(const Header &h, const Fingerprint &f) {
  std::vector<uint8_t> b(kMagic, kMagic + 8);
  put_le(b, !f.det_r0.empty() ? (f.det_void ? kVersionDetectorVoid : kVersionDetectors)
            : f.mu_edges.empty() ? kVersion
                                 : kVersionCosines,
         4);
  put_le(b, kEndianMarker, 4);
  put_header(b, h, f);
  put_le(b, crc32(b.data(), b.size()), 4);
  return put(b.data(), b.size());
}

bool Writer::section(uint32_t id, uint64_t bytes, size_t chunk_bytes,
                     const std::function<const void *(size_t, uint64_t, size_t)> &chunk) {
  std::vector<uint8_t> head;
  put_le(head, id, 4);
  put_le(head, bytes, 8);
  put_le(head, 0, 4);  // the CRC, patched below
  const uint64_t crc_at = pos_ + 12;
  if (!put(head.data(), head.size())) return false;
  uint32_t crc = 0;
  size_t k = 0;
  for (uint64_t off = 0; off < bytes; off += chunk_bytes, ++k) {
    const size_t len = size_t(std::min<uint64_t>(chunk_bytes, bytes - off));
    const void *p = chunk(k, off, len);
    if (!p) {
      err_ = "the section's data could not be read";
      return false;
    }
    crc = crc32(p, len, crc);
    if (!put(p, len)) return false;
  }
  uint8_t c[4];
  for (int i = 0; i < 4; ++i) c[i] = uint8_t(crc >> (8 * i));
  if (!patch_(crc_at, c, 4)) {
    err_ = "write failed";
    return false;
  }
  return true;
}

// ---------------------------------------------------------------- Reader

bool Reader::get(void *p, size_t n) {
  if (n > size_ - pos_ || !read_(p, n)) {
    err_ = "the file is truncated";
    return false;
  }
  pos_ += n;
  return true;
}

bool Reader::begin(Header *h, Fingerprint *f) {
  std::vector<uint8_t> b(16 + kHeaderBytes + kFingerprintFixed);
  if (!get(b.data(), b.size())) return false;
  if (std::memcmp(b.data(), kMagic, 8) != 0) {
    err_ = "not a checkpoint file (wrong magic)";
    return false;
  }
  const uint64_t version = get_le(b.data() + 8, 4);
  if (version != kVersion && version != kVersionCosines && version != kVersionDetectors &&
      version != kVersionDetectorVoid) {
    err_ = "unsupported format version " + std::to_string(version);
    return false;
  }
  const bool cosines = version == kVersionCosines, det_void = version == kVersionDetectorVoid,
             detectors = version == kVersionDetectors || det_void;
  if (get_le(b.data() + 12, 4) != kEndianMarker) {
    err_ = "wrong endianness marker";
    return false;
  }
  const uint32_t ne = uint32_t(get_le(b.data() + b.size() - 4, 4));
  if (ne > kMaxEdges) {
    err_ = "corrupt header (edge count)";
    return false;
  }
  const size_t fixed = b.size();
  b.resize(fixed + 8 * size_t(ne) + 4);
  if (!get(b.data() + fixed, b.size() - fixed)) return false;
  if (cosines) {  // the last 4 bytes read are the cosine-edge count, not the CRC
    const uint32_t nm = uint32_t(get_le(b.data() + b.size() - 4, 4));
    if (nm < 2 || nm > kMaxMuEdges) {
      err_ = "corrupt version 2 header (cosine-bin edge count)";
      return false;
    }
    const size_t at = b.size();
    b.resize(at + 8 * size_t(nm) + 4);
    if (!get(b.data() + at, b.size() - at)) return false;
  }
  if (detectors) {  // the last 4 bytes read are the cosine-edge count (0 or 2..65), then come the detectors
    const uint32_t nm = uint32_t(get_le(b.data() + b.size() - 4, 4));
    if (nm == 1 || nm > kMaxMuEdges) {
      err_ = "corrupt version 3 header (cosine-bin edge count)";
      return false;
    }
    size_t at = b.size();
    b.resize(at + 8 * size_t(nm) + 4);
    if (!get(b.data() + at, b.size() - at)) return false;
    const uint32_t nd = uint32_t(get_le(b.data() + b.size() - 4, 4));
    if (nd < 1 || nd > kMaxDetectors) {
      err_ = "corrupt version 3 header (detector count)";
      return false;
    }
    at = b.size();
    b.resize(at + 32 * size_t(nd) + 4 + 8 + 4);
    if (!get(b.data() + at, b.size() - at)) return false;
  }
  if (crc32(b.data(), b.size() - 4) != uint32_t(get_le(b.data() + b.size() - 4, 4))) {
    err_ = cosines ? "corrupt version 2 header or fingerprint (CRC mismatch)"
           : det_void  ? "corrupt version 4 header or fingerprint (CRC mismatch)"
           : detectors ? "corrupt version 3 header or fingerprint (CRC mismatch)"
                       : "corrupt header or fingerprint (CRC mismatch)";
    return false;
  }
  get_header(b.data() + 16, h, f, cosines, detectors);
  f->det_void = det_void ? 1 : 0;
  h->det_words = uint32_t(det_void ? kDetCountWordsVoid : kDetCountWords);
  if (h->open > 1 || (!h->open && h->open_len) || h->batches < 0 || h->open_len > kMaxLen ||
      h->stats_len > kMaxLen || h->region_len > kMaxLen || h->det_len > kMaxLen || (detectors && !h->det_len)) {
    err_ = "corrupt header (declared lengths)";
    return false;
  }
  uint64_t total = b.size();
  for (const auto &s : sections_of(*h)) total += kSectionHead + s.second;
  if (total != size_) {
    err_ = "the declared lengths (" + std::to_string(total) + " bytes) do not match the file size (" +
           std::to_string(size_) + " bytes)";
    return false;
  }
  return true;
}

bool Reader::section(uint32_t id, uint64_t bytes, size_t chunk_bytes, const std::function<void *(size_t)> &buffer,
                     const std::function<bool(size_t, uint64_t, const void *, size_t)> &consume) {
  uint8_t head[kSectionHead];
  if (!get(head, sizeof(head))) return false;
  if (get_le(head, 4) != id || get_le(head + 4, 8) != bytes) {
    err_ = "section " + std::to_string(id) + ": unexpected id or length";
    return false;
  }
  uint32_t crc = 0;
  size_t k = 0;
  for (uint64_t off = 0; off < bytes; off += chunk_bytes, ++k) {
    const size_t len = size_t(std::min<uint64_t>(chunk_bytes, bytes - off));
    void *p = buffer(k);
    if (!p || !get(p, len)) {
      if (err_.empty()) err_ = "no buffer for section " + std::to_string(id);
      return false;
    }
    crc = crc32(p, len, crc);
    if (!consume(k, off, p, len)) {
      err_ = "section " + std::to_string(id) + " could not be stored";
      return false;
    }
  }
  if (crc != uint32_t(get_le(head + 12, 4))) {
    err_ = "section " + std::to_string(id) + " is corrupt (CRC mismatch)";
    return false;
  }
  return true;
}

}  // namespace ckpt
}  // namespace ptb
