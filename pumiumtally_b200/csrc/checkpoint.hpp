// Checkpoint file format of the engine's tally state (engine.cu, save_checkpoint / load_checkpoint /
// merge_checkpoint).  Host only; this module owns the format and nothing else: the engine hands it a fingerprint, a
// header and the sections' bytes through callbacks, and never sees how they are laid out in the file.
//
// A file is little-endian throughout:
//   magic "PTBCKPT\0" (8 B), format version (u32), endianness marker 0x01020304 (u32),
//   the fixed header (Header: batches, open flag, declared lengths),
//   the fingerprint (Fingerprint: every value the layout and meaning of the arrays depend on; the time-bin edges last,
//     preceded by their count; in a version-2 file, the current cosine-bin edges after them, preceded by their count),
//   the CRC-32 of everything before it (u32),
//   then one section per present array, in the order of SectionId: id (u32), byte length (u64), CRC-32 of the payload
//   (u32), payload.
// Nothing may follow the last section.  The file holds no timestamp or path, so the same state always gives the same
// bytes.  Sections are written and read in chunks through callbacks, so the engine can feed them from pinned buffers
// (overlapping the device copies with the CRC and the file I/O) and the tests can feed them from memory.
#pragma once
#include <cstddef>
#include <cstdint>
#include <functional>
#include <string>
#include <vector>

namespace ptb {
namespace ckpt {

// Version 1: no cosine bins.  A file whose fingerprint holds cosine-bin edges is written as version 2, which a build
// that does not know them refuses instead of misreading; every other file keeps version 1's bytes.
constexpr uint32_t kVersion = 1;
constexpr uint32_t kVersionCosines = 2;
// Version 3: point detectors.  After the time-bin edges come the cosine-bin edges (count, possibly 0), the detectors
// (count D, positions [3D], exclusion radii [D]), the CRC-32 of the cross-section table and det_len (u64).  Only a file
// whose fingerprint holds detectors is written as version 3.
constexpr uint32_t kVersionDetectors = 3;
// Version 4: point detectors with the detector void (pumitally_set_detector_void) on.  The header is version 3's; the
// version itself records the mode, and kDetCounts holds kDetCountWordsVoid counters (the hull entries last).  Every
// file saved with the mode off keeps its version and bytes.
constexpr uint32_t kVersionDetectorVoid = 4;

// 64-bit hash of a byte string (not cryptographic: it tells configurations apart, it does not authenticate them).
// Chainable: hash64(b, nb, hash64(a, na)) hashes a then b.
uint64_t hash64(const void *data, size_t bytes, uint64_t seed = 0);

// CRC-32 (zlib's polynomial), chainable as zlib's crc32.
uint32_t crc32(const void *data, size_t bytes, uint32_t crc = 0);

// Everything the layout and meaning of the saved arrays depend on.  Load and merge refuse any difference.
struct Fingerprint {
  int64_t nelems = 0, nverts = 0;
  uint64_t mesh_hash = 0;   // coordinates and t2v (caller's numbering)
  uint64_t order_hash = 0;  // orig_of_internal: the internal element order the arrays are stored in
  int32_t nbins = 1, nscores = 1, stride = 1;
  int32_t moments = 0, collision = 0, batch_stats = 0;
  int32_t nregions = 0;
  uint64_t region_hash = 0;  // the region map in the caller's numbering
  int32_t norm_mode = 0;
  double norm_value = 0.0;  // compared for mode 2 only
  int32_t rank = 0, nranks = 1;
  uint64_t share = 0;
  std::vector<double> edges;  // time-bin edges (empty: no time filter), compared bit for bit
  std::vector<double> mu_edges;  // cosine-bin edges of the face currents (empty: none), compared bit for bit
  std::vector<double> det_xyz, det_r0;  // point detectors (empty: none), compared bit for bit
  uint32_t sigma_crc = 0;               // CRC-32 of the detector cross-section table as uploaded (0: no table)
  uint32_t det_void = 0;                // the detector void is on (with detectors only: version 4)
};

// The name of the first field in which `file` differs from `engine`, nullptr when they agree.  ignore_norm_value:
// the mode-2 value is not compared (merge: the folded values are already per source).
const char *fingerprint_mismatch(const Fingerprint &engine, const Fingerprint &file, bool ignore_norm_value);

struct Header {
  int64_t batches = 0;      // folded batches (0 without statistics)
  uint32_t open = 0;        // 1: the file holds an open batch (sections kOpenTally and kOpenScalars)
  uint64_t open_len = 0;    // doubles of the open tally (0 without one)
  uint64_t stats_len = 0;   // doubles of each of kMean and kM2 (0 without statistics)
  uint64_t region_len = 0;  // doubles of each of kRegionMean and kRegionM2 (0 without region statistics)
  uint64_t det_len = 0;     // doubles of the detector tally (versions 3 and 4; 0 without detectors)
  uint32_t det_words = 7;   // 64-bit words of kDetCounts: kDetCountWords, kDetCountWordsVoid in version 4 (not stored)
};

enum SectionId : uint32_t {
  kOpenTally = 1,     // the raw local tally [open_len] doubles
  kOpenScalars = 2,   // kOpenScalarWords 64-bit words (OpenScalars)
  kMean = 3,          // running means [stats_len]
  kM2 = 4,            // sums of squared deviations [stats_len]
  kRegionMean = 5,    // [region_len]
  kRegionM2 = 6,      // [region_len]
  kDetOpen = 7,       // the open detector tally [det_len] (with kOpenTally)
  kDetCounts = 8,     // kDetCountWords 64-bit detector counters (with kOpenTally)
  kDetMean = 9,       // [det_len] (with kMean)
  kDetM2 = 10,        // [det_len] (with kMean)
};
constexpr size_t kDetCountWords = 7;
constexpr size_t kDetCountWordsVoid = 8;

// The small state of the open batch, as 64-bit words in this order.
struct OpenScalars {
  double initial_weight = 0.0;
  uint64_t initial_weight_pending = 1;
  uint64_t coll_counts[3] = {0, 0, 0};
  uint64_t segments = 0, tracks = 0, relocations = 0, lost = 0, fallbacks = 0;
  uint64_t moves = 0, scored_moves = 0;
};
constexpr size_t kOpenScalarWords = 13;
std::vector<uint8_t> pack_open_scalars(const OpenScalars &s);
bool unpack_open_scalars(const void *bytes, size_t n, OpenScalars *s);

// The sections a header declares, in file order: (id, byte length).
std::vector<std::pair<uint32_t, uint64_t>> sections_of(const Header &h);

// Byte sink: write all n bytes, false on failure.
using WriteFn = std::function<bool(const void *data, size_t n)>;
// Byte source: read exactly n bytes, false on failure or end of data.
using ReadFn = std::function<bool(void *data, size_t n)>;

class Writer {
 public:
  // The payload of a section is written and checksummed before its CRC is known: the writer buffers nothing and
  // patches the CRC afterwards through `patch` (write n bytes at absolute offset off, then continue at the end).
  Writer(WriteFn write, std::function<bool(uint64_t off, const void *data, size_t n)> patch)
      : write_(std::move(write)), patch_(std::move(patch)) {}
  bool begin(const Header &h, const Fingerprint &f);
  // chunk(k, off, len) returns the k-th chunk of the payload, bytes [off, off + len) of it (chunk_bytes each but the
  // last); the pointer stays valid until the next call.  nullptr aborts the write.
  bool section(uint32_t id, uint64_t bytes, size_t chunk_bytes,
               const std::function<const void *(size_t k, uint64_t off, size_t len)> &chunk);
  const std::string &error() const { return err_; }

 private:
  bool put(const void *p, size_t n);
  WriteFn write_;
  std::function<bool(uint64_t, const void *, size_t)> patch_;
  uint64_t pos_ = 0;
  std::string err_;
};

class Reader {
 public:
  // file_bytes: the size of the whole file; the header's declared lengths must add up to it.
  Reader(ReadFn read, uint64_t file_bytes) : read_(std::move(read)), size_(file_bytes) {}
  // Reads and checks magic, version, endianness, header, fingerprint and their CRC, and that the declared sections
  // fill the file exactly.  Allocates nothing that depends on the declared lengths.
  bool begin(Header *h, Fingerprint *f);
  // The next section must be (id, bytes).  buffer(k) returns where chunk k (chunk_bytes each but the last) is to be
  // read; consume(k, off, data, len) receives it after its bytes arrived.  The CRC is checked after the last chunk;
  // a mismatch returns false after everything was consumed.
  bool section(uint32_t id, uint64_t bytes, size_t chunk_bytes, const std::function<void *(size_t k)> &buffer,
               const std::function<bool(size_t k, uint64_t off, const void *data, size_t len)> &consume);
  // true when every byte of the file has been read
  bool at_end() const { return pos_ == size_; }
  const std::string &error() const { return err_; }

 private:
  bool get(void *p, size_t n);
  ReadFn read_;
  uint64_t size_ = 0, pos_ = 0;
  std::string err_;
};

}  // namespace ckpt
}  // namespace ptb
