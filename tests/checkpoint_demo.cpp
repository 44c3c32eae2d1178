// A C++ caller of the checkpoints (PumiTallyExtras.h) next to the reference class: an engine on a 2x2x2 box with batch
// statistics folds three batches, tallies a fourth, and saves.  A second engine with the same configuration loads the
// file; its flux, statistics and counters must equal the first engine's bit for bit.  Then a run of three batches is
// merged into a third engine that has folded three batches of its own: B becomes 6.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

namespace {

const int n = 2048;

void setup(pumitally::PumiTally &t, std::vector<double> &init) {
  pumitally::SetBatchStatistics(t, 1);
  pumitally::SetSourceNormalization(t, 1);
  t.CopyInitialPosition(init.data(), 3 * n);
}

int batch(pumitally::PumiTally &t, std::vector<double> &init, std::vector<double> &dest, int b, bool end) {
  std::vector<double> w(n);
  for (int i = 0; i < n; ++i) w[i] = 1.0 + 0.25 * b + 0.5 * ((i * 7 + b * 3) % 5);
  std::vector<int8_t> flying(n, 1);
  t.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
  return end ? pumitally::EndBatch(t) : 0;
}

}  // namespace

int main(int argc, char **argv) {
  std::vector<double> init(3 * n), dest(3 * n);
  for (int i = 0; i < n; ++i) {
    init[3 * i] = 0.01 + 1.98 * ((i * 17) % n) / double(n);
    init[3 * i + 1] = 0.01 + 1.98 * ((i * 37) % n) / double(n);
    init[3 * i + 2] = 0.01 + 1.98 * ((i * 101) % n) / double(n);
    for (int a = 0; a < 3; ++a) dest[3 * i + a] = 2.0 - init[3 * i + a];
  }
  pumitally::PumiTally a("box:2,2,2", n, argc, argv), b("box:2,2,2", n, argc, argv), c("box:2,2,2", n, argc, argv);
  setup(a, init);
  setup(b, init);
  setup(c, init);
  pumitally_engine *ea = pumitally::engine_of(a), *eb = pumitally::engine_of(b), *ec = pumitally::engine_of(c);
  const int64_t E = pumitally_num_elements(ea);
  for (int k = 0; k < 3; ++k)
    if (batch(a, init, dest, k, true) != 0 || batch(c, init, dest, 10 + k, true) != 0) {
      printf("EndBatch failed\n");
      return 1;
    }
  if (pumitally::SaveCheckpoint(a, "end.ckpt") != 0) { printf("SaveCheckpoint at a batch end failed\n"); return 1; }
  batch(a, init, dest, 3, false);
  if (pumitally::SaveCheckpoint(a, "mid.ckpt") != 0) { printf("SaveCheckpoint mid-batch failed\n"); return 1; }
  if (pumitally::LoadCheckpoint(b, "mid.ckpt") != 0) { printf("LoadCheckpoint failed\n"); return 1; }
  std::vector<double> fa(E), fb(E), ma(E), mb(E), sa(E), sb(E);
  if (pumitally_get_flux(ea, fa.data(), E) || pumitally_get_flux(eb, fb.data(), E) ||
      pumitally::GetBatchResults(a, 0, 0, ma.data(), E) || pumitally::GetBatchResults(b, 0, 0, mb.data(), E) ||
      pumitally::GetBatchResults(a, 0, 1, sa.data(), E) || pumitally::GetBatchResults(b, 0, 1, sb.data(), E)) {
    printf("reading the results failed\n");
    return 1;
  }
  if (std::memcmp(fa.data(), fb.data(), E * sizeof(double)) || std::memcmp(ma.data(), mb.data(), E * sizeof(double)) ||
      std::memcmp(sa.data(), sb.data(), E * sizeof(double))) {
    printf("the loaded engine differs\n");
    return 1;
  }
  pumitally_stats ta, tb;
  if (pumitally_get_stats(ea, &ta) || pumitally_get_stats(eb, &tb) || pumitally_get_option(eb, "batches") != 3 ||
      ta.segments != tb.segments || ta.tracks != tb.tracks || ta.moves != tb.moves) {
    printf("batches %lld, segments %llu vs %llu\n", (long long)pumitally_get_option(eb, "batches"),
           (unsigned long long)tb.segments, (unsigned long long)ta.segments);
    return 1;
  }
  if (pumitally::MergeCheckpoint(c, "mid.ckpt") == 0) { printf("merged an open batch\n"); return 1; }
  if (pumitally::MergeCheckpoint(c, "end.ckpt") != 0 || pumitally_get_option(ec, "batches") != 6) {
    printf("MergeCheckpoint failed\n");
    return 1;
  }
  if (pumitally::LoadCheckpoint(b, "missing.ckpt") == 0) { printf("loaded a missing file\n"); return 1; }
  printf("CHECKPOINT_OK\n");
  return 0;
}
