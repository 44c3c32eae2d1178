// A C++ caller of the batch statistics (PumiTallyExtras.h) next to the reference class: four batches of the same flights
// with different weights, the per-source results captured before every EndBatch and their mean, standard error and
// relative error computed here, two-pass, against GetBatchResults and GetBatchMaxRelErr.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 2048, B = 4;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  if (pumitally::EndBatch(tally) == 0) { printf("EndBatch accepted with statistics off\n"); return 1; }
  if (pumitally::SetBatchStatistics(tally, 1) != 0) { printf("SetBatchStatistics failed\n"); return 1; }
  pumitally::SetSourceNormalization(tally, 3);
  const int64_t E = pumitally_num_elements(e);
  std::vector<double> init(3 * n), dest(3 * n), w(n);
  for (int i = 0; i < n; ++i) {
    init[3 * i] = 0.01 + 1.98 * ((i * 17) % n) / double(n);
    init[3 * i + 1] = 0.01 + 1.98 * ((i * 37) % n) / double(n);
    init[3 * i + 2] = 0.01 + 1.98 * ((i * 101) % n) / double(n);
    for (int a = 0; a < 3; ++a) dest[3 * i + a] = 2.0 - init[3 * i + a];
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  std::vector<std::vector<double>> x(B, std::vector<double>(E));
  std::vector<double> vol(E);
  for (int b = 0; b < B; ++b) {
    for (int i = 0; i < n; ++i) w[i] = 1.0 + 0.25 * b + 0.5 * ((i * 7 + b * 3) % 5);
    std::vector<int8_t> flying(n, 1);
    tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
    if (pumitally_get_normalized_flux(e, x[b].data(), vol.data(), E) != 0) { printf("get_normalized_flux failed\n"); return 1; }
    if (pumitally::EndBatch(tally) != 0) { printf("EndBatch failed\n"); return 1; }
  }
  if (pumitally_get_option(e, "batches") != B) { printf("batches %lld\n", (long long)pumitally_get_option(e, "batches")); return 1; }
  std::vector<double> got[3];
  for (int kind = 0; kind < 3; ++kind) {
    got[kind].resize(E);
    if (pumitally::GetBatchResults(tally, 0, kind, got[kind].data(), E) != 0) { printf("GetBatchResults failed\n"); return 1; }
  }
  double max_rel = 0.0, bad = 0.0;
  int64_t nonzero = 0;
  for (int64_t i = 0; i < E; ++i) {
    double m = 0.0, s2 = 0.0;
    for (int b = 0; b < B; ++b) m += x[b][i] / B;
    for (int b = 0; b < B; ++b) s2 += (x[b][i] - m) * (x[b][i] - m);
    const double se = std::sqrt(s2 / (B - 1) / B), rel = m != 0.0 ? se / std::fabs(m) : 0.0;
    if (m != 0.0) ++nonzero;
    max_rel = std::max(max_rel, rel);
    bad = std::max({bad, std::fabs(got[0][i] - m) / std::max(std::fabs(m), 1e-300),
                    std::fabs(got[1][i] - se) / std::max(se, 1e-300), std::fabs(got[2][i] - rel) / std::max(rel, 1e-300)});
  }
  double dev_max = 0.0;
  int64_t dev_nonzero = 0;
  if (pumitally::GetBatchMaxRelErr(tally, 0, 0, &dev_max, &dev_nonzero) != 0) { printf("GetBatchMaxRelErr failed\n"); return 1; }
  if (bad > 1e-12 || nonzero == 0 || dev_nonzero != nonzero || std::fabs(dev_max - max_rel) > 1e-12 * max_rel) {
    printf("worst relative difference %g, nonzero %lld / %lld, max rel err %g / %g\n", bad, (long long)nonzero,
           (long long)dev_nonzero, max_rel, dev_max);
    return 1;
  }
  printf("BATCH_STATS_OK\n");
  return 0;
}
