// A C++ caller of the region currents (PumiTallyExtras.h) next to the reference class: the elements of a 3x3x3 box in
// three regions (and one element in none), face currents and batch statistics on, three batches.  The partials into
// the outside are checked against GetLeakage, every net current against the negated net of its reverse pair, and
// GetRegionCurrentResults' batch means against the mean of the values captured before every EndBatch.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 2048, B = 3, G = 3;
  pumitally::PumiTally tally("box:3,3,3", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  const int64_t E = pumitally_num_elements(e);
  std::vector<int32_t> region(E);
  for (int64_t i = 0; i < E; ++i) region[i] = int32_t(i % G);
  region[E - 1] = -1;
  if (pumitally::SetRegions(tally, region.data(), E, G) != 0) { printf("SetRegions failed\n"); return 1; }
  if (pumitally::SetRegionCurrents(tally, 1) == 0) { printf("accepted without face currents\n"); return 1; }
  if (pumitally::SetFaceCurrents(tally, 1) != 0 || pumitally::SetBatchStatistics(tally, 1) != 0 ||
      pumitally::SetRegionCurrents(tally, 1) != 0 || pumitally_get_region_currents(e) != 1) {
    printf("SetRegionCurrents failed\n");
    return 1;
  }
  const int64_t P = pumitally::GetRegionCurrentPairCount(tally);
  std::vector<int32_t> from(P), to(P);
  std::vector<double> area(P), part(P), net(P), x(B * P), mean(P);
  if (P < 1 || pumitally::GetRegionCurrentPairs(tally, from.data(), to.data(), P) != 0 ||
      pumitally::GetRegionCurrentAreas(tally, area.data(), P) != 0) {
    printf("pairs failed\n");
    return 1;
  }
  std::vector<double> init(3 * n), dest(3 * n), w(n);
  for (int i = 0; i < n; ++i) {
    init[3 * i] = 0.01 + 2.98 * ((i * 17) % n) / double(n);
    init[3 * i + 1] = 0.01 + 2.98 * ((i * 37) % n) / double(n);
    init[3 * i + 2] = 0.01 + 2.98 * ((i * 101) % n) / double(n);
    for (int a = 0; a < 3; ++a) dest[3 * i + a] = 4.0 - 1.5 * init[3 * i + a];
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  double bad = 0.0;
  for (int b = 0; b < B; ++b) {
    for (int i = 0; i < n; ++i) w[i] = 1.0 + 0.25 * b + 0.5 * ((i * 7 + b * 3) % 5);
    std::vector<int8_t> flying(n, 1);
    tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
    double leak = 0.0, out = 0.0, scale = 0.0;
    if (pumitally::GetRegionCurrentResults(tally, 0, 0, part.data(), P) != 0 ||
        pumitally::GetRegionCurrentResults(tally, 1, 0, net.data(), P) != 0 ||
        pumitally::GetLeakage(tally, 0, &leak, 1) != 0) {
      printf("GetRegionCurrentResults failed\n");
      return 1;
    }
    for (int64_t p = 0; p < P; ++p) {
      scale += std::fabs(part[p]);
      if (to[p] == -2) out += part[p];
      for (int64_t q = 0; q < P; ++q)
        if (from[q] == to[p] && to[q] == from[p] && net[q] != -net[p]) bad = 1.0;
      x[b * P + p] = net[p];
    }
    if (!(leak > 0.0)) { printf("no leakage\n"); return 1; }
    bad = std::max(bad, std::fabs(out - leak) / leak);
    if (pumitally::EndBatch(tally) != 0) { printf("EndBatch failed\n"); return 1; }
  }
  if (pumitally::GetRegionCurrentResults(tally, 1, 1, mean.data(), P) != 0) { printf("batch mean failed\n"); return 1; }
  for (int64_t p = 0; p < P; ++p) {
    double m = 0.0, a = 0.0;
    for (int b = 0; b < B; ++b) m += x[b * P + p] / B, a += std::fabs(x[b * P + p]);
    bad = std::max(bad, std::fabs(mean[p] - m) / std::max(a, 1e-300));
    if (!(area[p] > 0.0)) bad = 1.0;
  }
  if (!(bad < 1e-12)) {
    printf("worst relative difference %g\n", bad);
    return 1;
  }
  if (pumitally::SetFaceCurrents(tally, 0) != 0 || pumitally_get_region_currents(e) != 0) {
    printf("SetFaceCurrents(0) left region currents on\n");
    return 1;
  }
  printf("REGION_CURRENTS_OK pairs %lld\n", (long long)P);
  return 0;
}
