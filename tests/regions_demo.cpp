// A C++ caller of the region tallies (PumiTallyExtras.h) next to the reference class: the elements of a 2x2x2 box in
// three regions (and one element in none), four batches with batch statistics on.  The region sums are checked against
// sums of pumitally_get_flux, the volumes against the element volumes, and GetRegionBatchResults against a two-pass
// mean and standard error of the region sums captured before every EndBatch.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 2048, B = 4, G = 3;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  const int64_t E = pumitally_num_elements(e);
  std::vector<int32_t> region(E);
  for (int64_t i = 0; i < E; ++i) region[i] = int32_t(i % G);
  region[E - 1] = -1;
  if (pumitally::SetRegions(tally, region.data(), E, 0) == 0) { printf("SetRegions accepted nregions 0\n"); return 1; }
  if (pumitally::SetBatchStatistics(tally, 1) != 0 || pumitally::SetRegions(tally, region.data(), E, G) != 0) {
    printf("SetRegions failed\n");
    return 1;
  }
  if (pumitally_get_regions(e) != G) { printf("regions %d\n", pumitally_get_regions(e)); return 1; }
  std::vector<double> init(3 * n), dest(3 * n), w(n);
  for (int i = 0; i < n; ++i) {
    init[3 * i] = 0.01 + 1.98 * ((i * 17) % n) / double(n);
    init[3 * i + 1] = 0.01 + 1.98 * ((i * 37) % n) / double(n);
    init[3 * i + 2] = 0.01 + 1.98 * ((i * 101) % n) / double(n);
    for (int a = 0; a < 3; ++a) dest[3 * i + a] = 2.0 - init[3 * i + a];
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  std::vector<double> flux(E), evol(E), vol(G), sums(G), x(B * G);
  double bad = 0.0;
  for (int b = 0; b < B; ++b) {
    for (int i = 0; i < n; ++i) w[i] = 1.0 + 0.25 * b + 0.5 * ((i * 7 + b * 3) % 5);
    std::vector<int8_t> flying(n, 1);
    tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
    if (pumitally_get_flux(e, flux.data(), E) != 0 || pumitally::GetRegionResults(tally, 0, 0, sums.data(), G) != 0) {
      printf("GetRegionResults failed\n");
      return 1;
    }
    for (int g = 0; g < G; ++g) {
      double s = 0.0, a = 0.0;
      for (int64_t i = 0; i < E; ++i)
        if (region[i] == g) s += flux[i], a += std::fabs(flux[i]);
      bad = std::max(bad, std::fabs(sums[g] - s) / std::max(a, 1e-300));
      x[b * G + g] = sums[g];  // source normalisation mode 0: the divisor is 1
    }
    if (pumitally::EndBatch(tally) != 0) { printf("EndBatch failed\n"); return 1; }
  }
  if (pumitally_get_normalized_flux(e, nullptr, evol.data(), E) != 0 ||
      pumitally::GetRegionVolumes(tally, vol.data(), G) != 0) {
    printf("GetRegionVolumes failed\n");
    return 1;
  }
  std::vector<double> got[3];
  for (int kind = 0; kind < 3; ++kind) {
    got[kind].resize(G);
    if (pumitally::GetRegionBatchResults(tally, 0, kind, got[kind].data(), G) != 0) {
      printf("GetRegionBatchResults failed\n");
      return 1;
    }
  }
  for (int g = 0; g < G; ++g) {
    double v = 0.0, m = 0.0, s2 = 0.0;
    for (int64_t i = 0; i < E; ++i)
      if (region[i] == g) v += evol[i];
    for (int b = 0; b < B; ++b) m += x[b * G + g] / B;
    for (int b = 0; b < B; ++b) s2 += (x[b * G + g] - m) * (x[b * G + g] - m);
    const double se = std::sqrt(s2 / (B - 1) / B), rel = se / std::fabs(m);
    bad = std::max({bad, std::fabs(vol[g] - v) / v, std::fabs(got[0][g] - m / v) / std::fabs(m / v),
                    std::fabs(got[1][g] - se / v) / (se / v), std::fabs(got[2][g] - rel) / rel});
  }
  if (!(bad < 1e-12)) {
    printf("worst relative difference %g\n", bad);
    return 1;
  }
  if (pumitally::SetRegions(tally, nullptr, 0, 0) != 0 || pumitally_get_regions(e) != 0) {
    printf("removing the regions failed\n");
    return 1;
  }
  printf("REGIONS_OK\n");
  return 0;
}
