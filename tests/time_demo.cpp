// A C++ caller of the time filter (PumiTallyExtras.h) next to the reference class: two scores split between
// four time bins.  Particles fly straight along +x through a 2x2x2 box of unit cells at speed v, starting at
// time t0, so the length flown in bin [T_j, T_j+1) is v times the overlap of [t0, t0 + L/v] with the bin.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 64, nscores = 2, nt = 4;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  const double edges[nt + 1] = {0.0, 1.0, 2.0, 3.0, 4.0};
  const double unsorted[3] = {0.0, 2.0, 1.0};
  if (pumitally::SetTimeBins(tally, unsorted, 3) == 0) { printf("unsorted edges accepted\n"); return 1; }
  if (pumitally::SetScores(tally, nscores) != 0 || pumitally::SetTimeBins(tally, edges, nt + 1) != 0) {
    printf("SetScores / SetTimeBins failed\n");
    return 1;
  }
  std::vector<double> init(3 * n), dest(3 * n), w(n), r(size_t(n) * nscores), t(n), v(n);
  std::vector<int8_t> flying(n, 1);
  std::vector<double> want(size_t(nt) * nscores, 0.0);
  for (int i = 0; i < n; ++i) {
    const double y = 0.1 + 1.8 * (i % 8) / 7.0, z = 0.1 + 1.8 * (i / 8) / 7.0, x0 = 0.05 + 0.01 * (i % 5);
    init[3 * i] = x0; init[3 * i + 1] = y; init[3 * i + 2] = z;
    dest[3 * i] = 3.0; dest[3 * i + 1] = y; dest[3 * i + 2] = z;  // leaves through x = 2: clipped
    w[i] = 0.5 + 0.01 * i;
    t[i] = -0.5 + 0.07 * i;
    v[i] = 0.4 + 0.05 * (i % 9);
    const double t1 = t[i] + (2.0 - x0) / v[i];
    for (int j = 0; j < nt; ++j) {
      const double overlap = std::max(0.0, std::min(t1, edges[j + 1]) - std::max(t[i], edges[j]));
      for (int k = 0; k < nscores; ++k) {
        r[size_t(i) * nscores + k] = k == 0 ? 1.0 : 0.25 + 0.001 * i;
        want[size_t(j) * nscores + k] += w[i] * r[size_t(i) * nscores + k] * v[i] * overlap;
      }
    }
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  // with time bins the plain move and the scored move are refused and leave flying[] alone
  bool refused = false;
  try {
    tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
  } catch (const std::runtime_error &) {
    refused = true;
  }
  if (!refused || flying[0] != 1) { printf("plain move not refused\n"); return 1; }
  if (pumitally::MoveToNextLocationScored(tally, init.data(), dest.data(), flying.data(), w.data(), r.data(), nullptr,
                                          3 * n) == 0 || flying[0] != 1) {
    printf("scored move not refused\n");
    return 1;
  }
  if (pumitally::MoveToNextLocationTimed(tally, init.data(), dest.data(), flying.data(), w.data(), t.data(), v.data(),
                                         r.data(), nullptr, 3 * n) != 0) {
    printf("timed move failed\n");
    return 1;
  }
  for (int i = 0; i < n; ++i)
    if (flying[i] != 0) { printf("flying not reset\n"); return 1; }
  pumitally_engine *e = pumitally::engine_of(tally);
  if (pumitally_get_time_bins(e) != nt) { printf("time bins %d\n", pumitally_get_time_bins(e)); return 1; }
  const int64_t E = pumitally_num_elements(e);
  std::vector<double> flux(size_t(E) * nscores * nt);
  if (pumitally_get_flux(e, flux.data(), int64_t(flux.size())) != 0) { printf("get_flux failed\n"); return 1; }
  for (int j = 0; j < nt; ++j)
    for (int k = 0; k < nscores; ++k) {
      double total = 0.0;
      for (int64_t x = 0; x < E; ++x) total += flux[(size_t(j) * nscores + k) * E + x];
      const double ref = want[size_t(j) * nscores + k];
      if (std::fabs(total - ref) > 1e-9 * std::max(ref, 1.0)) {
        printf("time %d score %d: %.17g, expected %.17g\n", j, k, total, ref);
        return 1;
      }
    }
  tally.WriteTallyResults();
  printf("TIME_OK\n");
  return 0;
}
