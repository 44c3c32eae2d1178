// A C++ caller of the scores (PumiTallyExtras.h) next to the reference class: three responses per particle
// tallied in one walk.  Particles fly straight along +x through a 2x2x2 box of unit cells, so every score
// must total sum_i w[i] * r[i,k] * (track length inside the box).
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 64, nscores = 3;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  if (pumitally::SetScores(tally, 9) == 0) { printf("nscores 9 accepted\n"); return 1; }
  if (pumitally::SetScores(tally, nscores) != 0) { printf("SetScores failed\n"); return 1; }
  std::vector<double> init(3 * n), dest(3 * n), w(n), r(size_t(n) * nscores);
  std::vector<int8_t> flying(n, 1);
  std::vector<double> want(nscores, 0.0);
  for (int i = 0; i < n; ++i) {
    const double y = 0.1 + 1.8 * (i % 8) / 7.0, z = 0.1 + 1.8 * (i / 8) / 7.0, x0 = 0.05 + 0.01 * (i % 5);
    init[3 * i] = x0; init[3 * i + 1] = y; init[3 * i + 2] = z;
    dest[3 * i] = 3.0; dest[3 * i + 1] = y; dest[3 * i + 2] = z;  // leaves through x = 2: clipped
    w[i] = 0.5 + 0.01 * i;
    for (int k = 0; k < nscores; ++k) {
      r[size_t(i) * nscores + k] = k == 0 ? 1.0 : 0.25 * k + 0.001 * i;
      want[k] += w[i] * r[size_t(i) * nscores + k] * (2.0 - x0);
    }
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  // with several scores the plain move is refused and leaves flying[] alone
  bool refused = false;
  try {
    tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
  } catch (const std::runtime_error &) {
    refused = true;
  }
  if (!refused || flying[0] != 1) { printf("plain move not refused\n"); return 1; }
  if (pumitally::MoveToNextLocationScored(tally, init.data(), dest.data(), flying.data(), w.data(), r.data(), nullptr,
                                          3 * n) != 0) {
    printf("scored move failed\n");
    return 1;
  }
  for (int i = 0; i < n; ++i)
    if (flying[i] != 0) { printf("flying not reset\n"); return 1; }
  pumitally_engine *e = pumitally::engine_of(tally);
  const int64_t E = pumitally_num_elements(e);
  std::vector<double> flux(size_t(E) * nscores);
  if (pumitally_get_flux(e, flux.data(), int64_t(flux.size())) != 0) { printf("get_flux failed\n"); return 1; }
  for (int k = 0; k < nscores; ++k) {
    double total = 0.0;
    for (int64_t j = 0; j < E; ++j) total += flux[size_t(k) * E + j];
    if (std::fabs(total - want[k]) > 1e-12 * want[k]) {
      printf("score %d: %.17g, expected %.17g\n", k, total, want[k]);
      return 1;
    }
  }
  tally.WriteTallyResults();
  printf("SCORES_OK\n");
  return 0;
}
