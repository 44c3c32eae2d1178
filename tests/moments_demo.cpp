// A C++ caller of the linear flux moments (PumiTallyExtras.h) next to the reference class: one SetMoments, and the
// reference's own MoveToNextLocation tallies gradients.  Particles fly along +x through a 2x2x2 box of unit cells from
// x = 0.01, with lengths spread evenly over [0, 1.98]: the flux falls linearly along x, so the gradient's x component
// is negative and its y and z components are small.
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 4096;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  if (pumitally::SetMoments(tally, 2) == 0) { printf("order 2 accepted\n"); return 1; }
  if (pumitally::SetMoments(tally, 1) != 0) { printf("SetMoments failed\n"); return 1; }
  pumitally_engine *e = pumitally::engine_of(tally);
  if (pumitally_get_moments(e) != 1) { printf("moments %d\n", pumitally_get_moments(e)); return 1; }
  std::vector<double> init(3 * n), dest(3 * n), w(n, 1.0);
  std::vector<int8_t> flying(n, 1);
  double total = 0.0;
  for (int i = 0; i < n; ++i) {
    const double y = 0.01 + 1.98 * ((i * 37) % n) / double(n), z = 0.01 + 1.98 * ((i * 101) % n) / double(n);
    const double len = 1.98 * (i + 0.5) / n;
    init[3 * i] = 0.01; init[3 * i + 1] = y; init[3 * i + 2] = z;
    dest[3 * i] = 0.01 + len; dest[3 * i + 1] = y; dest[3 * i + 2] = z;
    total += len;
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
  const int64_t E = pumitally_num_elements(e);
  std::vector<double> flux(E), m1(3 * E), g(3 * E), vol(E), nf(E);
  if (pumitally_get_flux(e, flux.data(), E) != 0 || pumitally_get_flux_moments(e, m1.data(), 3 * E) != 0 ||
      pumitally_get_flux_gradient(e, g.data(), 3 * E) != 0 || pumitally_get_normalized_flux(e, nf.data(), vol.data(), E) != 0) {
    printf("accessors failed\n");
    return 1;
  }
  double sum = 0.0, gv[3] = {0, 0, 0}, v = 0.0;
  for (int64_t x = 0; x < E; ++x) {
    sum += flux[x];
    for (int a = 0; a < 3; ++a) gv[a] += g[3 * x + a] * vol[x];
    v += vol[x];
  }
  for (int a = 0; a < 3; ++a) gv[a] /= v;
  if (std::fabs(sum - total) > 1e-9 * total) { printf("flux %.17g, expected %.17g\n", sum, total); return 1; }
  // phi(x) = (n / 4) * (1 - x / 1.98) per unit area: d phi / dx = -n / (4 * 1.98)
  const double want = -n / (4.0 * 1.98);
  if (!(std::fabs(gv[0] - want) < 0.1 * std::fabs(want)) || std::fabs(gv[1]) > 0.1 * std::fabs(want) ||
      std::fabs(gv[2]) > 0.1 * std::fabs(want)) {
    printf("mean gradient (%g, %g, %g), expected (%g, 0, 0)\n", gv[0], gv[1], gv[2], want);
    return 1;
  }
  tally.WriteTallyResults();
  printf("MOMENTS_OK\n");
  return 0;
}
