// A C++ caller of the mesh source (PumiTallyExtras.h) next to the reference class: an R2S-style step on a 2x2x2 box --
// one strength per element and two photon groups, SetSource with per_volume, SampleSource with placement, then one
// move from the placed particles.  Checks the group count, Q, the placed elements and positions, that
// CopyInitialPosition is refused after a placement, and that a NaN strength is refused.
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 4096;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  const int64_t E = pumitally_num_elements(e);
  std::vector<double> q(2 * E);
  for (int64_t k = 0; k < 2 * E; ++k) q[k] = (k < E) ? 1.0 : 0.5 * double(k % 3);
  if (pumitally::SetSource(tally, q.data(), nullptr, 2 * E, 2, 1) != 0 || pumitally::GetSourceGroups(tally) != 2) {
    printf("SetSource failed\n");
    return 1;
  }
  double Q = 0.0;
  if (pumitally::GetSourceStrength(tally, &Q) != 0 || !(std::fabs(Q - 12.0) < 1e-9)) {  // 8 * 1 + 8 * mean(0, .5, 1)
    printf("source strength %.17g\n", Q);
    return 1;
  }
  std::vector<double> xyz(3 * n), w(n);
  std::vector<int32_t> elem(n), group(n), ids(n);
  if (pumitally::SampleSource(tally, 2024, 0, n, xyz.data(), elem.data(), group.data(), w.data(), 1) != 0) {
    printf("SampleSource failed\n");
    return 1;
  }
  std::vector<double> pos(3 * n);
  if (pumitally_get_element_ids(e, ids.data(), n) != 0 || pumitally_get_positions(e, pos.data(), 3 * n) != 0) {
    printf("accessors failed\n");
    return 1;
  }
  int groups[2] = {0, 0};
  for (int i = 0; i < n; ++i) {
    if (ids[i] != elem[i] || pos[3 * i] != xyz[3 * i] || pos[3 * i + 2] != xyz[3 * i + 2] || w[i] != 1.0) {
      printf("particle %d not placed at its sample\n", i);
      return 1;
    }
    if (group[i] == 1 && q[E + elem[i]] == 0.0) {
      printf("sample %d in an entry of zero strength\n", i);
      return 1;
    }
    ++groups[group[i]];
  }
  if (groups[0] < n / 2 || groups[1] == 0) {  // 8 : 4 expected
    printf("group counts %d %d\n", groups[0], groups[1]);
    return 1;
  }
  if (pumitally_copy_initial_position(e, xyz.data(), 3 * n) == 0) {
    printf("CopyInitialPosition accepted after a placement\n");
    return 1;
  }
  std::vector<double> dest(xyz);
  for (int i = 0; i < n; ++i) dest[3 * i + 2] = 1.0;
  std::vector<int8_t> flying(n, 1);
  tally.MoveToNextLocation(xyz.data(), dest.data(), flying.data(), w.data(), 3 * n);
  std::vector<double> flux(E);
  double sum = 0.0, want = 0.0;
  if (pumitally_get_flux(e, flux.data(), E) != 0) { printf("get_flux failed\n"); return 1; }
  for (int64_t k = 0; k < E; ++k) sum += flux[k];
  for (int i = 0; i < n; ++i) want += std::fabs(xyz[3 * i + 2] - 1.0);
  if (!(std::fabs(sum - want) <= 1e-9 * want)) {
    printf("flux %.17g, track length %.17g\n", sum, want);
    return 1;
  }
  q[3] = NAN;
  if (pumitally::SetSource(tally, q.data(), nullptr, 2 * E, 2, 1) == 0 || pumitally::GetSourceGroups(tally) != 2) {
    printf("a NaN strength was accepted\n");
    return 1;
  }
  printf("SOURCE_OK\n");
  return 0;
}
