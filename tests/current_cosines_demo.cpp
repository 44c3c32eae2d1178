// A C++ caller of the cosine bins of the face currents (PumiTallyExtras.h): one move through a 3x3x3 box with face
// currents split into three cosine bins.  The cosine axis must follow the score-bin axis (n = C * E * 4 and C), the
// sum over the bins of edges that cover [0, 1] must be the current without bins, a bad edge set and a wrong n must be
// refused, and removing the bins must restore the shapes.
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 4096;
  pumitally::PumiTally tally("box:3,3,3", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  const int64_t E = pumitally_num_elements(e);
  const double edges[4] = {0.0, 0.3, 0.75, 1.0}, bad[3] = {0.0, 0.8, 0.5};
  if (pumitally::SetFaceCurrents(tally, 1) != 0 || pumitally::SetCurrentCosineBins(tally, edges, 4) != 0 ||
      pumitally::GetCurrentCosineBins(tally) != 3) {
    printf("SetCurrentCosineBins failed\n");
    return 1;
  }
  if (pumitally::SetCurrentCosineBins(tally, bad, 3) == 0 || pumitally::GetCurrentCosineBins(tally) != 3) {
    printf("decreasing edges were accepted\n");
    return 1;
  }
  std::vector<double> init(3 * n), dest(3 * n), w(n);
  for (int i = 0; i < n; ++i) {
    init[3 * i] = 0.05 + 2.9 * ((i * 17) % n) / double(n);
    init[3 * i + 1] = 0.05 + 2.9 * ((i * 37) % n) / double(n);
    init[3 * i + 2] = 0.05 + 2.9 * ((i * 71) % n) / double(n);
    dest[3 * i] = init[3 * i] + 2.0 * std::cos(0.37 * i);
    dest[3 * i + 1] = init[3 * i + 1] + 2.0 * std::sin(0.37 * i);
    dest[3 * i + 2] = init[3 * i + 2] + 1.5 * std::cos(0.11 * i);
    w[i] = 0.125 * (1 + i % 16);
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  std::vector<int8_t> flying(n, 1);
  tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
  std::vector<double> out(3 * 4 * E), leak(3);
  if (pumitally::GetFaceCurrentResults(tally, 0, 0, out.data(), 3 * 4 * E) != 0 ||
      pumitally::GetLeakage(tally, 0, leak.data(), 3) != 0) {
    printf("readout failed\n");
    return 1;
  }
  if (pumitally::GetFaceCurrentResults(tally, 0, 0, out.data(), 4 * E) == 0 ||
      pumitally::GetLeakage(tally, 0, leak.data(), 1) == 0) {
    printf("the n of a tally without cosine bins was accepted\n");
    return 1;
  }
  double binned = 0.0, leaked = 0.0;
  for (double v : out) binned += v;
  for (double v : leak) leaked += v;
  // the same move again without cosine bins: the same totals (dyadic weights: exact in any order)
  if (pumitally::SetCurrentCosineBins(tally, nullptr, 0) != 0 || pumitally::GetCurrentCosineBins(tally) != 0) {
    printf("removing the cosine bins failed\n");
    return 1;
  }
  std::vector<int8_t> flying2(n, 1);  // (from init again: a relocation with the tally off, then the same flights)
  tally.MoveToNextLocation(init.data(), dest.data(), flying2.data(), w.data(), 3 * n);
  std::vector<double> plain(4 * E), leak1(1);
  if (pumitally::GetFaceCurrentResults(tally, 0, 0, plain.data(), 4 * E) != 0 ||
      pumitally::GetLeakage(tally, 0, leak1.data(), 1) != 0) {
    printf("readout without cosine bins failed\n");
    return 1;
  }
  double total = 0.0;
  for (double v : plain) total += v;
  if (total != binned || leak1[0] != leaked || !(total > 0.0)) {
    printf("binned %g, without bins %g; leakage %g, %g\n", binned, total, leaked, leak1[0]);
    return 1;
  }
  printf("CURRENT_COSINES_OK %g %g\n", total, leaked);
  return 0;
}
