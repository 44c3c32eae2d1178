// A C++ caller of the weight windows (PumiTallyExtras.h) next to the reference class: three batches through a 2x2x2 box
// with batch statistics on, GenerateWeightWindows, and the lookups at the particles and at points checked against
// GetWeightWindows gathered through the particles' elements and LocatePoints.  SetWeightWindows round-trips a table and
// refuses a NaN bound.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 2048, B = 3;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  const int64_t E = pumitally_num_elements(e);
  std::vector<int32_t> groups(n, 0);
  std::vector<double> lo(n), hi(n);
  if (pumitally::WeightWindowsAtParticles(tally, groups.data(), lo.data(), hi.data(), n) == 0) {
    printf("lookup accepted before CopyInitialPosition\n");
    return 1;
  }
  if (pumitally::SetBatchStatistics(tally, 1) != 0) { printf("SetBatchStatistics failed\n"); return 1; }
  std::vector<double> init(3 * n), dest(3 * n), w(n);
  for (int i = 0; i < n; ++i) {
    init[3 * i] = 0.01 + 1.98 * ((i * 17) % n) / double(n);
    init[3 * i + 1] = 0.01 + 1.98 * ((i * 37) % n) / double(n);
    init[3 * i + 2] = 0.01;
    dest[3 * i] = init[3 * i];
    dest[3 * i + 1] = init[3 * i + 1];
    dest[3 * i + 2] = 0.2 + 1.7 * ((i * 101) % n) / double(n);
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  for (int b = 0; b < B; ++b) {
    for (int i = 0; i < n; ++i) w[i] = 1.0 + 0.25 * b + 0.5 * ((i * 7 + b * 3) % 5);
    std::vector<int8_t> flying(n, 1);
    tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
    if (pumitally::EndBatch(tally) != 0) { printf("EndBatch failed\n"); return 1; }
  }
  const double ratio = 5.0;
  if (pumitally::GenerateWeightWindows(tally, 0, 0, 0, ratio, INFINITY) != 0 || pumitally_get_weight_window_groups(e) != 1) {
    printf("GenerateWeightWindows failed\n");
    return 1;
  }
  std::vector<double> tlo(E), thi(E);
  if (pumitally::GetWeightWindows(tally, tlo.data(), thi.data(), E) != 0) { printf("GetWeightWindows failed\n"); return 1; }
  double top = 0.0;
  for (int64_t i = 0; i < E; ++i) top = std::fmax(top, tlo[i]);
  if (top != 2.0 / (ratio + 1.0)) { printf("largest lower bound %.17g\n", top); return 1; }
  std::vector<int32_t> elem(n);
  if (pumitally_get_element_ids(e, elem.data(), n) != 0 ||
      pumitally::WeightWindowsAtParticles(tally, nullptr, lo.data(), hi.data(), n) != 0) {
    printf("WeightWindowsAtParticles failed\n");
    return 1;
  }
  for (int i = 0; i < n; ++i)
    if (lo[i] != tlo[size_t(elem[i])] || hi[i] != thi[size_t(elem[i])]) { printf("particle %d\n", i); return 1; }
  std::vector<double> pts(3 * n);
  std::vector<int32_t> pe(n);
  for (int i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) pts[3 * i + a] = -0.5 + 3.0 * (((i + 1) * (a + 3) * 7919) % 1000) / 1000.0;
  if (pumitally::LocatePoints(tally, pts.data(), n, pe.data()) != 0 ||
      pumitally::WeightWindowsAtPoints(tally, pts.data(), n, nullptr, lo.data(), hi.data()) != 0) {
    printf("WeightWindowsAtPoints failed\n");
    return 1;
  }
  for (int i = 0; i < n; ++i) {
    const double wl = pe[i] >= 0 ? tlo[size_t(pe[i])] : -1.0, wh = pe[i] >= 0 ? thi[size_t(pe[i])] : -1.0;
    if (lo[i] != wl || hi[i] != wh) { printf("point %d\n", i); return 1; }
  }
  // a table of two groups round-trips; a NaN bound is refused and changes nothing
  std::vector<double> slo(2 * E), shi(2 * E), glo(2 * E), ghi(2 * E);
  for (int64_t i = 0; i < 2 * E; ++i) {
    slo[i] = i % 5 == 0 ? 0.0 : 0.1 * double(i + 1);
    shi[i] = 3.0 * slo[i] + 1.0;
  }
  if (pumitally::SetWeightWindows(tally, slo.data(), shi.data(), 2 * E, 2) != 0 ||
      pumitally::GetWeightWindows(tally, glo.data(), ghi.data(), 2 * E) != 0) {
    printf("SetWeightWindows failed\n");
    return 1;
  }
  slo[3] = NAN;
  if (pumitally::SetWeightWindows(tally, slo.data(), shi.data(), 2 * E, 2) == 0) { printf("NaN accepted\n"); return 1; }
  std::vector<double> again(2 * E), again_hi(2 * E);
  pumitally::GetWeightWindows(tally, again.data(), again_hi.data(), 2 * E);
  for (int64_t i = 0; i < 2 * E; ++i) {
    const bool none = i % 5 == 0;
    if (glo[i] != (none ? -1.0 : 0.1 * double(i + 1)) || ghi[i] != (none ? -1.0 : shi[i]) || again[i] != glo[i]) {
      printf("round trip %lld\n", (long long)i);
      return 1;
    }
  }
  printf("WEIGHT_WINDOWS_OK\n");
  return 0;
}
