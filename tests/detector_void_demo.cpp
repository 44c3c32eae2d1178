// A C++ caller of the detector void (PumiTallyExtras.h): a detector outside a homogeneous 2x2x2 box and a few isotropic
// source points inside and outside it; the estimate of each is exp(-Sigma l_inside) / (4 pi R^2).
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  pumitally::PumiTally tally("box:2,2,2", 16, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  const double det[] = {5.0, 1.0, 1.0}, r0[] = {0.0};
  if (pumitally::SetPointDetectors(tally, det, 1, r0) == 0) { printf("an outside detector was accepted\n"); return 1; }
  if (pumitally::SetDetectorVoid(tally, true) != 0 || !pumitally::GetDetectorVoid(tally)) {
    printf("SetDetectorVoid failed\n");
    return 1;
  }
  if (pumitally::SetPointDetectors(tally, det, 1, r0) != 0) { printf("SetPointDetectors failed\n"); return 1; }
  const int64_t E = pumitally_num_elements(e);
  const double sig = 0.7;
  std::vector<double> sigma(E, sig);
  if (pumitally::SetDetectorCrossSections(tally, sigma.data(), E) != 0) { printf("SetDetectorCrossSections failed\n"); return 1; }
  // on the line y = z = 1: the events at x = 0.5 and 1.5 cross 1.5 and 0.5 of the box, the one at x = -1 all 2
  const double pts[] = {0.5, 1.0, 1.0, 1.5, 1.0, 1.0, -1.0, 1.0, 1.0};
  const double w[] = {1.0, 2.0, 1.0}, inside[] = {1.5, 0.5, 2.0};
  if (pumitally::TallyDetectors(tally, pts, 3, w) != 0) { printf("TallyDetectors failed\n"); return 1; }
  double got = 0.0;
  if (pumitally::GetDetectorResults(tally, 0, &got, 1) != 0) { printf("GetDetectorResults failed\n"); return 1; }
  double want = 0.0;
  for (int i = 0; i < 3; ++i) {
    const double R = det[0] - pts[3 * i];
    want += w[i] * std::exp(-sig * inside[i]) / (4.0 * M_PI * R * R);
  }
  const int64_t rays = pumitally_get_option(e, "detector_rays"), outside = pumitally_get_option(e, "detector_events_outside"),
                entries = pumitally_get_option(e, "detector_hull_entries");
  if (std::fabs(got - want) > 1e-12 * want || rays != 3 || outside != 0 || entries != 1) {
    printf("got %.17g want %.17g, rays %lld, outside %lld, hull entries %lld\n", got, want, (long long)rays,
           (long long)outside, (long long)entries);
    return 1;
  }
  if (pumitally::SetDetectorVoid(tally, false) == 0) { printf("switching off with a detector outside was accepted\n"); return 1; }
  printf("DETECTOR_VOID_OK\n");
  return 0;
}
