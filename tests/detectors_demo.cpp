// A C++ caller of the point detectors (PumiTallyExtras.h) next to the reference class: one detector in the middle of a
// homogeneous 2x2x2 box and a few isotropic source points; the estimate of each is exp(-Sigma R) / (4 pi R^2).
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  pumitally::PumiTally tally("box:2,2,2", 16, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  const double det[] = {1.0, 1.0, 1.0}, r0[] = {0.0};
  if (pumitally::SetPointDetectors(tally, det, 1, r0) != 0) { printf("SetPointDetectors failed\n"); return 1; }
  const int64_t E = pumitally_num_elements(e);
  const double sig = 0.7;
  std::vector<double> sigma(E, sig);
  if (pumitally::SetDetectorCrossSections(tally, sigma.data(), E) != 0) { printf("SetDetectorCrossSections failed\n"); return 1; }
  const double pts[] = {0.3, 0.4, 0.5, 1.7, 1.2, 0.9, 3.0, 1.0, 1.0, NAN, 1.0, 1.0};
  const double w[] = {1.0, 2.0, 1.0, 1.0};
  if (pumitally::TallyDetectors(tally, pts, 4, w) != 0) { printf("TallyDetectors failed\n"); return 1; }
  double got = 0.0;
  if (pumitally::GetDetectorResults(tally, 0, &got, 1) != 0) { printf("GetDetectorResults failed\n"); return 1; }
  double want = 0.0;
  for (int i = 0; i < 2; ++i) {
    const double dx = det[0] - pts[3 * i], dy = det[1] - pts[3 * i + 1], dz = det[2] - pts[3 * i + 2];
    const double R = std::sqrt(dx * dx + dy * dy + dz * dz);
    want += w[i] * std::exp(-sig * R) / (4.0 * M_PI * R * R);
  }
  const int64_t rays = pumitally_get_option(e, "detector_rays"), outside = pumitally_get_option(e, "detector_events_outside"),
                rejected = pumitally_get_option(e, "detector_events_rejected");
  if (std::fabs(got - want) > 1e-12 * want || rays != 2 || outside != 1 || rejected != 1) {
    printf("got %.17g want %.17g, rays %lld, outside %lld, rejected %lld\n", got, want, (long long)rays,
           (long long)outside, (long long)rejected);
    return 1;
  }
  printf("DETECTORS_OK\n");
  return 0;
}
