// A C++ caller of the collision estimator (PumiTallyExtras.h) next to the reference class: after one move every flight
// that ended inside the 2x2x2 box is a collision with weight 1, then a few collision sites elsewhere are located.
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 2048;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  if (pumitally::SetCollisionEstimator(tally, 1) != 0) { printf("SetCollisionEstimator failed\n"); return 1; }
  std::vector<double> init(3 * n), dest(3 * n), w(n, 1.0);
  std::vector<int8_t> flying(n, 1), collided(n, 1);
  for (int i = 0; i < n; ++i) {
    init[3 * i] = 0.01 + 1.98 * ((i * 17) % n) / double(n);
    init[3 * i + 1] = 0.01 + 1.98 * ((i * 37) % n) / double(n);
    init[3 * i + 2] = 0.01 + 1.98 * ((i * 101) % n) / double(n);
    for (int a = 0; a < 3; ++a) dest[3 * i + a] = 2.0 - init[3 * i + a];
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
  if (pumitally::TallyCollisionsAtParticles(tally, collided.data(), w.data(), n) != 0) {
    printf("TallyCollisionsAtParticles failed\n");
    return 1;
  }
  const double pts[] = {0.3, 0.4, 0.5, 1.7, 1.2, 0.9, 3.0, 1.0, 1.0, NAN, 1.0, 1.0};
  const double pw[] = {2.0, 2.0, 2.0, 2.0};
  if (pumitally::TallyCollisions(tally, pts, 4, pw) != 0) { printf("TallyCollisions failed\n"); return 1; }
  const int64_t E = pumitally_num_elements(e);
  std::vector<double> raw(E);
  if (pumitally_get_collision_results(e, 0, raw.data(), E) != 0) { printf("get_collision_results failed\n"); return 1; }
  double sum = 0.0;
  for (double v : raw) sum += v;
  const int64_t tallied = pumitally_get_option(e, "collisions"), outside = pumitally_get_option(e, "collisions_outside"),
                rejected = pumitally_get_option(e, "collisions_rejected");
  if (sum != n + 4.0 || tallied != n + 2 || outside != 1 || rejected != 1) {
    printf("sum %g, tallied %lld, outside %lld, rejected %lld\n", sum, (long long)tallied, (long long)outside,
           (long long)rejected);
    return 1;
  }
  printf("COLLISIONS_OK\n");
  return 0;
}
