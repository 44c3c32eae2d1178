// A C++ caller of the point queries (PumiTallyExtras.h) next to the reference class: a thermal solver's points -- some
// inside the 2x2x2 box, some outside -- located and given the normalised flux of the tally after one move.
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 2048;
  pumitally::PumiTally tally("box:2,2,2", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  std::vector<double> init(3 * n), dest(3 * n), w(n, 1.0);
  std::vector<int8_t> flying(n, 1);
  for (int i = 0; i < n; ++i) {
    init[3 * i] = 0.01 + 1.98 * ((i * 17) % n) / double(n);
    init[3 * i + 1] = 0.01 + 1.98 * ((i * 37) % n) / double(n);
    init[3 * i + 2] = 0.01 + 1.98 * ((i * 101) % n) / double(n);
    for (int a = 0; a < 3; ++a) dest[3 * i + a] = 2.0 - init[3 * i + a];
  }
  // points may be located before any particle is placed
  const double pts[] = {0.3, 0.4, 0.5, 1.7, 1.2, 0.9, 3.0, 1.0, 1.0, -0.1, 0.5, 0.5, NAN, 1.0, 1.0};
  const int64_t npts = 5;
  std::vector<int32_t> elem(npts), elem2(npts);
  if (pumitally::LocatePoints(tally, pts, npts, elem.data()) != 0) { printf("LocatePoints failed\n"); return 1; }
  if (elem[0] < 0 || elem[1] < 0 || elem[2] != -1 || elem[3] != -1 || elem[4] != -1) {
    printf("elements %d %d %d %d %d\n", elem[0], elem[1], elem[2], elem[3], elem[4]);
    return 1;
  }
  tally.CopyInitialPosition(init.data(), 3 * n);
  tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
  const int64_t E = pumitally_num_elements(e);
  std::vector<double> nf(E), vol(E), val(npts);
  if (pumitally_get_normalized_flux(e, nf.data(), vol.data(), E) != 0 ||
      pumitally::EvaluatePoints(tally, pts, npts, val.data(), npts, elem2.data()) != 0) {
    printf("EvaluatePoints failed\n");
    return 1;
  }
  for (int k = 0; k < 2; ++k)
    if (elem2[k] != elem[k] || val[k] != nf[elem[k]]) { printf("point %d: %g vs %g\n", k, val[k], nf[elem[k]]); return 1; }
  for (int k = 2; k < 5; ++k)
    if (!std::isnan(val[k])) { printf("point %d outside: %g\n", k, val[k]); return 1; }
  if (pumitally::EvaluatePoints(tally, pts, npts, val.data(), npts + 1) == 0) { printf("bad n accepted\n"); return 1; }
  printf("LOCATE_OK\n");
  return 0;
}
