// A C++ caller of the face currents (PumiTallyExtras.h) next to the reference class: two batches through a 3x3x3 box
// with batch statistics on.  The incoming current of every interior face must equal the outgoing current of the same
// face seen from the neighbour (pumitally_get_adjacency), the leakage must be the outgoing current summed over the hull
// faces, and a call with the wrong n must be refused.
#include <cmath>
#include <cstdio>
#include <vector>

#include "pumitally/PumiTallyExtras.h"

int main(int argc, char **argv) {
  const int n = 4096;
  pumitally::PumiTally tally("box:3,3,3", n, argc, argv);
  pumitally_engine *e = pumitally::engine_of(tally);
  const int64_t E = pumitally_num_elements(e);
  if (pumitally::SetFaceCurrents(tally, 1) != 0 || pumitally::GetFaceCurrents(tally) != 1) {
    printf("SetFaceCurrents failed\n");
    return 1;
  }
  if (pumitally::SetBatchStatistics(tally, 1) != 0) { printf("SetBatchStatistics failed\n"); return 1; }
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
  for (int b = 0; b < 2; ++b) {
    std::vector<int8_t> flying(n, 1);
    tally.MoveToNextLocation(init.data(), dest.data(), flying.data(), w.data(), 3 * n);
    if (b == 0) {
      std::vector<double> out(4 * E), in(4 * E), leak(1);
      std::vector<int32_t> adj(4 * E);
      if (pumitally::GetFaceCurrentResults(tally, 0, 0, out.data(), 4 * E) != 0 ||
          pumitally::GetFaceCurrentResults(tally, 1, 0, in.data(), 4 * E) != 0 ||
          pumitally::GetLeakage(tally, 0, leak.data(), 1) != 0 || pumitally_get_adjacency(e, adj.data(), 4 * E) != 0) {
        printf("readout failed\n");
        return 1;
      }
      double hull = 0.0, total = 0.0;
      for (int64_t i = 0; i < E; ++i)
        for (int f = 0; f < 4; ++f) {
          const int32_t nb = adj[4 * i + f];
          total += out[4 * i + f];
          if (nb < 0) {
            hull += out[4 * i + f];
            if (in[4 * i + f] != 0.0) { printf("current entering through the hull\n"); return 1; }
            continue;
          }
          int back = -1;
          for (int q = 0; q < 4; ++q)
            if (adj[4 * nb + q] == i) back = q;
          if (back < 0 || in[4 * i + f] != out[4 * nb + back]) {
            printf("element %lld face %d: in %g, neighbour's out %g\n", (long long)i, f, in[4 * i + f],
                   back < 0 ? -1.0 : out[4 * nb + back]);
            return 1;
          }
        }
      if (hull != leak[0] || !(hull > 0.0) || !(total > hull)) {
        printf("leakage %g, hull sum %g, total %g\n", leak[0], hull, total);
        return 1;
      }
      if (pumitally::GetFaceCurrentResults(tally, 0, 0, out.data(), 4 * E - 1) == 0 ||
          pumitally::GetLeakage(tally, 0, leak.data(), 2) == 0 ||
          pumitally::GetFaceCurrentResults(tally, 0, 1, out.data(), 4 * E) == 0) {
        printf("a wrong n, or batch results before a batch, was accepted\n");
        return 1;
      }
    }
    if (pumitally::EndBatch(tally) != 0) { printf("EndBatch failed\n"); return 1; }
  }
  std::vector<double> mean(4 * E), err(4 * E), leak(1);
  if (pumitally::GetFaceCurrentResults(tally, 0, 1, mean.data(), 4 * E) != 0 ||
      pumitally::GetFaceCurrentResults(tally, 0, 2, err.data(), 4 * E) != 0 ||
      pumitally::GetLeakage(tally, 1, leak.data(), 1) != 0 || !(leak[0] > 0.0)) {
    printf("batch readout failed\n");
    return 1;
  }
  printf("FACE_CURRENTS_OK %lld elements, leakage %g\n", (long long)E, leak[0]);
  return 0;
}
