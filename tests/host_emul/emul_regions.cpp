// TEST-ONLY host build of the region-sum order (batch_stats.cuh: build_region_plan, chunk_sum, region_sums_host), the
// order the region kernel of stats_kernels.cu runs.  Compiled by g++ so that it can be checked against math.fsum on a
// machine without a GPU; never linked into libpumitally.so.
#include <cstdint>

#include "batch_stats.cuh"

extern "C" {
// out[g] = the sum of values[e] over the elements e with region_of_internal[e] == g, in the plan's order.  Returns the
// number of levels of the plan.
int32_t ptb_region_sums(const int32_t *region_of_internal, int64_t E, int32_t nregions, const double *values,
                        double *out) {
  const ptb::RegionPlan p = ptb::build_region_plan(region_of_internal, E, nregions);
  const std::vector<double> s = ptb::region_sums_host(p, values);
  for (int32_t g = 0; g < nregions; ++g) out[g] = s[size_t(g)];
  return int32_t(p.levels.size());
}

int32_t ptb_region_chunk() { return ptb::kRegionChunk; }
}
