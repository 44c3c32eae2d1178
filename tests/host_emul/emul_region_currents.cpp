// TEST-ONLY host build of the region-current pair plan (batch_stats.cuh: build_region_current_plan, face_area), the
// plan the engine uploads for launch_region_sums and launch_region_net.  Compiled by g++ so that it can be checked
// against an independent numpy construction on a machine without a GPU; never linked into libpumitally.so.
#include <cstdint>
#include <cstring>

#include "batch_stats.cuh"

namespace {
ptb::RegionCurrentPlan g_plan;
}

extern "C" {
// Builds the plan of region[E] over t2t [4E] with slot_area [4E]; returns the pair count P.
int64_t ptb_rc_build(const int32_t *region, const int32_t *t2t, int64_t E, const double *slot_area) {
  g_plan = ptb::build_region_current_plan(region, t2t, E, slot_area);
  return int64_t(g_plan.from.size());
}
int64_t ptb_rc_nslots() { return int64_t(g_plan.sums.elems.size()); }
int32_t ptb_rc_levels() { return int32_t(g_plan.sums.levels.size()); }
// from, to, rev, area [P]; first [P + 1]; slots [nslots]
void ptb_rc_get(int32_t *from, int32_t *to, int32_t *rev, double *area, int64_t *first, int32_t *slots) {
  const size_t P = g_plan.from.size();
  std::memcpy(from, g_plan.from.data(), P * sizeof(int32_t));
  std::memcpy(to, g_plan.to.data(), P * sizeof(int32_t));
  std::memcpy(rev, g_plan.rev.data(), P * sizeof(int32_t));
  std::memcpy(area, g_plan.area.data(), P * sizeof(double));
  std::memcpy(first, g_plan.first.data(), (P + 1) * sizeof(int64_t));
  std::memcpy(slots, g_plan.sums.elems.data(), g_plan.sums.elems.size() * sizeof(int32_t));
}
// out[4 e + f] = face_area of every face
void ptb_face_areas(const double *coords, const int32_t *t2v, int64_t E, double *out) {
  for (int64_t e = 0; e < E; ++e)
    for (int f = 0; f < 4; ++f) out[4 * e + f] = ptb::face_area(coords, t2v, e, f);
}
}
