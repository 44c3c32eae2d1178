// TEST-ONLY host build of the weight-window arithmetic (weight_windows.cuh), the code the kernels of ww_kernels.cu run.
// Compiled by g++ with -ffp-contract=off so that it can be checked against numpy bit for bit on a machine without a
// GPU; never linked into libpumitally.so.
#include <cmath>
#include <cstdint>

#include "weight_windows.cuh"

extern "C" {
// The MAGIC step over ngroups groups of E m0 results each, [group][element], in the order the two kernels run it: the
// largest eligible phi of every group (phimax[g]), then every window with c = 2 / (ratio + 1) computed once.
void ptb_ww_generate(const double *mean, const double *m2, const double *volume, int64_t E, int32_t ngroups, double nb,
                     double max_rel_err, double ratio, double *lower, double *upper, double *phimax) {
  const double c = 2.0 / (ratio + 1.0);
  for (int64_t g = 0; g < ngroups; ++g) {
    double best = 0.0;
    for (int64_t e = 0; e < E; ++e)
      best = std::fmax(best, ptb::ww_max_candidate(mean[g * E + e], m2[g * E + e], nb, volume[e], max_rel_err));
    phimax[g] = best;
    for (int64_t e = 0; e < E; ++e)
      ptb::ww_generate(mean[g * E + e], m2[g * E + e], nb, volume[e], max_rel_err, best, c, ratio, lower[g * E + e],
                       upper[g * E + e]);
  }
}

int32_t ptb_ww_entry(double lower, double upper) { return ptb::ww_entry(lower, upper); }

int64_t ptb_ww_slot(int32_t group, int32_t ngroups, int32_t elem, int64_t E) {
  return ptb::ww_slot(group, ngroups, elem, E);
}

double ptb_ww_no_window() { return ptb::kNoWindow; }
}
