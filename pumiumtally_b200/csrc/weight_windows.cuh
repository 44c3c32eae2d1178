// Weight windows (engine.cu, set_weight_windows / generate_weight_windows / the lookups; ww_kernels.cu): one (lower,
// upper) pair per energy group and element, generated from the batch statistics by the MAGIC step.
//
// __host__ __device__ so that tests/ can compile the same arithmetic with g++ (tests/host_emul/emul_weight_windows.cpp).
#pragma once
#include <cfloat>

#include "batch_stats.cuh"

namespace ptb {

// The stored value of "no window", both bounds.
constexpr double kNoWindow = -1.0;

// A set_weight_windows entry: 0 no window (lower <= 0, upper unread), 1 a window, -1 refused (a bound that is NaN or
// infinite, or upper <= lower).
PTB_HD int ww_entry(double lower, double upper) {
  if (lower <= 0.0) return 0;
  return (lower <= DBL_MAX && upper <= DBL_MAX && upper > lower) ? 1 : -1;
}

// phi and r of one m0 result of nb batches in an element of volume `volume`: kinds 0 and 2 of batch_readout, the values
// pumitally_get_batch_results returns.  The element is eligible when phi is finite and > 0 and r <= max_rel_err.
PTB_HD bool ww_eligible(double mean, double m2, double nb, double volume, double max_rel_err, double &phi) {
  phi = batch_readout(mean, 0.0, nb, volume, 0);
  const double r = batch_readout(mean, m2, nb, volume, 2);
  return phi > 0.0 && phi <= DBL_MAX && r <= max_rel_err;
}

// What the element adds to its group's maximum: phi when eligible, 0 otherwise (the maximum of a group without an
// eligible element stays 0).
PTB_HD double ww_max_candidate(double mean, double m2, double nb, double volume, double max_rel_err) {
  double phi;
  return ww_eligible(mean, m2, nb, volume, max_rel_err, phi) ? phi : 0.0;
}

// The window of one element, phimax the largest eligible phi of its group and c = 2 / (ratio + 1), computed once by the
// caller: lower = (phi / phimax) * c, upper = lower * ratio, so that the window's centre (lower + upper) / 2 is
// phi / phimax.  An ineligible element gets (kNoWindow, kNoWindow).
PTB_HD void ww_generate(double mean, double m2, double nb, double volume, double max_rel_err, double phimax, double c,
                        double ratio, double &lower, double &upper) {
  double phi;
  if (ww_eligible(mean, m2, nb, volume, max_rel_err, phi)) {
    lower = (phi / phimax) * c;
    upper = lower * ratio;
  } else {
    lower = upper = kNoWindow;
  }
}

// Index of the window of (group, internal element) in the [group][element] table of ngroups * E entries; -1 for a group
// outside [0, ngroups) or an element < 0, which get (kNoWindow, kNoWindow).
PTB_HD int64_t ww_slot(int32_t group, int32_t ngroups, int32_t elem, int64_t E) {
  return (group >= 0 && group < ngroups && elem >= 0) ? int64_t(group) * E + elem : -1;
}

}  // namespace ptb
