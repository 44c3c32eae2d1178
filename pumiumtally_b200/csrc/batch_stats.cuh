// Batch statistics of the tally results (engine.cu, end_batch; stats_kernels.cu): a running mean and sum of squared
// deviations per result, folded one batch at a time by Welford's update.  Sum and sum of squares would cost the same
// memory traffic, but S2 - S1^2 / B cancels catastrophically when the relative error is small; Welford does not.
//
// __host__ __device__ so that tests/ can compile the same arithmetic with g++ (tests/host_emul/emul_batch_stats.cpp).
#pragma once
#include "walk_core.cuh"

#if !defined(__CUDACC__)
#include <cmath>
#endif

namespace ptb {

// Folds batch value x into (mean, m2) of the batches before it; nb is the number of batches including this one.
PTB_HD void welford_fold(double x, double nb, double &mean, double &m2) {
  const double d = x - mean;
  mean += d / nb;
  m2 += d * (x - mean);
}

// Standard error of the mean of nb >= 2 batches: sqrt(m2 / (nb (nb - 1))).
PTB_HD double batch_std_err(double m2, double nb) { return sqrt(m2 / (nb * (nb - 1.0))); }

// Relative error: std_err / |mean|, 0 where the mean is 0.
PTB_HD double batch_rel_err(double mean, double std_err) { return mean != 0.0 ? std_err / fabs(mean) : 0.0; }

// What pumitally_get_batch_results returns for one result of an element of volume `volume`: kind 0 the mean, 1 its
// standard error (both divided by the volume), 2 the relative error.
PTB_HD double batch_readout(double mean, double m2, double nb, double volume, int kind) {
  const double m = mean / volume;
  if (kind == 0) return m;
  const double s = batch_std_err(m2, nb) / volume;
  return kind == 1 ? s : batch_rel_err(m, s);
}

}  // namespace ptb
