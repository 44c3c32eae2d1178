// TEST-ONLY host build of the batch-statistics arithmetic (batch_stats.cuh: welford_fold, batch_readout), the code the
// fold and readout kernels of stats_kernels.cu run.  Compiled by g++ so that it can be checked against numpy on a
// machine without a GPU; never linked into libpumitally.so.
#include <cstdint>

#include "batch_stats.cuh"

extern "C" {
// x [B][n]: batch b's value of result i, already divided by its batch's divisor.  Folds the batches in order into
// mean[n], m2[n] (zeroed here), as end_batch does once per batch.
void ptb_fold_batches(const double *x, int64_t B, int64_t n, double *mean, double *m2) {
  for (int64_t i = 0; i < n; ++i) mean[i] = m2[i] = 0.0;
  for (int64_t b = 0; b < B; ++b)
    for (int64_t i = 0; i < n; ++i) ptb::welford_fold(x[b * n + i], double(b + 1), mean[i], m2[i]);
}

// out[i] = batch_readout(mean[i], m2[i], nb, volume[i], kind)
void ptb_readout(const double *mean, const double *m2, const double *volume, int64_t n, double nb, int32_t kind,
                 double *out) {
  for (int64_t i = 0; i < n; ++i) out[i] = ptb::batch_readout(mean[i], m2[i], nb, volume[i], kind);
}
}
