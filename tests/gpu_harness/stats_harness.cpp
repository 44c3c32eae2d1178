// TEST-ONLY C wrappers of the batch-statistics launchers of libpumitally.so (stats_kernels.cu), so that
// tests/test_gpu_stats_kernels.py can call each kernel on raw device pointers it chose itself (rank shares, odd
// offsets, lengths the engine never produces on one GPU).  Not part of the library and not a C ABI of the project.
#include <cstdint>

#include "walk_kernels.hpp"

extern "C" {

int ptb_test_batch_fold(const double *x, double *mean, double *m2, int64_t n, const double *divisor, double nb,
                        void *stream) {
  return int(ptb::launch_batch_fold(x, mean, m2, n, divisor, nb, static_cast<cudaStream_t>(stream)));
}

int ptb_test_batch_readout(const double *mean, const double *m2, const double *volume,
                           const int32_t *orig_of_internal, double *out, int64_t E, int32_t R, int32_t nscores,
                           int32_t stride, double nb, int kind, void *stream) {
  return int(ptb::launch_batch_readout(mean, m2, volume, orig_of_internal, out, E, R, nscores, stride, nb, kind,
                                       static_cast<cudaStream_t>(stream)));
}

int ptb_test_batch_max_rel_err(const double *mean, const double *m2, int64_t n, int64_t goff, int64_t base,
                               int64_t len, int32_t stride, int32_t score, double nb, unsigned long long *red,
                               void *stream) {
  return int(ptb::launch_batch_max_rel_err(mean, m2, n, goff, base, len, stride, score, nb, red,
                                           static_cast<cudaStream_t>(stream)));
}

}  // extern "C"
