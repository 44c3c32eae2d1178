// TEST-ONLY C wrappers of the batch-statistics launchers of libpumitally.so (stats_kernels.cu, ww_kernels.cu), so that
// tests/test_gpu_stats_kernels.py can call each kernel on raw device pointers it chose itself (rank shares, odd
// offsets, lengths the engine never produces on one GPU).  Not part of the library and not a C ABI of the project.
#include <cstdint>
#include <cstring>
#include <vector>

#include "batch_stats.cuh"
#include "walk_kernels.hpp"

namespace {

constexpr int64_t kScratchCanaries = 64;  // doubles after the region-sum scratch
constexpr uint64_t kCanary = 0x7ff5a5a5c3c3e1e1ull;  // a signalling NaN: a sum that read it would show
constexpr uint64_t kScratchFill = 0x7ff8dead0000beefull;  // scratch the kernels must write before they read it

}  // namespace

extern "C" {

int ptb_test_batch_fold(const double *x, double *mean, double *m2, int64_t n, const double *divisor, double nb,
                        void *stream) {
  return int(ptb::launch_batch_fold(x, mean, m2, n, divisor, nb, static_cast<cudaStream_t>(stream)));
}

int ptb_test_batch_merge(const double *mean_b, const double *m2_b, double *mean, double *m2, int64_t n, double na,
                         double nb, void *stream) {
  return int(ptb::launch_batch_merge(mean_b, m2_b, mean, m2, n, na, nb, static_cast<cudaStream_t>(stream)));
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

// The region sums of region_of_internal[E] (values in [-1, nregions)) over the m0 slots [0, nscores) of narrays
// arrays [E][stride] at src + a * pitch, into out[(a * nregions + g) * nscores + k], through the product's plan
// (build_region_plan) and launcher.  The scratch is sized by region_scratch_len, filled with NaN and followed by
// canaries.  Returns the CUDA error, or -1 when a canary after the scratch changed; *nlevels gets the plan's levels.
int ptb_test_region_sums(const int32_t *region_of_internal, int64_t E, int32_t nregions, int32_t nscores,
                         int32_t stride, int64_t narrays, int64_t pitch, const double *src, double *out, int *nlevels,
                         void *stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const ptb::RegionPlan p = ptb::build_region_plan(region_of_internal, E, nregions);
  *nlevels = int(p.levels.size());
  const int64_t scratch_len = ptb::region_scratch_len(p, narrays, nscores);
  std::vector<uint64_t> host(size_t(scratch_len + kScratchCanaries), kScratchFill);
  for (int64_t i = scratch_len; i < scratch_len + kScratchCanaries; ++i) host[size_t(i)] = kCanary;
  int32_t *d_elems = nullptr, *d_starts = nullptr;
  double *d_scratch = nullptr;
  cudaError_t e = cudaMalloc(&d_elems, (p.elems.size() + 1) * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&d_starts, p.starts.size() * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&d_scratch, host.size() * sizeof(double));
  if (e == cudaSuccess)
    e = cudaMemcpy(d_elems, p.elems.data(), p.elems.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = cudaMemcpy(d_starts, p.starts.data(), p.starts.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_scratch, host.data(), host.size() * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = ptb::launch_region_sums(src, pitch, stride, nscores, narrays, d_elems, d_starts, p.levels.data(),
                                int(p.levels.size()), d_scratch, scratch_len, out, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  std::vector<uint64_t> back(host.size());
  if (e == cudaSuccess) e = cudaMemcpy(back.data(), d_scratch, back.size() * sizeof(double), cudaMemcpyDeviceToHost);
  cudaFree(d_elems);
  cudaFree(d_starts);
  cudaFree(d_scratch);
  if (e != cudaSuccess) return int(e);
  return std::memcmp(back.data() + scratch_len, host.data() + scratch_len, kScratchCanaries * sizeof(double)) ? -1 : 0;
}

int ptb_test_ww_generate(const double *mean, const double *m2, const double *volume, int64_t E, int32_t ngroups,
                         int64_t pitch, int32_t stride, double nb, double max_rel_err, double c, double ratio,
                         unsigned long long *red, double *table, void *stream) {
  return int(ptb::launch_ww_generate(mean, m2, volume, E, ngroups, pitch, stride, nb, max_rel_err, c, ratio, red,
                                     reinterpret_cast<double2 *>(table), static_cast<cudaStream_t>(stream)));
}

int ptb_test_leakage(const double *cur, int64_t E, int32_t R, const uint32_t *hull, int64_t nhull, double *out,
                     void *stream) {
  return int(ptb::launch_leakage(cur, E, R, hull, nhull, out, static_cast<cudaStream_t>(stream)));
}

}  // extern "C"
