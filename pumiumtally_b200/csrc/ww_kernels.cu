// sm_90a kernels of the weight windows (weight_windows.cuh; engine.cu, generate_weight_windows and the lookups): the
// MAGIC step over the batch statistics, and the lookup of the window at every particle's parent element or at located
// points.  Thread per element, particle or point; nothing here writes the particle state, the tally or the statistics.
#include <algorithm>
#include <cstdint>

#include "fetch_record.cuh"
#include "walk_kernels.hpp"
#include "weight_windows.cuh"

namespace ptb {
namespace {

// red[b] <- the largest eligible phi of group b (ww_max_candidate) as the bits of a non-negative double (0: none), for
// every group b < ngroups: blockIdx.y (and every gridDim.y-th group after it) is the group, x strides the elements.
// Group b's m0 value of element e is mean[b * pitch + e * stride] (m2 alike).  red must be zeroed.
__global__ void __launch_bounds__(256) ww_group_max_kernel(const double *__restrict__ mean, const double *__restrict__ m2,
                                                           const double *__restrict__ volume, int64_t E, int32_t ngroups,
                                                           int64_t pitch, int32_t stride, double nb, double max_rel_err,
                                                           unsigned long long *__restrict__ red) {
  __shared__ double wbest[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int32_t b = blockIdx.y; b < ngroups; b += gridDim.y) {
    const double *mu = mean + int64_t(b) * pitch, *q = m2 + int64_t(b) * pitch;
    double best = 0.0;
    for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < E; e += int64_t(gridDim.x) * blockDim.x)
      best = fmax(best, ww_max_candidate(__ldg(mu + e * stride), __ldg(q + e * stride), nb, __ldg(volume + e),
                                         max_rel_err));
    for (int s = 16; s > 0; s >>= 1) best = fmax(best, __shfl_xor_sync(0xffffffffu, best, s));
    if (lane == 0) wbest[warp] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < int(blockDim.x >> 5); ++w) best = fmax(best, wbest[w]);
      if (best > 0.0) atomicMax(red + b, (unsigned long long)__double_as_longlong(best));
    }
    __syncthreads();  // wbest is reused by the next group
  }
}

// table[b * E + e] <- ww_generate of group b's m0 value of element e, with phimax from red[b]
__global__ void __launch_bounds__(256) ww_generate_kernel(const double *__restrict__ mean, const double *__restrict__ m2,
                                                          const double *__restrict__ volume, int64_t E, int32_t ngroups,
                                                          int64_t pitch, int32_t stride, double nb, double max_rel_err,
                                                          const unsigned long long *__restrict__ red, double c,
                                                          double ratio, double2 *__restrict__ table) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= E * ngroups) return;
  const int64_t b = t / E, e = t - b * E, rec = b * pitch + e * stride;
  double lo, hi;
  ww_generate(__ldg(mean + rec), __ldg(m2 + rec), nb, __ldg(volume + e), max_rel_err,
              __longlong_as_double((long long)__ldg(red + b)), c, ratio, lo, hi);
  table[t] = make_double2(lo, hi);
}

// The window of (group, internal element): one 16-byte load, or (kNoWindow, kNoWindow) (ww_slot).
__device__ __forceinline__ double2 ww_fetch(const double2 *__restrict__ table, int32_t ngroups, int64_t E,
                                            int32_t group, int32_t elem) {
  const int64_t s = ww_slot(group, ngroups, elem, E);
  return s >= 0 ? __ldg(table + s) : make_double2(kNoWindow, kNoWindow);
}

__global__ void __launch_bounds__(256) ww_particles_kernel(const ParticleState *__restrict__ state, int32_t n,
                                                           const int32_t *__restrict__ groups,
                                                           const double2 *__restrict__ table, int32_t ngroups, int64_t E,
                                                           double *__restrict__ lower, double *__restrict__ upper) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ParticleState s = load_state(state + i);
  const double2 w = ww_fetch(table, ngroups, E, groups ? __ldg(groups + i) : 0, s.elem);
  lower[i] = w.x;
  upper[i] = w.y;
}

// locate_point exactly as locate_kernel calls it, then the window of the element
__global__ void __launch_bounds__(256) ww_points_kernel(const LocateParams P, const double *__restrict__ xyz, int64_t n,
                                                        const int32_t *__restrict__ groups,
                                                        const double2 *__restrict__ table, int32_t ngroups, int64_t E,
                                                        double *__restrict__ lower, double *__restrict__ upper) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
  const int32_t e = locate_point(P, x, y, z, [&](int32_t t, double (&r)[16]) { fetch_record(P.tets, t, r); });
  const double2 w = ww_fetch(table, ngroups, E, groups ? __ldg(groups + i) : 0, e);
  lower[i] = w.x;
  upper[i] = w.y;
}

unsigned blocks_for(int64_t work, int block) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t want = (work + block - 1) / block, cap = int64_t(sms) * 8;
  return unsigned(want < 1 ? 1 : want < cap ? want : cap);
}

}  // namespace

cudaError_t launch_ww_generate(const double *mean, const double *m2, const double *volume, int64_t E, int32_t ngroups,
                               int64_t pitch, int32_t stride, double nb, double max_rel_err, double c, double ratio,
                               unsigned long long *red, double2 *table, cudaStream_t stream) {
  if (E <= 0 || ngroups <= 0) return cudaSuccess;
  cudaError_t err = cudaMemsetAsync(red, 0, size_t(ngroups) * sizeof(unsigned long long), stream);
  if (err != cudaSuccess) return err;
  const int block = 256;
  const int64_t gy = ngroups < 65535 ? ngroups : 65535;
  // about 8 blocks per SM in all: split between the groups, at least one per group
  const unsigned gx = unsigned(std::max<int64_t>(1, blocks_for(E, block) / gy));
  ww_group_max_kernel<<<dim3(gx, unsigned(gy)), block, 0, stream>>>(mean, m2, volume, E, ngroups, pitch, stride, nb,
                                                                     max_rel_err, red);
  if ((err = cudaGetLastError()) != cudaSuccess) return err;
  const int64_t n = E * ngroups;
  ww_generate_kernel<<<unsigned((n + block - 1) / block), block, 0, stream>>>(mean, m2, volume, E, ngroups, pitch,
                                                                             stride, nb, max_rel_err, red, c, ratio,
                                                                             table);
  return cudaGetLastError();
}

cudaError_t launch_ww_particles(const ParticleState *state, int32_t n, const int32_t *groups, const double2 *table,
                                int32_t ngroups, int64_t E, double *lower, double *upper, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  ww_particles_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(state, n, groups, table, ngroups, E, lower, upper);
  return cudaGetLastError();
}

cudaError_t launch_ww_points(const LocateParams &p, const double *xyz, int64_t n, const int32_t *groups,
                             const double2 *table, int32_t ngroups, int64_t E, double *lower, double *upper,
                             cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  ww_points_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(p, xyz, n, groups, table, ngroups, E, lower, upper);
  return cudaGetLastError();
}

}  // namespace ptb
