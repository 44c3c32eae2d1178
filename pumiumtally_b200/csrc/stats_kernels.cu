// Batch statistics kernels (batch_stats.cuh; engine.cu, end_batch / get_batch_results / get_batch_max_rel_err).
// All three are memory-bound flat passes over the [time][bin][element][stride] record of the reported tally.
#include <cstdint>

#include "batch_stats.cuh"
#include "walk_kernels.hpp"

namespace ptb {
namespace {

// Every double x of [0, n): (mean, m2) <- welford_fold(x / *divisor, nb).  Two doubles per thread and step when the
// three arrays are 16-byte aligned (the rank shares of a reduce-scatter may start at an odd double).
template <bool kVec>
__global__ void batch_fold_kernel(const double *__restrict__ x, double *__restrict__ mean, double *__restrict__ m2,
                                  int64_t n, const double *__restrict__ divisor, double nb) {
  const double d = *divisor;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x, t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  auto fold1 = [&](int64_t i) {
    double mu = mean[i], q = m2[i];
    welford_fold(x[i] / d, nb, mu, q);
    mean[i] = mu;
    m2[i] = q;
  };
  if (!kVec) {
    for (int64_t i = t; i < n; i += stride) fold1(i);
    return;
  }
  const int64_t pairs = n / 2;
  for (int64_t p = t; p < pairs; p += stride) {
    const double2 v = reinterpret_cast<const double2 *>(x)[p];
    double2 mu = reinterpret_cast<double2 *>(mean)[p], q = reinterpret_cast<double2 *>(m2)[p];
    welford_fold(v.x / d, nb, mu.x, q.x);
    welford_fold(v.y / d, nb, mu.y, q.y);
    reinterpret_cast<double2 *>(mean)[p] = mu;
    reinterpret_cast<double2 *>(m2)[p] = q;
  }
  if (t == 0 && (n & 1)) fold1(n - 1);
}

// Every entry i of [0, n): (mean[i], m2[i]) <- welford_merge(mean_b[i], m2_b[i], na, nb), in place.  Two doubles per
// thread and step when the four arrays are 16-byte aligned, as batch_fold_kernel.
template <bool kVec>
__global__ void batch_merge_kernel(const double *__restrict__ mean_b, const double *__restrict__ m2_b,
                                   double *__restrict__ mean, double *__restrict__ m2, int64_t n, double na, double nb) {
  const int64_t stride = int64_t(gridDim.x) * blockDim.x, t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  auto merge1 = [&](int64_t i) {
    double mu = mean[i], q = m2[i];
    welford_merge(mean_b[i], m2_b[i], na, nb, mu, q);
    mean[i] = mu;
    m2[i] = q;
  };
  if (!kVec) {
    for (int64_t i = t; i < n; i += stride) merge1(i);
    return;
  }
  const int64_t pairs = n / 2;
  for (int64_t p = t; p < pairs; p += stride) {
    const double2 mb = reinterpret_cast<const double2 *>(mean_b)[p], qb = reinterpret_cast<const double2 *>(m2_b)[p];
    double2 mu = reinterpret_cast<double2 *>(mean)[p], q = reinterpret_cast<double2 *>(m2)[p];
    welford_merge(mb.x, qb.x, na, nb, mu.x, q.x);
    welford_merge(mb.y, qb.y, na, nb, mu.y, q.y);
    reinterpret_cast<double2 *>(mean)[p] = mu;
    reinterpret_cast<double2 *>(m2)[p] = q;
  }
  if (t == 0 && (n & 1)) merge1(n - 1);
}

// out[(r * nscores + k) * E + orig[e]] = batch_readout(...) of score k of element e in result array r
__global__ void batch_readout_kernel(const double *__restrict__ mean, const double *__restrict__ m2,
                                     const double *__restrict__ volume, const int32_t *__restrict__ orig_of_internal,
                                     double *__restrict__ out, int64_t E, int32_t R, int32_t nscores, int32_t stride,
                                     double nb, int kind) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= E * R) return;
  const int64_t r = t / E, e = t - r * E;
  const double v = volume[e];
  const int32_t o = orig_of_internal[e];
  const int64_t rec = t * stride;  // (r * E + e) * stride
  for (int k = 0; k < nscores; ++k)
    out[(r * nscores + k) * E + o] = batch_readout(mean[rec + k], kind == 0 ? 0.0 : m2[rec + k], nb, v, kind);
}

// Face currents (walk_kernels.hpp, launch_current_readout): thread per (array r, internal element e), four faces each.
__global__ void current_readout_kernel(const double *__restrict__ mean, const double *__restrict__ m2,
                                       const uint32_t *__restrict__ opp, const int32_t *__restrict__ orig_of_internal,
                                       double *__restrict__ out, int64_t E, int32_t R, int direction, int kind, double nb,
                                       double div) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= E * R) return;
  const int64_t r = t / E, e = t - r * E;
  const double *mu = mean + r * E * 4, *q = m2 ? m2 + r * E * 4 : nullptr;
  double *o = out + (r * E + orig_of_internal[e]) * 4;
  for (int f = 0; f < 4; ++f) {
    const uint32_t o4 = opp[4 * e + f];
    const int64_t s = o4 == kNoFace ? -1 : int64_t(o4), own = 4 * e + f;
    // the slot that holds the current asked for: -1 for the incoming current of a hull face
    const int64_t src = direction == 0 ? (s >= 0 ? s : own) : (s >= 0 ? own : -1);
    const double x = src >= 0 ? mu[src] : 0.0;
    o[f] = kind < 0 ? x / div : batch_readout(x, (kind == 0 || src < 0) ? 0.0 : q[src], nb, 1.0, kind);
  }
}

// Leakage (walk_kernels.hpp, launch_leakage): block r sums array r's hull slots, thread k taking slots k, k + kLeakBlock,
// ... left to right, then a fixed tree over the threads.
constexpr int kLeakBlock = 256;
__global__ void __launch_bounds__(kLeakBlock) leakage_kernel(const double *__restrict__ cur, int64_t E,
                                                             const uint32_t *__restrict__ hull, int64_t nhull,
                                                             double *__restrict__ out) {
  __shared__ double part[kLeakBlock];
  const double *c = cur + int64_t(blockIdx.x) * E * 4;
  double s = 0.0;
  for (int64_t k = threadIdx.x; k < nhull; k += kLeakBlock) s += c[hull[k]];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int h = kLeakBlock / 2; h > 0; h >>= 1) {
    if (int(threadIdx.x) < h) part[threadIdx.x] += part[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = part[0];
}

// Over local entries j of [0, n), global index g = goff + j: the entries of the tally [base, base + len) that are the
// m0 slot of score `score` ((g - base) % stride == score) with a nonzero mean.  red[0] <- max of their relative errors
// (as the bits of a non-negative double), red[1] += how many there are.
__global__ void batch_max_rel_err_kernel(const double *__restrict__ mean, const double *__restrict__ m2, int64_t n,
                                         int64_t goff, int64_t base, int64_t len, int32_t stride, int32_t score,
                                         double nb, unsigned long long *red) {
  double best = 0.0;
  unsigned long long cnt = 0;
  // first local entry of the tally's score slots at or after j = 0
  int64_t g0 = goff > base ? goff : base;
  const int64_t rem = (g0 - base) % stride;
  g0 += rem <= score ? score - rem : stride - rem + score;
  const int64_t gend = (goff + n < base + len) ? goff + n : base + len;
  const int64_t step = int64_t(gridDim.x) * blockDim.x * stride;
  for (int64_t g = g0 + (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * stride; g < gend; g += step) {
    const double mu = mean[g - goff];
    if (mu != 0.0) {
      best = fmax(best, batch_rel_err(mu, batch_std_err(m2[g - goff], nb)));
      ++cnt;
    }
  }
  for (int s = 16; s > 0; s >>= 1) {
    best = fmax(best, __shfl_xor_sync(0xffffffffu, best, s));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, s);
  }
  __shared__ double wbest[32];
  __shared__ unsigned long long wcnt[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    wbest[warp] = best;
    wcnt[warp] = cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < int(blockDim.x >> 5); ++w) {
      best = fmax(best, wbest[w]);
      cnt += wcnt[w];
    }
    if (best > 0.0) atomicMax(red, (unsigned long long)__double_as_longlong(best));
    if (cnt) atomicAdd(red + 1, cnt);
  }
}

// One level of the region sums (batch_stats.cuh, chunk_sum): unit u = a * nchunks + c sums chunk c of array a, one
// lane per score (2^lane_bits >= nscores lanes per unit), into out[u * nscores + k].  Input i of array a is the record
// src + a * pitch + (idx ? idx[i] : i) * stride.  The lanes of a unit read one record together, and neighbouring units
// take neighbouring chunks, so single-element regions read neighbouring records.
__global__ void region_level_kernel(const double *__restrict__ src, const int32_t *__restrict__ idx, int64_t pitch,
                                    int32_t stride, const int32_t *__restrict__ starts, int64_t nchunks,
                                    int64_t narrays, int32_t nscores, int lane_bits, double *__restrict__ out) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x, u = t >> lane_bits;
  const int k = int(t & ((1 << lane_bits) - 1));
  if (u >= nchunks * narrays || k >= nscores) return;
  const int64_t a = u / nchunks, c = u - a * nchunks;
  const int32_t lo = __ldg(starts + c), hi = __ldg(starts + c + 1);
  const double *s = src + a * pitch + k;
  double acc[kMaxScores];
  chunk_sum(hi - lo, 1, [&](int64_t i, int) {
    const int64_t rec = idx ? int64_t(__ldg(idx + lo + i)) : lo + i;
    return __ldg(s + rec * stride);
  }, acc);
  out[u * nscores + k] = acc[0];
}

// Region currents (batch_stats.cuh, RegionCurrentPlan): thread per (array a, pair p) of the partials [a][P],
// net[a * P + p] = partial[a * P + p] - partial[a * P + rev[p]] (0 for rev[p] < 0).
__global__ void region_net_kernel(const double *__restrict__ partial, const int32_t *__restrict__ rev, int64_t P,
                                  int64_t narrays, double *__restrict__ net) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= P * narrays) return;
  const int64_t a = t / P, p = t - a * P;
  const int32_t r = __ldg(rev + p);
  net[t] = partial[t] - (r < 0 ? 0.0 : partial[a * P + r]);
}

unsigned grid_for(int64_t work, int block) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t want = (work + block - 1) / block, cap = int64_t(sms) * 8;
  return unsigned(want < 1 ? 1 : want < cap ? want : cap);
}

}  // namespace

cudaError_t launch_batch_fold(const double *x, double *mean, double *m2, int64_t n, const double *divisor, double nb,
                              cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  auto aligned16 = [](const void *q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
  const int block = 256;
  if (aligned16(x) && aligned16(mean) && aligned16(m2))
    batch_fold_kernel<true><<<grid_for((n + 1) / 2, block), block, 0, stream>>>(x, mean, m2, n, divisor, nb);
  else
    batch_fold_kernel<false><<<grid_for(n, block), block, 0, stream>>>(x, mean, m2, n, divisor, nb);
  return cudaGetLastError();
}

cudaError_t launch_batch_merge(const double *mean_b, const double *m2_b, double *mean, double *m2, int64_t n, double na,
                               double nb, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  auto aligned16 = [](const void *q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
  const int block = 256;
  if (aligned16(mean_b) && aligned16(m2_b) && aligned16(mean) && aligned16(m2))
    batch_merge_kernel<true><<<grid_for((n + 1) / 2, block), block, 0, stream>>>(mean_b, m2_b, mean, m2, n, na, nb);
  else
    batch_merge_kernel<false><<<grid_for(n, block), block, 0, stream>>>(mean_b, m2_b, mean, m2, n, na, nb);
  return cudaGetLastError();
}

cudaError_t launch_batch_readout(const double *mean, const double *m2, const double *volume,
                                 const int32_t *orig_of_internal, double *out, int64_t E, int32_t R, int32_t nscores,
                                 int32_t stride, double nb, int kind, cudaStream_t stream) {
  const int64_t n = E * int64_t(R);
  if (n <= 0) return cudaSuccess;
  batch_readout_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(mean, m2, volume, orig_of_internal, out, E, R,
                                                                     nscores, stride, nb, kind);
  return cudaGetLastError();
}

cudaError_t launch_batch_max_rel_err(const double *mean, const double *m2, int64_t n, int64_t goff, int64_t base,
                                     int64_t len, int32_t stride, int32_t score, double nb, unsigned long long *red,
                                     cudaStream_t stream) {
  cudaError_t e = cudaMemsetAsync(red, 0, 2 * sizeof(unsigned long long), stream);
  if (e != cudaSuccess || n <= 0) return e;
  const int block = 256;
  batch_max_rel_err_kernel<<<grid_for(n / stride + 1, block), block, 0, stream>>>(mean, m2, n, goff, base, len, stride,
                                                                                  score, nb, red);
  return cudaGetLastError();
}

cudaError_t launch_current_readout(const double *mean, const double *m2, const uint32_t *opp, const int32_t *orig_of_internal,
                                   double *out, int64_t E, int32_t R, int direction, int kind, double nb, double div,
                                   cudaStream_t stream) {
  const int64_t n = E * int64_t(R);
  if (n <= 0) return cudaSuccess;
  current_readout_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(mean, m2, opp, orig_of_internal, out, E, R,
                                                                       direction, kind, nb, div);
  return cudaGetLastError();
}

cudaError_t launch_leakage(const double *cur, int64_t E, int32_t R, const uint32_t *hull, int64_t nhull, double *out,
                           cudaStream_t stream) {
  if (R <= 0) return cudaSuccess;
  leakage_kernel<<<unsigned(R), kLeakBlock, 0, stream>>>(cur, E, hull, nhull, out);
  return cudaGetLastError();
}

cudaError_t launch_region_sums(const double *flux, int64_t array_len, int32_t stride, int32_t nscores, int64_t narrays,
                               const int32_t *elems, const int32_t *starts, const RegionLevel *levels, int nlevels,
                               double *scratch, int64_t scratch_len, double *out, cudaStream_t stream) {
  if (narrays <= 0 || nlevels <= 0) return cudaSuccess;
  const int block = 256;
  int lane_bits = 0;
  while ((1 << lane_bits) < nscores) ++lane_bits;
  const double *src = flux;
  for (int l = 0; l < nlevels; ++l) {
    const RegionLevel &v = levels[l];
    double *dst = l + 1 == nlevels ? out : scratch + (l & 1) * (scratch_len / 2);
    const int64_t n = (v.chunks * narrays) << lane_bits;
    region_level_kernel<<<unsigned((n + block - 1) / block), block, 0, stream>>>(
        src, l == 0 ? elems : nullptr, l == 0 ? array_len : v.inputs * nscores, l == 0 ? stride : nscores,
        starts + v.start_off, v.chunks, narrays, nscores, lane_bits, dst);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    src = dst;
  }
  return cudaSuccess;
}

cudaError_t launch_region_net(const double *partial, const int32_t *rev, int64_t P, int64_t narrays, double *net,
                              cudaStream_t stream) {
  const int64_t n = P * narrays;
  if (n <= 0) return cudaSuccess;
  region_net_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(partial, rev, P, narrays, net);
  return cudaGetLastError();
}

}  // namespace ptb
