// sm_90a kernels of the point detectors (walk_core.cuh, detector_event / detector_ray): one thread per (event, detector)
// ray, detector-major (q = d * n + i), so that the lanes of a warp walk toward the same point and share its records.
// Nothing here writes the particle state, the tally in d_flux_ or the statistics.
//
// Every ray of a call adds to one of ntime * nbins * nscores * D slots, so the scores are aggregated within the block
// before they reach global memory: into a shared-memory copy of the slots when they fit (kDetSmemSlots), flushed with one
// reduction per nonzero slot; otherwise per warp, the lanes of one slot found with match.any and summed with shuffles.
#include <cmath>

#include "fetch_record.cuh"
#include "walk_kernels.hpp"

namespace ptb {
namespace {

constexpr int kDetBlock = 256;
// The void kernels take ~140 registers (the entry search on top of the walk): blocks of 128 let three share an SM (12
// warps) where one block of 256 would fit (8 warps).
constexpr int kDetVoidBlock = 128;

// counts[c] += the lanes of the warp with ray outcome c, counts[kDetCountCrossings] += crossings; the event outcomes
// (outside, rejected) only from the lanes with ev set (one ray per event).  Called by all 32
// lanes; outcome -1: no ray.  Layout of counts: kDetCount* in walk_kernels.hpp.
__device__ __forceinline__ void count_rays(unsigned long long *counts, int outcome, bool ev, uint32_t crossings) {
  const int lane = threadIdx.x & 31;
  const bool hit[6] = {outcome == kRayTraced, outcome == kRayShadowed, outcome == kRayLost, outcome == kRayInsideR0,
                       outcome == kDetOutside && ev,
                       outcome == kDetRejected && ev};
  const int slot[6] = {kDetCountTraced, kDetCountShadowed, kDetCountLost, kDetCountInsideR0, kDetCountOutside,
                       kDetCountRejected};
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    const unsigned m = __ballot_sync(0xffffffffu, hit[c]);
    if (m && lane == __ffs(m) - 1) atomicAdd(counts + slot[c], (unsigned long long)__popc(m));
  }
  const unsigned x = __reduce_add_sync(0xffffffffu, crossings);
  if (x && lane == 0) atomicAdd(counts + kDetCountCrossings, (unsigned long long)x);
}

// counts[kDetCountHullEntries] += the entries of the warp's rays into the mesh through the hull (the detector void).
// Called by all 32 lanes.
__device__ __forceinline__ void count_entries(unsigned long long *counts, uint32_t entries) {
  const unsigned x = __reduce_add_sync(0xffffffffu, entries);
  if (x && (threadIdx.x & 31) == 0) atomicAdd(counts + kDetCountHullEntries, (unsigned long long)x);
}

// The scores val[0..nscores) of this lane's ray at slot + k D (on: the ray scored), added to the tally.  SMEM: into the
// block's shared copy acc of the slots; otherwise the warp's lanes of one slot are summed and one of them adds the sum.
// Called by all 32 lanes.
template <bool SMEM>
__device__ __forceinline__ void add_scores(const DetectorParams &P, double *acc, const double *val, int64_t slot,
                                           bool on) {
  if constexpr (SMEM) {
    if (on) {
#pragma unroll
      for (int k = 0; k < kMaxScores; ++k)
        if (k < P.nscores && val[k] != 0.0) atomicAdd(acc + slot + (int64_t)k * P.ndet, val[k]);
    }
  } else {
    const int lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(0xffffffffu, on ? slot : -1 - (int64_t)lane);
    const int leader = __ffs(peers) - 1;
#pragma unroll
    for (int k = 0; k < kMaxScores; ++k) {
      if (k >= P.nscores) break;
      double sum = 0.0;
      unsigned m = peers;
      while (__any_sync(0xffffffffu, m != 0)) {
        const int src = m ? __ffs(m) - 1 : lane;
        const double x = __shfl_sync(0xffffffffu, val[k], src);
        if (m) { sum += x; m &= m - 1; }
      }
      if (on && lane == leader && sum != 0.0) PTB_TALLY_ADD(P.tally + slot + (int64_t)k * P.ndet, sum);
    }
  }
}

// SMEM: the shared copy of the slots is zeroed before the rays and flushed after them.
template <bool SMEM>
__device__ __forceinline__ void zero_slots(double *acc, int64_t nslots) {
  if constexpr (SMEM) {
    for (int64_t s = threadIdx.x; s < nslots; s += blockDim.x) acc[s] = 0.0;
    __syncthreads();
  }
}
template <bool SMEM>
__device__ __forceinline__ void flush_slots(const DetectorParams &P, const double *acc, int64_t nslots) {
  if constexpr (SMEM) {
    __syncthreads();
    for (int64_t s = threadIdx.x; s < nslots; s += blockDim.x)
      if (acc[s] != 0.0) PTB_TALLY_ADD(P.tally + s, acc[s]);
  }
}

// Rays of events at arbitrary points: locate_point, then detector_event.  n events, D = P.ndet detectors, q < D n.
// No early exit: the counters, the warp aggregation and the block flush need every thread.
template <bool SMEM>
__global__ void __launch_bounds__(kDetBlock) detect_located_kernel(
    const LocateParams L, const DetectorParams P, const double *__restrict__ xyz, int64_t n,
    const double *__restrict__ w, const double *__restrict__ pdf, const double *__restrict__ resp,
    const int32_t *__restrict__ bins, const double *__restrict__ times, const double *__restrict__ speeds,
    unsigned long long *__restrict__ counts) {
  extern __shared__ double acc[];
  const int64_t nslots = int64_t(P.nt > 0 ? P.nt : 1) * P.nbins * P.nscores * P.ndet;
  zero_slots<SMEM>(acc, nslots);
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int outcome = -1;
  bool ev = false;
  uint32_t crossings = 0;
  double val[kMaxScores] = {};
  int64_t slot = 0;
  if (q < n * P.ndet) {
    const int d = int(q / n);
    const int64_t i = q - (int64_t)d * n;
    ev = d == 0;
    auto fetch = [&](int32_t t, double (&r)[16]) { fetch_record(L.tets, t, r); };
    const double x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
    const int32_t e = locate_point(L, x, y, z, fetch);
    const bool timed = P.nt > 0;
    outcome = detector_event(L, P, d, e, x, y, z, __ldg(w + i), resp ? resp + i * P.nscores : nullptr,
                             bins ? __ldg(bins + i) : 0, timed ? __ldg(times + i) : 0.0, timed ? __ldg(speeds + i) : 1.0,
                             pdf ? pdf + i * P.ndet : nullptr, val, &slot, crossings, fetch);
  }
  add_scores<SMEM>(P, acc, val, slot, outcome == kRayTraced || outcome == kRayInsideR0);
  count_rays(counts, outcome, ev, crossings);
  flush_slots<SMEM>(P, acc, nslots);
}

// Rays of events at the stored positions of the particles i < n with flagged[i] != 0, in their parent elements.
template <bool SMEM>
__global__ void __launch_bounds__(kDetBlock) detect_particles_kernel(
    const WalkParams W, const DetectorParams P, const ParticleState *__restrict__ state,
    const int8_t *__restrict__ flagged, int32_t n, const double *__restrict__ w, const double *__restrict__ pdf,
    const double *__restrict__ resp, const int32_t *__restrict__ bins, const double *__restrict__ times,
    const double *__restrict__ speeds, unsigned long long *__restrict__ counts) {
  extern __shared__ double acc[];
  const int64_t nslots = int64_t(P.nt > 0 ? P.nt : 1) * P.nbins * P.nscores * P.ndet;
  zero_slots<SMEM>(acc, nslots);
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int outcome = -1;
  bool ev = false;
  uint32_t crossings = 0;
  double val[kMaxScores] = {};
  int64_t slot = 0;
  if (q < (int64_t)n * P.ndet) {
    const int d = int(q / n);
    const int32_t i = int32_t(q - (int64_t)d * n);
    if (__ldg(flagged + i) != 0) {
      ev = d == 0;
      auto fetch = [&](int32_t t, double (&r)[16]) { fetch_record(W.tets, t, r); };
      const ParticleState s = load_state(state + i);
      const bool timed = P.nt > 0;
      outcome = detector_event(W, P, d, s.elem, s.x, s.y, s.z, __ldg(w + i),
                               resp ? resp + (int64_t)i * P.nscores : nullptr, bins ? __ldg(bins + i) : 0,
                               timed ? __ldg(times + i) : 0.0, timed ? __ldg(speeds + i) : 1.0,
                               pdf ? pdf + (int64_t)i * P.ndet : nullptr, val, &slot, crossings, fetch);
    }
  }
  add_scores<SMEM>(P, acc, val, slot, outcome == kRayTraced || outcome == kRayInsideR0);
  count_rays(counts, outcome, ev, crossings);
  flush_slots<SMEM>(P, acc, nslots);
}

// The detector void's twins of the two kernels above (walk_core.cuh, detector_ray<true>): H is the hull grid, and the
// hull entries are counted as the crossings are.  The kernels above are kept as they are, so that their code does not
// change with the mode's.
template <bool SMEM>
__global__ void __launch_bounds__(kDetVoidBlock, 3) detect_located_void_kernel(
    const LocateParams L, const DetectorParams P, const double *__restrict__ xyz, int64_t n,
    const double *__restrict__ w, const double *__restrict__ pdf, const double *__restrict__ resp,
    const int32_t *__restrict__ bins, const double *__restrict__ times, const double *__restrict__ speeds,
    unsigned long long *__restrict__ counts, const __grid_constant__ HullGrid H) {
  extern __shared__ double acc[];
  const int64_t nslots = int64_t(P.nt > 0 ? P.nt : 1) * P.nbins * P.nscores * P.ndet;
  zero_slots<SMEM>(acc, nslots);
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int outcome = -1;
  bool ev = false;
  uint32_t crossings = 0, entries = 0;
  double val[kMaxScores] = {};
  int64_t slot = 0;
  if (q < n * P.ndet) {
    const int d = int(q / n);
    const int64_t i = q - (int64_t)d * n;
    ev = d == 0;
    auto fetch = [&](int32_t t, double (&r)[16]) { fetch_record(L.tets, t, r); };
    const double x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
    const int32_t e = locate_point(L, x, y, z, fetch);
    const bool timed = P.nt > 0;
    outcome = detector_event<true>(L, P, d, e, x, y, z, __ldg(w + i), resp ? resp + i * P.nscores : nullptr,
                                   bins ? __ldg(bins + i) : 0, timed ? __ldg(times + i) : 0.0,
                                   timed ? __ldg(speeds + i) : 1.0, pdf ? pdf + i * P.ndet : nullptr, val, &slot,
                                   crossings, fetch, &H, &entries);
  }
  add_scores<SMEM>(P, acc, val, slot, outcome == kRayTraced || outcome == kRayInsideR0);
  count_rays(counts, outcome, ev, crossings);
  count_entries(counts, entries);
  flush_slots<SMEM>(P, acc, nslots);
}

template <bool SMEM>
__global__ void __launch_bounds__(kDetVoidBlock, 3) detect_particles_void_kernel(
    const WalkParams W, const DetectorParams P, const ParticleState *__restrict__ state,
    const int8_t *__restrict__ flagged, int32_t n, const double *__restrict__ w, const double *__restrict__ pdf,
    const double *__restrict__ resp, const int32_t *__restrict__ bins, const double *__restrict__ times,
    const double *__restrict__ speeds, unsigned long long *__restrict__ counts, const __grid_constant__ HullGrid H) {
  extern __shared__ double acc[];
  const int64_t nslots = int64_t(P.nt > 0 ? P.nt : 1) * P.nbins * P.nscores * P.ndet;
  zero_slots<SMEM>(acc, nslots);
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int outcome = -1;
  bool ev = false;
  uint32_t crossings = 0, entries = 0;
  double val[kMaxScores] = {};
  int64_t slot = 0;
  if (q < (int64_t)n * P.ndet) {
    const int d = int(q / n);
    const int32_t i = int32_t(q - (int64_t)d * n);
    if (__ldg(flagged + i) != 0) {
      ev = d == 0;
      auto fetch = [&](int32_t t, double (&r)[16]) { fetch_record(W.tets, t, r); };
      const ParticleState s = load_state(state + i);
      const bool timed = P.nt > 0;
      outcome = detector_event<true>(W, P, d, s.elem, s.x, s.y, s.z, __ldg(w + i),
                                     resp ? resp + (int64_t)i * P.nscores : nullptr, bins ? __ldg(bins + i) : 0,
                                     timed ? __ldg(times + i) : 0.0, timed ? __ldg(speeds + i) : 1.0,
                                     pdf ? pdf + (int64_t)i * P.ndet : nullptr, val, &slot, crossings, fetch, &H,
                                     &entries);
    }
  }
  add_scores<SMEM>(P, acc, val, slot, outcome == kRayTraced || outcome == kRayInsideR0);
  count_rays(counts, outcome, ev, crossings);
  count_entries(counts, entries);
  flush_slots<SMEM>(P, acc, nslots);
}

int64_t detector_slots(const DetectorParams &P) { return int64_t(P.nt > 0 ? P.nt : 1) * P.nbins * P.nscores * P.ndet; }

}  // namespace

cudaError_t launch_detect_located(const LocateParams &l, const DetectorParams &p, const double *xyz, int64_t n,
                                  const double *w, const double *pdf, const double *resp, const int32_t *bins,
                                  const double *times, const double *speeds, unsigned long long *counts,
                                  cudaStream_t stream, const HullGrid *hull) {
  if (n <= 0) return cudaSuccess;
  const int64_t slots = detector_slots(p);
  const unsigned blocks = (unsigned)((n * p.ndet + kDetBlock - 1) / kDetBlock);
  const bool smem = slots <= kDetSmemSlots;
  const size_t bytes = smem ? size_t(slots) * sizeof(double) : 0;
  if (hull) {
    const unsigned vb = (unsigned)((n * p.ndet + kDetVoidBlock - 1) / kDetVoidBlock);
    if (smem)
      detect_located_void_kernel<true><<<vb, kDetVoidBlock, bytes, stream>>>(l, p, xyz, n, w, pdf, resp, bins, times,
                                                                           speeds, counts, *hull);
    else
      detect_located_void_kernel<false><<<vb, kDetVoidBlock, 0, stream>>>(l, p, xyz, n, w, pdf, resp, bins, times,
                                                                        speeds, counts, *hull);
  } else if (smem) {
    detect_located_kernel<true><<<blocks, kDetBlock, bytes, stream>>>(l, p, xyz, n, w, pdf, resp, bins, times, speeds,
                                                                      counts);
  } else {
    detect_located_kernel<false><<<blocks, kDetBlock, 0, stream>>>(l, p, xyz, n, w, pdf, resp, bins, times, speeds,
                                                                   counts);
  }
  return cudaGetLastError();
}

cudaError_t launch_detect_particles(const WalkParams &wp, const DetectorParams &p, const ParticleState *state,
                                    const int8_t *flagged, int32_t n, const double *w, const double *pdf,
                                    const double *resp, const int32_t *bins, const double *times, const double *speeds,
                                    unsigned long long *counts, cudaStream_t stream, const HullGrid *hull) {
  if (n <= 0) return cudaSuccess;
  const int64_t slots = detector_slots(p);
  const unsigned blocks = (unsigned)(((int64_t)n * p.ndet + kDetBlock - 1) / kDetBlock);
  const bool smem = slots <= kDetSmemSlots;
  const size_t bytes = smem ? size_t(slots) * sizeof(double) : 0;
  if (hull) {
    const unsigned vb = (unsigned)(((int64_t)n * p.ndet + kDetVoidBlock - 1) / kDetVoidBlock);
    if (smem)
      detect_particles_void_kernel<true><<<vb, kDetVoidBlock, bytes, stream>>>(wp, p, state, flagged, n, w, pdf, resp,
                                                                             bins, times, speeds, counts, *hull);
    else
      detect_particles_void_kernel<false><<<vb, kDetVoidBlock, 0, stream>>>(wp, p, state, flagged, n, w, pdf, resp,
                                                                          bins, times, speeds, counts, *hull);
  } else if (smem) {
    detect_particles_kernel<true><<<blocks, kDetBlock, bytes, stream>>>(wp, p, state, flagged, n, w, pdf, resp, bins,
                                                                        times, speeds, counts);
  } else {
    detect_particles_kernel<false><<<blocks, kDetBlock, 0, stream>>>(wp, p, state, flagged, n, w, pdf, resp, bins,
                                                                     times, speeds, counts);
  }
  return cudaGetLastError();
}

}  // namespace ptb
