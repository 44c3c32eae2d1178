// sm_90a kernels of the point queries: locate arbitrary points in the mesh (walk_core.cuh, locate_point) and evaluate
// the normalised results there; and of the collision estimator, which scores events at located points or at the
// particles' positions into the collision region of the tally (walk_core.cuh, collision_event).  Thread per point or
// event; nothing here writes the particle state, the track-length tally or the statistics.
#include <cmath>

#include "fetch_record.cuh"
#include "walk_kernels.hpp"

namespace ptb {
namespace {

// internal[i]: the internal element id of point i (for the evaluation kernel), out[i]: the caller's element id; either
// may be nullptr.
__global__ void __launch_bounds__(256) locate_kernel(const LocateParams P, const double *__restrict__ xyz, int64_t n,
                                                     int32_t *__restrict__ internal,
                                                     int32_t *__restrict__ out, const int32_t *__restrict__ orig_of_internal) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
  const int32_t e = locate_point(P, x, y, z, [&](int32_t t, double (&r)[16]) { fetch_record(P.tets, t, r); });
  if (internal) internal[i] = e;
  if (out) out[i] = e >= 0 ? __ldg(orig_of_internal + e) : -1;
}

// out[r * pitch + i] = vals[r * E + e] (+ grads[r * E + e] . (x - cen[e]) with moments) for the R results of the
// element e = internal[i] that contains point i; NaN where e < 0.
__global__ void __launch_bounds__(256) evaluate_kernel(const double *__restrict__ xyz, const int32_t *__restrict__ internal,
                                                       int64_t n, const double *__restrict__ vals,
                                                       const double *__restrict__ grads, const double *__restrict__ cen,
                                                       int64_t E, int32_t R, double *__restrict__ out, int64_t pitch) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t e = internal[i];
  if (e < 0) {
    for (int32_t r = 0; r < R; ++r) out[r * pitch + i] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  double dx = 0.0, dy = 0.0, dz = 0.0;
  if (grads) {
    dx = xyz[3 * i] - __ldg(cen + 3 * (int64_t)e);
    dy = xyz[3 * i + 1] - __ldg(cen + 3 * (int64_t)e + 1);
    dz = xyz[3 * i + 2] - __ldg(cen + 3 * (int64_t)e + 2);
  }
  for (int32_t r = 0; r < R; ++r) {
    const int64_t j = r * E + e;
    double v = __ldg(vals + j);
    if (grads) v += __ldg(grads + 3 * j) * dx + __ldg(grads + 3 * j + 1) * dy + __ldg(grads + 3 * j + 2) * dz;
    out[r * pitch + i] = v;
  }
}

// counts[c] += the lanes of the warp whose event ended as outcome c (c < 3): one atomic per warp and counter.  Called
// by all 32 lanes; outcome -1: no event.
__device__ __forceinline__ void count_events(unsigned long long *counts, int outcome) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const unsigned m = __ballot_sync(0xffffffffu, outcome == c);
    if (m && lane == __ffs(m) - 1) atomicAdd(counts + c, (unsigned long long)__popc(m));
  }
}

// Collision events at arbitrary points: locate_point, then collision_event.  Thread per event; no early exit, the
// counters need the whole warp.
__global__ void __launch_bounds__(256) collide_located_kernel(const LocateParams L, const CollisionParams C,
                                                              const double *__restrict__ xyz, int64_t n,
                                                              const double *__restrict__ w,
                                                              const double *__restrict__ resp,
                                                              const int32_t *__restrict__ bins,
                                                              const double *__restrict__ times,
                                                              unsigned long long *__restrict__ counts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int outcome = -1;
  if (i < n) {
    const double x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
    const int32_t e = locate_point(L, x, y, z, [&](int32_t t, double (&r)[16]) { fetch_record(L.tets, t, r); });
    outcome = collision_event(C, e, x, y, z, __ldg(w + i), resp ? resp + i * C.nscores : nullptr,
                              bins ? __ldg(bins + i) : 0, C.nt > 0 ? __ldg(times + i) : 0.0);
  }
  count_events(counts, outcome);
}

// Collision events at the stored positions of the particles i with collided[i] != 0, in their parent elements.
__global__ void __launch_bounds__(256) collide_particles_kernel(const ParticleState *__restrict__ state,
                                                                const int8_t *__restrict__ collided, int32_t n,
                                                                const CollisionParams C,
                                                                const double *__restrict__ w,
                                                                const double *__restrict__ resp,
                                                                const int32_t *__restrict__ bins,
                                                                const double *__restrict__ times,
                                                                unsigned long long *__restrict__ counts) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  int outcome = -1;
  if (i < n && __ldg(collided + i) != 0) {
    const ParticleState s = load_state(state + i);
    outcome = collision_event(C, s.elem, s.x, s.y, s.z, __ldg(w + i), resp ? resp + (int64_t)i * C.nscores : nullptr,
                              bins ? __ldg(bins + i) : 0, C.nt > 0 ? __ldg(times + i) : 0.0);
  }
  count_events(counts, outcome);
}

}  // namespace

cudaError_t launch_collide_located(const LocateParams &l, const CollisionParams &c, const double *xyz, int64_t n,
                                   const double *w, const double *resp, const int32_t *bins, const double *times,
                                   unsigned long long *counts, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  collide_located_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(l, c, xyz, n, w, resp, bins, times, counts);
  return cudaGetLastError();
}

cudaError_t launch_collide_particles(const ParticleState *state, const int8_t *collided, int32_t n,
                                     const CollisionParams &c, const double *w, const double *resp, const int32_t *bins,
                                     const double *times, unsigned long long *counts, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  collide_particles_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(state, collided, n, c, w, resp, bins, times,
                                                                            counts);
  return cudaGetLastError();
}

cudaError_t launch_locate(const LocateParams &p, const double *xyz, int64_t n, int32_t *internal, int32_t *out,
                          const int32_t *orig_of_internal, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  locate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p, xyz, n, internal, out, orig_of_internal);
  return cudaGetLastError();
}

cudaError_t launch_evaluate(const double *xyz, const int32_t *internal, int64_t n, const double *vals, const double *grads,
                            const double *cen, int64_t E, int32_t R, double *out, int64_t pitch, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  evaluate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(xyz, internal, n, vals, grads, cen, E, R, out, pitch);
  return cudaGetLastError();
}

}  // namespace ptb
