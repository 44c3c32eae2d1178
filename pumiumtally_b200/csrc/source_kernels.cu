// sm_90a kernel of the mesh source (source_sample.cuh; engine.cu, sample_source): one thread per sample, grid-stride
// over 64-bit sample indices.  Each sample searches the CDF, gathers its element's four vertices and stores what the
// caller asked for; with placement it also stores the particle's position and parent element, without a walk.
#include <cstdint>

#include "source_sample.cuh"
#include "walk_kernels.hpp"

namespace ptb {
namespace {

// Sample first + j for j < n.  Outputs may be nullptr; state != nullptr places sample j as particle j.
__global__ void __launch_bounds__(256) source_sample_kernel(const SourceTable S, uint64_t seed, uint64_t first,
                                                            int64_t n, double *__restrict__ xyz,
                                                            int32_t *__restrict__ elem, int32_t *__restrict__ group,
                                                            double *__restrict__ weight,
                                                            ParticleState *__restrict__ state,
                                                            const int32_t *__restrict__ internal_of_orig) {
  const int64_t step = int64_t(gridDim.x) * blockDim.x;
  for (int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < n; j += step) {
    int64_t k;
    double p[3], w;
    source_sample(S, seed, first + uint64_t(j), k, p, w);
    const int64_t g = k / S.E, e = k - g * S.E;
    if (xyz) {
      xyz[3 * j] = p[0];
      xyz[3 * j + 1] = p[1];
      xyz[3 * j + 2] = p[2];
    }
    if (elem) elem[j] = int32_t(e);
    if (group) group[j] = int32_t(g);
    if (weight) weight[j] = w;
    if (state) store_state(state + j, p[0], p[1], p[2], __ldg(internal_of_orig + e));
  }
}

}  // namespace

cudaError_t launch_source_sample(const SourceTable &S, uint64_t seed, uint64_t first, int64_t n, double *xyz,
                                 int32_t *elem, int32_t *group, double *weight, ParticleState *state,
                                 const int32_t *internal_of_orig, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int block = 256;
  const int64_t want = (n + block - 1) / block, cap = int64_t(sms) * 8;  // 2048 threads per SM
  source_sample_kernel<<<unsigned(want < cap ? want : cap), block, 0, stream>>>(S, seed, first, n, xyz, elem, group,
                                                                               weight, state, internal_of_orig);
  return cudaGetLastError();
}

}  // namespace ptb
