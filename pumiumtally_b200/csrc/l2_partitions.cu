// Which SMs share an L2 partition?  (On a GPU whose L2 partitions each cache what their own SMs read, a line held
// only by the far partition costs a longer trip; on an H100 this probe finds no two groups.)  One SM reads a set of
// disjoint regions; then every SM chases a pointer chain through "its" region for the first time: SMs of the
// warming SM's partition see L2-hit latency, the others pay the trip to the other partition.  The engine
// uses the map to give each partition its own end of a sorted particle sequence
// (walk_persist.cuh, "die split"); when the result is not clearly two groups the split stays off.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include <cuda_runtime.h>

#include "walk_kernels.hpp"

namespace ptb {
namespace {

constexpr int kLines = 1024;                          // 128-byte lines per region
constexpr size_t kRegionWords = size_t(kLines) * 32;  // uint32 words per region
constexpr int kMaxSMs = 256;

__device__ __forceinline__ unsigned this_sm() {
  unsigned s;
  asm("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}

// word 0 of line i holds the index of the next line: a full-period walk over the region's lines
__global__ void probe_build_chains(uint32_t *mem, int nregions) {
  const int r = blockIdx.x;
  if (r >= nregions) return;
  uint32_t *base = mem + size_t(r) * kRegionWords;
  for (int i = threadIdx.x; i < kLines; i += blockDim.x) base[size_t(i) * 32] = (uint32_t(i) * 5u + 1u) & (kLines - 1);
}

__global__ void probe_warm(const uint32_t *mem, size_t words, unsigned warm_sm, int *claimed) {
  if (this_sm() != warm_sm) return;
  __shared__ int mine;
  if (threadIdx.x == 0) mine = atomicCAS(claimed, 0, 1) == 0;
  __syncthreads();
  if (!mine) return;
  uint32_t acc = 0;
  for (size_t w = size_t(threadIdx.x) * 8; w < words; w += size_t(blockDim.x) * 8) {  // one load per sector
    uint32_t v;
    asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(mem + w));
    acc += v;
  }
  if (acc == 0xdeadbeefu) claimed[1] = 1;
}

__global__ void probe_first_touch(const uint32_t *mem, float *lat, int *claimed, int nsms) {
  const unsigned s = this_sm();
  if (threadIdx.x || int(s) >= nsms) return;
  if (atomicCAS(claimed + 2 + s, 0, 1) != 0) return;  // one block per SM does the chase
  const uint32_t *base = mem + size_t(s) * kRegionWords;
  uint32_t i = 0;
  const long long t0 = clock64();
  for (int k = 0; k < kLines; ++k) asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(i) : "l"(base + size_t(i) * 32));
  const long long t1 = clock64();
  lat[s] = float(t1 - t0) / kLines + (i == 0xffffffffu);
}

}  // namespace

// mask bit s = partition of SM s (the partition of SM 0 is 0).  Returns 0 and fills the outputs when two clear
// groups were found in two independent runs that agree; 1 otherwise (single-partition GPU, MIG slice, noise).
int probe_l2_partitions(uint32_t mask[8], int *die0_sms, int *nsms_out, cudaStream_t stream) {
  for (int i = 0; i < 8; ++i) mask[i] = 0;
  *die0_sms = 0;
  int dev = 0, nsms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&nsms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 1;
  *nsms_out = nsms;
  if (nsms < 2 || nsms > kMaxSMs) return 1;
  int l2 = 0;
  cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev);
  const size_t words = kRegionWords * size_t(nsms), flush_bytes = std::max<size_t>(size_t(l2) * 3, size_t(64) << 20);
  uint32_t *mem = nullptr;
  float *lat = nullptr;
  int *claimed = nullptr;
  char *flush = nullptr;
  int rc = 1;
  std::vector<std::vector<int>> maps;
  if (cudaMalloc(&mem, words * 4) != cudaSuccess || cudaMalloc(&lat, size_t(nsms) * 4) != cudaSuccess ||
      cudaMalloc(&claimed, size_t(nsms + 2) * 4) != cudaSuccess || cudaMalloc(&flush, flush_bytes) != cudaSuccess)
    goto done;
  probe_build_chains<<<nsms, 256, 0, stream>>>(mem, nsms);
  for (unsigned warm_sm : {0u, unsigned(nsms) - 1u, unsigned(nsms) / 2u}) {
    cudaMemsetAsync(flush, 1, flush_bytes, stream);  // evict the regions from both partitions
    cudaMemsetAsync(claimed, 0, size_t(nsms + 2) * 4, stream);
    cudaMemsetAsync(lat, 0, size_t(nsms) * 4, stream);
    probe_warm<<<nsms * 8, 1024, 0, stream>>>(mem, words, warm_sm, claimed);
    probe_first_touch<<<nsms * 16, 32, 0, stream>>>(mem, lat, claimed, nsms);
    std::vector<float> h(size_t(nsms), 0.f);
    if (cudaMemcpyAsync(h.data(), lat, size_t(nsms) * 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess ||
        cudaStreamSynchronize(stream) != cudaSuccess)
      goto done;
    std::vector<float> s(h);
    std::sort(s.begin(), s.end());
    if (s[0] <= 0.f) goto done;  // an SM got no block: no map
    double gap = 0, cut = 0;
    for (int i = nsms / 4; i + 1 < nsms - nsms / 4; ++i)
      if (s[i + 1] - s[i] > gap) { gap = s[i + 1] - s[i]; cut = 0.5 * (s[i] + s[i + 1]); }
    if (gap < 0.2 * s[0]) goto done;  // not two groups
    std::vector<int> near(size_t(nsms), 0);
    for (int i = 0; i < nsms; ++i) near[i] = h[i] < cut;
    if (!near[warm_sm]) goto done;
    std::vector<int> m(size_t(nsms), 0);  // partition relative to SM 0
    for (int i = 0; i < nsms; ++i) m[i] = near[i] == near[0] ? 0 : 1;
    maps.push_back(m);
  }
  if (maps.size() == 3 && maps[0] == maps[1] && maps[1] == maps[2]) {
    int n0 = 0;
    for (int i = 0; i < nsms; ++i) {
      if (maps[0][i]) mask[i >> 5] |= 1u << (i & 31);
      else ++n0;
    }
    if (n0 * 5 >= nsms * 2 && n0 * 5 <= nsms * 3) {  // 40 % .. 60 %
      *die0_sms = n0;
      rc = 0;
    } else {
      for (int i = 0; i < 8; ++i) mask[i] = 0;
    }
  }
done:
  cudaGetLastError();
  cudaFree(mem);
  cudaFree(lat);
  cudaFree(claimed);
  cudaFree(flush);
  return rc;
}

}  // namespace ptb
