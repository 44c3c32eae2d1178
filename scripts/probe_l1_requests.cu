// Request-rate probe of the L1TEX/L2 path: what a warp-wide 128-bit L1-allocating load costs when its 32 lanes
// touch 32 lines, 4 lines (8 lanes per line) or 16 sectors of 16 lines (2 lanes per 32-byte sector).  Every pattern
// moves 512 bytes per warp instruction, so a difference in cycles per instruction is a difference in the number of
// lines (tag lookups, L2 requests) the instruction asks for, not in bytes.  Each pattern runs with a footprint
// that fits the L1 of one SM, one that fits L2 and one far larger than L2.  The load is the one the binned walk
// uses for tet records: ld.global.nc with an L2::evict_last policy, allocating in L1.
//
// Built and run by scripts/probe_l1_requests.py.  Output: one line per (pattern, footprint) with the time per launch
// (CUDA events), the SM cycles of the run (clock64, mean over blocks) and the SM cycles per warp instruction.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cuda_runtime.h>

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      std::fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));       \
      std::exit(1);                                                                        \
    }                                                                                      \
  } while (0)

constexpr int kBlock = 256;  // 8 warps
constexpr int kLoads = 8;    // independent loads in flight per lane and iteration

__device__ __forceinline__ uint32_t mix(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

// LPL: lanes per line (1: 32 lines; 8: 4 lines), or 2 lanes per sector when SECTOR (16 lines, one sector each).
// Lines are drawn at random from [0, nlines) (nlines a power of two); per_block: each block keeps to its own
// window of nlines lines (the L1 case), else the whole buffer is shared.
template <int LPL, bool SECTOR>
__global__ void __launch_bounds__(kBlock) probe(const double *buf, uint32_t nlines, int iters, bool per_block,
                                                long long *cycles, double *sink) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * kBlock + threadIdx.x) >> 5;
  const char *base = reinterpret_cast<const char *>(buf) + (per_block ? (size_t)blockIdx.x * nlines * 128 : 0);
  const int group = SECTOR ? lane >> 1 : lane / LPL;
  const uint32_t off = SECTOR ? 16u * (lane & 1) : 16u * (lane % LPL);
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  double acc = 0.0;
  __syncthreads();
  const long long t0 = clock64();
  for (int i = 0; i < iters; ++i) {
    double a[kLoads], b[kLoads];
#pragma unroll
    for (int k = 0; k < kLoads; ++k) {
      const uint32_t line = mix(warp * 0x9e3779b9u + (uint32_t)(i * kLoads + k) * 0x85ebca6bu + (uint32_t)group * 0xc2b2ae35u) &
                            (nlines - 1);
      const char *p = base + (size_t)line * 128 + off;
      asm volatile("ld.global.nc.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;" : "=d"(a[k]), "=d"(b[k]) : "l"(p), "l"(pol));
    }
#pragma unroll
    for (int k = 0; k < kLoads; ++k) acc += a[k] + b[k];
  }
  __syncthreads();
  const long long t1 = clock64();
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
  if (acc == 1.2345) sink[0] = acc;  // keeps the loads
}

template <int LPL, bool SECTOR>
static void run(const char *name, const char *where, const double *buf, uint32_t nlines, bool per_block, int grid,
                int iters, long long *d_cycles, double *sink, int blocks_per_sm) {
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  probe<LPL, SECTOR><<<grid, kBlock>>>(buf, nlines, iters, per_block, d_cycles, sink);  // warm-up
  CK(cudaGetLastError());
  CK(cudaEventRecord(e0));
  const int reps = 5;
  for (int r = 0; r < reps; ++r) probe<LPL, SECTOR><<<grid, kBlock>>>(buf, nlines, iters, per_block, d_cycles, sink);
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  long long *h = (long long *)std::malloc(sizeof(long long) * grid);
  CK(cudaMemcpy(h, d_cycles, sizeof(long long) * grid, cudaMemcpyDeviceToHost));
  double mean = 0.0;
  for (int b = 0; b < grid; ++b) mean += (double)h[b];
  mean /= grid;
  std::free(h);
  // warp instructions one SM issues during a block's run: its resident blocks x warps x loads
  const double per_sm = (double)blocks_per_sm * (kBlock / 32) * iters * kLoads;
  std::printf("%-22s %-5s %9.3f ms/launch %12.0f cycles  %7.2f cycles/warp-instr  %6.2f B/cycle/SM\n", name, where,
              ms / reps, mean, mean / per_sm, per_sm * 512.0 / mean);
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
}

int main() {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, probe<1, false>, kBlock, 0));
  const int grid = prop.multiProcessorCount * occ;  // one full wave: every block runs from start to end
  std::printf("device %s, %d SMs, %d blocks of %d per SM, L2 %d MB\n", prop.name, prop.multiProcessorCount, occ, kBlock,
              prop.l2CacheSize >> 20);
  const size_t dram_lines = (size_t)1 << 25;  // 4 GiB
  double *buf = nullptr, *sink = nullptr;
  long long *d_cycles = nullptr;
  CK(cudaMalloc(&buf, dram_lines * 128));
  CK(cudaMemset(buf, 0, dram_lines * 128));
  CK(cudaMalloc(&sink, sizeof(double)));
  CK(cudaMalloc(&d_cycles, sizeof(long long) * grid));
  struct Where {
    const char *name;
    uint32_t nlines;
    bool per_block;
    int iters;
  };
  // L1: each block reads its own 8 KB (so the SM's resident blocks read at most 64 KB); L2: 16 MB shared by all;
  // DRAM: 4 GB shared by all
  const Where ws[3] = {{"L1", 64, true, 2048}, {"L2", 1u << 17, false, 512}, {"DRAM", (uint32_t)dram_lines, false, 64}};
  for (const Where &w : ws) {
    run<1, false>("(a) 32 lanes 32 lines", w.name, buf, w.nlines, w.per_block, grid, w.iters, d_cycles, sink, occ);
    run<8, false>("(b) 8 lanes/line 4", w.name, buf, w.nlines, w.per_block, grid, w.iters, d_cycles, sink, occ);
    run<2, true>("(c) 2 lanes/sector", w.name, buf, w.nlines, w.per_block, grid, w.iters, d_cycles, sink, occ);
  }
  CK(cudaFree(buf));
  CK(cudaFree(sink));
  CK(cudaFree(d_cycles));
  return 0;
}
