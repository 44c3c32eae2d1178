// Measured alternatives to the product walk kernels (DESIGN.md section 4):
// thread-per-particle TMA fetch (1), four lanes per particle (2), persistent kernel without /
// with other L2 policies (3-7, 13), binned gather without L1 (15, 17), compact layout +
// edge-function walk (20-23), packed rows with L1-allocating loads (25, 26).  All share the
// per-ray state machine of walk_core.cuh and pass the same parity tests, none is chosen by the
// engine.  NOT part of libpumitally.so: this file is only compiled into libpumitally_exp.so
// (`python -m pumiumtally_b200.build --experiments`, build flag PTB_EXPERIMENTS).
#include "../walk_kernels.hpp"

#include "../walk_persist.cuh"

namespace ptb {
namespace {

// ---------------------------------------------------------------- variant 1
// Thread per particle; each lane's record is staged into its own shared-memory
// row by one cp.async.bulk (TMA unit, bypasses L1/LSU), completion signalled
// on a per-warp mbarrier.  Rows are 144 bytes apart so the eight 16-byte reads
// of a quarter-warp hit distinct bank groups.

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) walk_bulk_kernel(const WalkParams P) {
  constexpr int WARPS = BLOCK / 32;
  __shared__ __align__(128) unsigned char rows[WARPS][32 * kRowBytes];
  __shared__ __align__(8) unsigned long long bars[WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t bar = smem_u32(&bars[warp]);
  const uint32_t row = smem_u32(&rows[warp][lane * kRowBytes]);
  if (lane == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();

  const int i = P.begin + blockIdx.x * BLOCK + threadIdx.x;
  Counters c;
  Ray r;
  r.stage = kStageDone;
  if (i < P.end) begin_particle(P, i, r, c, true);
  uint32_t parity = 0;
  for (;;) {
    // the ballot is also the point where every lane has left the previous wait,
    // so the leader may re-arm the barrier
    const unsigned act = __ballot_sync(0xffffffffu, r.stage != kStageDone);
    if (!act) break;
    if (lane == __ffs(act) - 1) mbar_expect_tx(bar, 128u * __popc(act));
    if (r.stage != kStageDone) bulk_g2s(row, P.tets + r.e, 128u, bar);
    mbar_wait(bar, parity);
    parity ^= 1u;
    if (r.stage != kStageDone) {
      double raw[16];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        asm volatile("ld.shared.v2.f64 {%0,%1}, [%2];"
                     : "=d"(raw[2 * j]), "=d"(raw[2 * j + 1])
                     : "r"(row + 16 * j));
      ExitScan sc;
      scan_record(raw, r.e, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz, sc);
      advance(P, i, r, exit_parameter(sc), sc.nbr, sc.back, c, true);
    }
  }
  flush_counters(P, c);
}

// ---------------------------------------------------------------- variant 2
// Four lanes per particle, lane f owns face f: each lane loads its 32-byte
// plane (the quad's four loads cover the record's 128-byte line exactly),
// evaluates one num/den, and the quad agrees on the exit with two shuffles.

__global__ void __launch_bounds__(256) walk_quad_kernel(const WalkParams P) {
  const int lane = threadIdx.x & 31;
  const int f = lane & 3;
  const unsigned qmask = 0xfu << (lane & ~3);
  const long long gt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long ii = (long long)P.begin + (gt >> 2);
  const int i = (int)ii;
  const bool writer = (f == 0);
  Counters c;
  Ray r;
  r.stage = kStageDone;
  if (ii < (long long)P.end) begin_particle(P, i, r, c, writer);
  while (r.stage != kStageDone) {
    double a, b, cc, d;
    load_face_256(P.tets[r.e].d + 4 * f, a, b, cc, d);
    int32_t nbf, bkf;
    face_payload(a, b, cc, d, r.e, f, nbf, bkf);
    const double nx = a, ny = b, nz = cc, pc = d;
    const double den = nx * r.ux + ny * r.uy + nz * r.uz;
    const double num = pc - (nx * r.ox + ny * r.oy + nz * r.oz);
    const bool out = den > kParallelTol * (fabs(r.ux) + fabs(r.uy) + fabs(r.uz));  // see scan_face()
    double tb = out ? num / den : __builtin_huge_val();
    int32_t nb = out ? nbf : -2;
    int32_t bk = out ? bkf : -1;
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      const double to = __shfl_xor_sync(qmask, tb, m);
      const int32_t no = __shfl_xor_sync(qmask, nb, m);
      const int32_t bo = __shfl_xor_sync(qmask, bk, m);
      // ties go to the lower face index, as in the sequential scan
      const bool take = (to < tb) || (to == tb && (lane & m));
      tb = take ? to : tb;
      nb = take ? no : nb;
      bk = take ? bo : bk;
    }
    if (!(tb < 1.0)) tb = __builtin_huge_val();
    advance(P, i, r, tb, nb, bk, c, writer);
  }
  flush_counters(P, c);
}


// ---------------------------------------------------------------- variant 27
// Two rays per lane (VERDICT r01, item 6: "settle the latency-vs-L2 question with measurements").
// The streaming kernel (variant 8) keeps 28 warps x 1 ray per SM in flight and stalls ~10 warps per
// issue slot on the long scoreboard.  Here every lane owns two independent rays; each iteration
// issues the record loads of both before either is used, so a warp has twice the loads in flight
// at the same occupancy -- if the kernel were latency-bound this would pay, if it is bound by L2
// request throughput it cannot.  Same staging (TMA bulk copies of 16-particle chunks, two stages per
// warp), same per-ray state machine, same results.
__device__ __forceinline__ void plane_load(const WalkParams &P, const Ray &r, uint64_t pol, double (&q)[3][4],
                                           double (&q3)[4]) {
  const double *rec = P.tets[r.e].d;
  const int en = r.entry;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int fk = k + ((en >= 0 && k >= en) ? 1 : 0);
    load_face<kFetchPolicy>(rec + 4 * fk, pol, q[k][0], q[k][1], q[k][2], q[k][3]);
  }
  if (en < 0) load_face<kFetchPolicy>(rec + 12, pol, q3[0], q3[1], q3[2], q3[3]);
}
__device__ __forceinline__ void plane_compute(const WalkParams &P, int my_i, Ray &r, Counters &c, const double (&q)[3][4],
                                              const double (&q3)[4]) {
  ExitScan sc;
  const int en = r.entry;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int fk = k + ((en >= 0 && k >= en) ? 1 : 0);
    int32_t nb, bk;
    face_payload(q[k][0], q[k][1], q[k][2], q[k][3], r.e, fk, nb, bk);
    scan_face(sc, q[k][0], q[k][1], q[k][2], q[k][3], nb, bk, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
  }
  if (en < 0) {
    int32_t nb, bk;
    face_payload(q3[0], q3[1], q3[2], q3[3], r.e, 3, nb, bk);
    scan_face(sc, q3[0], q3[1], q3[2], q3[3], nb, bk, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
  }
  advance(P, my_i, r, exit_parameter(sc), sc.nbr, sc.back, c, true);
}

template <int BLOCK, int MINB, int REFILL_T>
__global__ void __launch_bounds__(BLOCK, MINB) walk_tworays_kernel(const WalkParams P) {
  constexpr int WARPS = BLOCK / 32;
  __shared__ ParticleStage stages[WARPS][2];
  __shared__ __align__(8) unsigned long long bars[WARPS][2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t bar0 = smem_u32(&bars[warp][0]);
  if (lane == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();
  const uint64_t keep = l2_policy_keep(), strm = l2_policy_stream();
  const int total = P.end - P.begin;
  const int nchunks = (total + kChunk - 1) / kChunk;
  auto claim = [&]() -> int {
    int c = 0;
    if (lane == 0) c = (int)atomicAdd(P.work_counter, 1u);
    c = __shfl_sync(0xffffffffu, c, 0);
    return c < nchunks ? c : -1;
  };
  int cur = 0, cursor = 0, cur_count = 0;
  uint32_t parity = 0;
  int chunk_cur = claim();
  if (chunk_cur >= 0) stage_load_hint(P, chunk_cur, &stages[warp][0], bar0, lane, strm);
  int chunk_next = chunk_cur >= 0 ? claim() : -1;
  if (chunk_next >= 0) stage_load_hint(P, chunk_next, &stages[warp][1], bar0 + 8, lane, strm);
  if (chunk_cur >= 0) {
    mbar_wait(bar0, 0);
    parity ^= 1u;
    cur_count = min(kChunk, total - chunk_cur * kChunk);
  }
  Counters c;
  Ray r[2];
  int my_i[2] = {0, 0};
  r[0].stage = r[1].stage = kStageDone;
  for (;;) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      unsigned idle = __ballot_sync(0xffffffffu, r[k].stage == kStageDone);
      while (cur_count > 0 && (int)__popc(idle) >= REFILL_T) {
        const int slot = cursor + __popc(idle & ((1u << lane) - 1u));
        if (r[k].stage == kStageDone && slot < cur_count) {
          my_i[k] = P.begin + chunk_cur * kChunk + slot;
          begin_from_stage(P, &stages[warp][cur], slot, r[k], c);
        }
        __syncwarp();
        cursor += __popc(idle);
        if (cursor >= cur_count) {
          const int recycled = cur;
          chunk_cur = chunk_next;
          cur ^= 1;
          cursor = 0;
          cur_count = 0;
          chunk_next = -1;
          if (chunk_cur >= 0) {
            mbar_wait(bar0 + 8 * cur, (parity >> cur) & 1u);
            parity ^= 1u << cur;
            cur_count = min(kChunk, total - chunk_cur * kChunk);
            chunk_next = claim();
            if (chunk_next >= 0) {
              if (lane == 0) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
              stage_load_hint(P, chunk_next, &stages[warp][recycled], bar0 + 8 * recycled, lane, strm);
            }
          }
        }
        idle = __ballot_sync(0xffffffffu, r[k].stage == kStageDone);
      }
    }
    const bool a0 = r[0].stage != kStageDone, a1 = r[1].stage != kStageDone;
    if (!__any_sync(0xffffffffu, a0 || a1)) break;  // nothing in flight and nothing left to hand out
    double qa[3][4], qa3[4], qb[3][4], qb3[4];
    if (a0) plane_load(P, r[0], keep, qa, qa3);  // both rays' records are requested ...
    if (a1) plane_load(P, r[1], keep, qb, qb3);
    if (a0) plane_compute(P, my_i[0], r[0], c, qa, qa3);  // ... before either is used
    if (a1) plane_compute(P, my_i[1], r[1], c, qb, qb3);
  }
  flush_counters(P, c);
}

template <int BLOCK, int MINB, int REFILL_T>
cudaError_t launch_tworays(const WalkParams &p, long long n, cudaStream_t stream) {
  static int sms = 0, occ = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(walk_tworays_kernel<BLOCK, MINB, REFILL_T>, cudaFuncAttributePreferredSharedMemoryCarveout,
                         (int)cudaSharedmemCarveoutMaxShared);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, walk_tworays_kernel<BLOCK, MINB, REFILL_T>, BLOCK, 0);
    if (occ < 1) occ = 1;
  }
  const long long nchunks = (n + kChunk - 1) / kChunk;
  const long long want = (nchunks + BLOCK / 32 - 1) / (BLOCK / 32);
  const unsigned grid = (unsigned)std::min<long long>(want, (long long)sms * occ);
  cudaError_t e = cudaMemsetAsync(p.work_counter, 0, sizeof(unsigned int), stream);
  if (e != cudaSuccess) return e;
  walk_tworays_kernel<BLOCK, MINB, REFILL_T><<<grid, BLOCK, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_walk_experiment(const WalkParams &p, int variant, int block, cudaStream_t stream) {
  const long long n = (long long)p.end - p.begin;
  switch (variant) {
    case kVariantBulk: {
      const unsigned grid = (unsigned)((n + block - 1) / block);
      if (block == 64) walk_bulk_kernel<64><<<grid, 64, 0, stream>>>(p);
      else if (block == 128) walk_bulk_kernel<128><<<grid, 128, 0, stream>>>(p);
      else walk_bulk_kernel<256><<<grid, 256, 0, stream>>>(p);
      break;
    }
    case kVariantQuad: {
      const unsigned grid = (unsigned)((4 * n + block - 1) / block);
      walk_quad_kernel<<<grid, block, 0, stream>>>(p);
      break;
    }
    case kVariantPersist:
      if (block == 64) return launch_persist<64, kFetchPlain, 14>(p, n, stream);
      if (block == 256) return launch_persist<256, kFetchPlain, 3>(p, n, stream);
      return launch_persist<128, kFetchPlain, 7>(p, n, stream);
    case kVariantPersistPolicy:
      return launch_persist<128, kFetchPolicy, 7>(p, n, stream);
    case kVariantPersistPolicy128:
      return launch_persist<128, kFetchPolicy128, 7>(p, n, stream);
    case kVariantPersistBulk:
      return launch_persist<128, kFetchBulk, 5>(p, n, stream);
    case kVariantPersistPolicy128Occ8:
      return launch_persist<128, kFetchPolicy128, 8>(p, n, stream);
    case kVariantPersistGather:
      return launch_persist<128, kFetchPolicy, 7, 8, true>(p, n, stream);
    case kVariantPersistGatherPlain:
      return launch_persist<128, kFetchPlain, 7, 1, true, 40>(p, n, stream);
    case kVariantPersistRefill8Occ8:
      return launch_persist<128, kFetchPolicy, 8, 8>(p, n, stream);
    case kVariantTwoRays:
      if (p.order || p.rows) return cudaErrorInvalidValue;
      if (block == 64) return launch_tworays<128, 3, 8>(p, n, stream);   // block=64 selects 3 resident blocks
      if (block == 256) return launch_tworays<128, 5, 8>(p, n, stream);  // block=256 selects 5
      return launch_tworays<128, 4, 8>(p, n, stream);
    case kVariantLean:
      return launch_persist<128, kFetchLean, 7, 8>(p, n, stream);
    case kVariantLeanGather:
      return launch_persist<128, kFetchLeanL1, 6, 8, true, 40>(p, n, stream);
    case kVariantLeanPacked:
      if (!p.rows) return cudaErrorInvalidValue;
      return launch_persist<128, kFetchLean, 7, 8, 2>(p, n, stream);
    case kVariantPersistAggTally:
      return launch_persist<128, kFetchPolicyAgg, 7, 8>(p, n, stream);
    case kVariantGatherAggTally:
      return launch_persist<128, kFetchPolicyL1Agg, 6, 8, true, 40>(p, n, stream);
    case kVariantPersistBulkOcc7:
      return launch_persist<128, kFetchBulk, 7>(p, n, stream);
    case kVariantPackedL1:
      if (!p.rows) return cudaErrorInvalidValue;
      return launch_persist<128, kFetchPolicyL1, 7, 8, 2, 40>(p, n, stream);
    case kVariantPackedL1Occ6:
      if (!p.rows) return cudaErrorInvalidValue;
      return launch_persist<128, kFetchPolicyL1, 6, 8, 2, 40>(p, n, stream);
    case kVariantEdge:
      if (!p.links) return cudaErrorInvalidValue;
      return launch_persist<128, kFetchEdge, 4, 8, false, 40>(p, n, stream);
    case kVariantEdgeOcc5:
      if (!p.links) return cudaErrorInvalidValue;
      return launch_persist<128, kFetchEdge, 5, 8, false, 40>(p, n, stream);
    case kVariantEdgeOcc6:
      if (!p.links) return cudaErrorInvalidValue;
      return launch_persist<128, kFetchEdge, 6, 8, false, 40>(p, n, stream);
    case kVariantEdgeGather:
      if (!p.links) return cudaErrorInvalidValue;
      return launch_persist<128, kFetchEdge, 4, 8, true, 40>(p, n, stream);
    default:
      return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace ptb
