// Persistent-warp walk kernel (template) and its staging helpers, shared by the product
// translation unit (walk_kernels.cu: the kernels the engine actually chooses) and the
// experiments translation unit (experiments/walk_experiments.cu: measured alternatives that are
// not part of libpumitally.so).  Everything lives in an anonymous namespace: each TU gets its own
// instantiations.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <type_traits>

#include "walk_compact.cuh"
#include "walk_core.cuh"
#include "walk_kernels.hpp"

namespace ptb {
namespace {
__device__ __forceinline__ void flush_counters(const WalkParams &P, const Counters &c) {
  const unsigned segs = __reduce_add_sync(0xffffffffu, c.segs);
  const unsigned tracks = __reduce_add_sync(0xffffffffu, c.tracks);
  const unsigned relocs = __reduce_add_sync(0xffffffffu, c.relocs);
  const unsigned lost = __reduce_add_sync(0xffffffffu, c.lost);
  const unsigned fallbacks = __reduce_add_sync(0xffffffffu, c.fallbacks);
  if ((threadIdx.x & 31) == 0) {
    if (fallbacks) atomicAdd(&P.stats->fallbacks, (unsigned long long)fallbacks);
    if (segs) atomicAdd(&P.stats->segments, (unsigned long long)segs);
    if (tracks) atomicAdd(&P.stats->tracks, (unsigned long long)tracks);
    if (relocs) atomicAdd(&P.stats->relocations, (unsigned long long)relocs);
    if (lost) atomicAdd(&P.stats->lost, (unsigned long long)lost);
  }
}

// One 32-byte face sector as two 128-bit loads (the widest global access on sm_90), issued back to back.
__device__ __forceinline__ void load_face_256(const double *p, double &a, double &b, double &c,
                                              double &d) {
  asm volatile(
      "ld.global.nc.v2.f64 {%0,%1}, [%4];\n\t"
      "ld.global.nc.v2.f64 {%2,%3}, [%4+16];"
      : "=d"(a), "=d"(b), "=d"(c), "=d"(d) : "l"(p));
}

constexpr int kRowBytes = 144;

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes,
                                         uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}

// ---------------------------------------------------------------- variant 3
// Persistent warps with per-lane refill.  Track lengths are roughly geometric
// and relocation walks are ~10x longer than tally walks, so with one particle
// per thread a warp idles most of its lanes.  Here every warp owns two shared-memory stages of 32
// particles each, filled asynchronously by the TMA unit (cp.async.bulk of the
// SoA/AoS slices, completion on an mbarrier); a lane that finishes its particle
// takes the next slot of the current stage in the same loop iteration, and
// chunks of 32 particles are claimed from a global counter so long walks never
// hold back the rest of the range.

constexpr int kChunk = 16;  // particles per staged chunk (all slice sizes stay multiples of 16 bytes)
constexpr uint32_t kB8 = 8u * kChunk, kB24 = 24u * kChunk, kB32 = 32u * kChunk, kB1 = 1u * kChunk;

struct __align__(64) ParticleStage {
  double origin[3 * kChunk];
  double dest[3 * kChunk];
  ParticleState state[kChunk];
  double w[kChunk];
  int8_t fly[kChunk];
  int32_t id[kChunk];  // gather mode: particle id of each slot
};
static_assert(sizeof(ParticleStage) >= kChunk * sizeof(PackedRow) && sizeof(ParticleStage) % 32 == 0 && offsetof(ParticleStage, state) % 32 == 0 && offsetof(ParticleStage, w) % 16 == 0 && offsetof(ParticleStage, fly) % 16 == 0, "stage layout");

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

__device__ __forceinline__ void stage_load(const WalkParams &P, int chunk, ParticleStage *st,
                                           uint32_t bar, int lane) {
  const long long base = (long long)P.begin + (long long)chunk * kChunk;
  const int count = (int)min((long long)kChunk, (long long)P.end - base);
  if (count == kChunk && P.bulk_ok) {
    if (lane == 0) {
      const uint32_t bytes = kB32 + (P.origin ? kB24 : 0u) + (P.dest ? kB24 + kB8 : 0u) +
                             (P.flying ? kB1 : 0u);
      mbar_expect_tx(bar, bytes);
      bulk_g2s(smem_u32(st->state), P.state + base, kB32, bar);
      if (P.origin) bulk_g2s(smem_u32(st->origin), P.origin + 3 * base, kB24, bar);
      if (P.dest) {
        bulk_g2s(smem_u32(st->dest), P.dest + 3 * base, kB24, bar);
        bulk_g2s(smem_u32(st->w), P.weights + base, kB8, bar);
      }
      if (P.flying) bulk_g2s(smem_u32(st->fly), P.flying + base, kB1, bar);
    }
  } else {
    // ragged last chunk, or caller pointers that are not 16-byte aligned
    if (lane < count) {
      const long long i = base + lane;
      st->state[lane] = load_state(P.state + i);
      if (P.origin)
        for (int k = 0; k < 3; ++k) st->origin[3 * lane + k] = P.origin[3 * i + k];
      if (P.dest) {
        for (int k = 0; k < 3; ++k) st->dest[3 * lane + k] = P.dest[3 * i + k];
        st->w[lane] = P.weights[i];
      }
      if (P.flying) st->fly[lane] = P.flying[i];
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar);
  }
}

// begin_particle() reading the staged copy instead of global memory (i: the slot's particle index)
template <int NS = 0, bool TM = false, bool MO = false, bool CU = false, bool MU = false>
__device__ __forceinline__ void begin_from_stage(const WalkParams &P, const ParticleStage *st, int s,
                                                 Ray &r, Counters &c, int i = 0, const ScoreLane *sl = nullptr) {
  r.stage = kStageDone;
  const bool fly = P.flying ? (st->fly[s] == 1) : true;
  if (!fly) return;
  const double x = st->state[s].x, y = st->state[s].y, z = st->state[s].z;
  r.e = st->state[s].elem;
  if (P.origin) {
    const double tx = st->origin[3 * s], ty = st->origin[3 * s + 1], tz = st->origin[3 * s + 2];
    if (tx != x || ty != y || tz != z) {
      if (!all_finite(tx, ty, tz)) {  // unusable origin: the particle sits this move out
        c.lost++;
        return;
      }
      start_reloc(P, r, x, y, z, tx, ty, tz);
      return;
    }
  }
  if (P.dest)
    start_tally_to<NS, TM, MO, CU, MU>(P, r, x, y, z, st->dest[3 * s], st->dest[3 * s + 1], st->dest[3 * s + 2], st->w[s], c,
                                       true, i, sl);
}

// begin_particle() for a packed row (only flying particles have rows).  Returns the particle id.
template <int NS = 0, bool TM = false, bool MO = false, bool CU = false, bool MU = false>
__device__ __forceinline__ int begin_from_row(const WalkParams &P, const PackedRow *row, Ray &r, Counters &c,
                                              const ScoreLane *sl = nullptr) {
  const int id = row->id;
  const uint32_t el = row->elem;
  const double ox = row->ox, oy = row->oy, oz = row->oz;
  if (el >> 31) {  // re-sourced: phase 1 from the stored position (rare)
    if (!all_finite(ox, oy, oz)) {  // unusable origin: the particle sits this move out
      c.lost++;
      return id;
    }
    const ParticleState s0 = load_state(P.state + id);
    r.e = s0.elem;
    start_reloc(P, r, s0.x, s0.y, s0.z, ox, oy, oz);
    return id;
  }
  r.e = (int32_t)(el & kIdMask);
  start_tally_to<NS, TM, MO, CU, MU>(P, r, ox, oy, oz, row->dx, row->dy, row->dz, row->w, c, true, id, sl);
  return id;
}

// Fetch modes of the persistent kernel (how a lane gets its 128-byte tet record):
//   0  four plain 32-byte sector loads (two 128-bit loads each)
//   1  as 0, tet loads carry an L2 evict_last policy and skip L1; the particle stream
//      (staging copies, state stores) is evict_first -- keeps the tet table L2-resident
//   2  as 1, plus the L2::128B prefetch size (first sector miss pulls the whole line)
//   3  one cp.async.bulk of 128 B per lane into a shared-memory row (policies as 1)
//   (4 was a cooperative quad-load + shared-memory transpose: slower, removed)
//   5  cooperative line fetch (coop_plane_step): the warp copies the records of its active lanes into
//      per-warp shared-memory rows, eight lanes per record, so one 128-bit load touches 4 lines instead of 32;
//      L1-allocating, evict_last in L2 (the binned kernel, variant 16)
//   11 as 1 but the tet loads allocate in L1, each lane fetching its own record
//   6  compact layout + edge-function exit test (walk_compact.cuh): one 32-byte TetLinks sector and
//      one 32-byte vertex per crossing, both L2-resident; degenerate rays finish on the plane records
//   7, 8  as 1 and 11 with the warp-aggregated tally of walk_core.cuh (experiment)
//   9, 10 as 1 and 11 with the lean crossing step (plane_step_lean: the three record loads issued as one
//         block, payload decoded once, ray target re-read at the end of the ray instead of held in registers)
enum : int { kFetchPlain = 0, kFetchPolicy = 1, kFetchPolicy128 = 2, kFetchBulk = 3, kFetchCoopL1 = 5, kFetchEdge = 6,
             kFetchPolicyAgg = 7, kFetchPolicyL1Agg = 8, kFetchLean = 9, kFetchLeanL1 = 10, kFetchPolicyL1 = 11 };

__device__ __forceinline__ uint64_t l2_policy_keep() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_stream() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// same values, created where they are used (volatile: not hoisted out of the loop): keeps the
// policies out of the registers that stay live across the crossing loop of the persistent kernel
__device__ __forceinline__ uint64_t l2_policy_keep_now() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_stream_now() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst, const void *src, uint32_t bytes,
                                              uint32_t bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], "
      "%2, [%3], %4;" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar), "l"(pol)
      : "memory");
}
template <int FETCH>
__device__ __forceinline__ void load_face(const double *p, uint64_t pol, double &a, double &b,
                                          double &c, double &d) {
  if constexpr (FETCH == kFetchPolicy || FETCH == kFetchPolicyAgg)
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%4], %5;\n\t"
                 "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%2,%3}, [%4+16], %5;"
        : "=d"(a), "=d"(b), "=d"(c), "=d"(d) : "l"(p), "l"(pol));
  else if constexpr (FETCH == kFetchPolicyL1 || FETCH == kFetchPolicyL1Agg)
    asm volatile("ld.global.nc.L2::cache_hint.v2.f64 {%0,%1}, [%4], %5;\n\t"
                 "ld.global.nc.L2::cache_hint.v2.f64 {%2,%3}, [%4+16], %5;"
        : "=d"(a), "=d"(b), "=d"(c), "=d"(d) : "l"(p), "l"(pol));
  else if constexpr (FETCH == kFetchPolicy128)
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.L2::128B.v2.f64 {%0,%1}, [%4], %5;\n\t"
                 "ld.global.nc.L1::no_allocate.L2::cache_hint.L2::128B.v2.f64 {%2,%3}, [%4+16], %5;"
        : "=d"(a), "=d"(b), "=d"(c), "=d"(d) : "l"(p), "l"(pol));
  else
    load_face_256(p, a, b, c, d);
}

// stage_load() with an L2 policy on the streamed particle data
__device__ __forceinline__ void stage_load_hint(const WalkParams &P, int chunk, ParticleStage *st,
                                                uint32_t bar, int lane, uint64_t pol) {
  const long long base = (long long)P.begin + (long long)chunk * kChunk;
  const int count = (int)min((long long)kChunk, (long long)P.end - base);
  if (count == kChunk && P.bulk_ok) {
    if (lane == 0) {
      const uint32_t bytes = kB32 + (P.origin ? kB24 : 0u) + (P.dest ? kB24 + kB8 : 0u) +
                             (P.flying ? kB1 : 0u);
      mbar_expect_tx(bar, bytes);
      bulk_g2s_hint(smem_u32(st->state), P.state + base, kB32, bar, pol);
      if (P.origin) bulk_g2s_hint(smem_u32(st->origin), P.origin + 3 * base, kB24, bar, pol);
      if (P.dest) {
        bulk_g2s_hint(smem_u32(st->dest), P.dest + 3 * base, kB24, bar, pol);
        bulk_g2s_hint(smem_u32(st->w), P.weights + base, kB8, bar, pol);
      }
      if (P.flying) bulk_g2s_hint(smem_u32(st->fly), P.flying + base, kB1, bar, pol);
    }
  } else {
    stage_load(P, chunk, st, bar, lane);  // ragged / unaligned: plain path
  }
}

// ---- gather mode: the chunk's particles are not contiguous (order[] comes from the binning
// pass); every lane pulls its particle's fields with 8/4-byte cp.async copies that complete on
// the stage's mbarrier (cp.async.mbarrier.arrive.noinc: one arrival per lane, barrier count 32)
// (the gathered particle data is used once: evict_first keeps it from displacing tet records in L2)
__device__ __forceinline__ void cp_async_8(uint32_t dst, const void *src, uint64_t pol) {
  asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void *src, uint64_t pol) {
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// The ticket ids of gather mode: 4-byte copies committed as one group per ticket and waited for with
// cp_async_wait_ids() when the ticket becomes current (the stage copies complete on their mbarriers instead).
__device__ __forceinline__ void cp_async_4(uint32_t dst, const void *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_ids() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
// `id` = this lane's particle for the chunk (lanes >= count hold garbage and copy nothing)
__device__ __forceinline__ void stage_gather(const WalkParams &P, int id, int count, ParticleStage *st,
                                             uint32_t bar, int lane, uint64_t pol) {
  if (lane < count) {
    const int i = id;
    st->id[lane] = i;
    cp_async_16(smem_u32(&st->state[lane]), P.state + i, pol);
    cp_async_16(smem_u32(&st->state[lane]) + 16u, reinterpret_cast<const char *>(P.state + i) + 16, pol);
    if (P.origin) {
#pragma unroll
      for (int k = 0; k < 3; ++k)
        cp_async_8(smem_u32(&st->origin[3 * lane + k]), P.origin + 3 * (size_t)i + k, pol);
    }
    if (P.dest) {
#pragma unroll
      for (int k = 0; k < 3; ++k)
        cp_async_8(smem_u32(&st->dest[3 * lane + k]), P.dest + 3 * (size_t)i + k, pol);
      cp_async_8(smem_u32(&st->w[lane]), P.weights + i, pol);
    }
  }
  cp_async_arrive_noinc(bar);
}

// The ray target (Ray::tx,ty,tz) and the particle id live in the lane's shared-memory slots `tgt` and
// `id`, not in registers across the crossing loop: only end_ray() reads them.  target_in() returns the
// id and puts the target into the ray in the step that ends the ray -- the test is advance()'s own --
// and target_out() saves the target of a ray that starts in that step (phase 2 after phase 1, or
// phase 1 again from the stored position).
__device__ __forceinline__ int target_in(const WalkParams &P, Ray &r, double texit, int32_t next,
                                         const double *tgt, const int32_t *id) {
  int i = 0;
  if (!(texit < 1.0) || next < 0 || r.iters + 1 >= P.max_iters) {
    r.tx = tgt[0]; r.ty = tgt[1]; r.tz = tgt[2];
    i = *id;
  }
  return i;
}
__device__ __forceinline__ void target_out(const Ray &r, double *tgt) {
  if (r.iters == 0 && r.stage != kStageDone) {
    tgt[0] = r.tx; tgt[1] = r.ty; tgt[2] = r.tz;
  }
}

// The rest of a crossing once the record's faces are in registers: q holds the three faces other than the entry
// face, in face order (all but the fourth on a ray's first tet, r.entry < 0), q3 the fourth face of a first tet.
template <bool AGG, int NS, bool TM, bool MO, bool CU, bool MU = false>
__device__ __forceinline__ void plane_exit(const WalkParams &P, Ray &r, Counters &c, const double (&q)[3][4],
                                           const double (&q3)[4], double *tgt, const int32_t *id, const ScoreLane *sl) {
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
  const double texit = exit_parameter(sc);
  const int my_i = target_in(P, r, texit, sc.nbr, tgt, id);
  advance<false, AGG, NS, TM, MO, CU, MU>(P, my_i, r, texit, sc.nbr, sc.back, c, true, sl, sc.bden);
  target_out(r, tgt);
}

// One crossing on the plane records.  Entry-face elision: after a crossing the face the ray came
// in through is known (r.entry) and can never be the exit, so only the other three 32-byte
// sectors of the record are fetched; the first tet of a ray needs all four.  tgt, id: the lane's slots.
template <int FETCH, int NS = 0, bool TM = false, bool MO = false, bool CU = false, bool MU = false>
__device__ __forceinline__ void plane_step(const WalkParams &P, Ray &r, Counters &c, uint64_t pol, double *tgt,
                                           const int32_t *id, const ScoreLane *sl = nullptr) {
  ExitScan sc;
  const double *rec = P.tets[r.e].d;
  const int en = r.entry;
  // q3, the fourth face of a ray's first tet, is zero when it is not loaded: left undefined, it would be
  // carried round the crossing loop in registers (or on the stack) from the last first tet.
  double q[3][4], q3[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int fk = k + ((en >= 0 && k >= en) ? 1 : 0);
    load_face<FETCH>(rec + 4 * fk, pol, q[k][0], q[k][1], q[k][2], q[k][3]);
  }
  if (en < 0) load_face<FETCH>(rec + 12, pol, q3[0], q3[1], q3[2], q3[3]);
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
  const double texit = exit_parameter(sc);
  const int my_i = target_in(P, r, texit, sc.nbr, tgt, id);
  advance<false, FETCH == kFetchPolicyAgg || FETCH == kFetchPolicyL1Agg, NS, TM, MO, CU, MU>(P, my_i, r, texit, sc.nbr,
                                                                                          sc.back, c, true, sl, sc.bden);
  target_out(r, tgt);
}

// ---- cooperative record fetch (kFetchCoopL1) ------------------------------------------------
// A lane's own record load touches a line no other lane of the warp asks for, so a warp-wide 128-bit load
// costs 32 line lookups in L1TEX and up to 32 L2 requests, and each record line is asked for six times per
// crossing.  Here the warp fetches the records of its active lanes together: lanes 8j..8j+7 copy the eight
// 16-byte pieces of one record (cp.async, L1-allocating, evict_last in L2) into a per-warp shared-memory row,
// so every copy instruction touches 4 lines and asks each of them once.  The pieces of the entry face are not
// copied and the others are packed into three 32-byte slots, so each lane reads back exactly the faces
// plane_step() would have loaded; the fourth face of a ray's first tet comes with the lane's own load.
constexpr int kCoopRowBytes = 96;

// Shared-memory address of 16-byte chunk p (0..5) of row m.  Rows are packed at 96 bytes; in rows 4..7 of every
// eight the two chunks of each face trade places, so that eight consecutive rows read at the same chunk land in
// eight different 16-byte bank groups (a quarter-warp phase of ld.shared.v2.f64 is then conflict-free).
__device__ __forceinline__ uint32_t coop_chunk(uint32_t rows, int m, int p) {
  return rows + (uint32_t)(kCoopRowBytes * m + 16 * (p ^ ((m >> 2) & 1)));
}

// The (element, face not to copy) slots: rank m sits in group m & 3 at position m >> 2, so the slots of the
// eight records lanes 8g..8g+7 copy are one contiguous 64-byte run.  Groups are 80 bytes apart, so the four groups
// a 128-bit read asks for lie in different banks.  (96 would also spare the slot stores a bank conflict, but with
// 256 bytes more per block, launch_persist's carveout for five plain blocks passes the 164 KB configuration.)
constexpr int kCoopSlotGroupBytes = 80;

// Per-warp shared memory of the cooperative fetch: 32 rows by rank, then the four slot groups.
constexpr int kCoopWarpBytes = 32 * kCoopRowBytes + 4 * kCoopSlotGroupBytes;

// One crossing for every active lane of the warp (act: the active mask; every lane of the warp calls it).
// rows: shared-memory address of the warp's kCoopWarpBytes.
template <int NS = 0, bool TM = false, bool MO = false, bool CU = false, bool MU = false>
__device__ __forceinline__ void coop_plane_step(const WalkParams &P, Ray &r, Counters &c, unsigned act, uint32_t rows,
                                                double *tgt, const int32_t *id, const ScoreLane *sl = nullptr) {
  const int lane = threadIdx.x & 31;
  const bool on = (act >> lane) & 1u;
  const int n = __popc(act);
  const int rank = __popc(act & ((1u << lane) - 1u));  // idle lanes leave no gap between the rows
  const int en = r.entry;
  const uint64_t pol = l2_policy_keep_now();
  const uint32_t slots = rows + 32 * kCoopRowBytes;
  double q[3][4], q3[4] = {0.0, 0.0, 0.0, 0.0};
  if (on) {
    // the face not to copy: the entry face, or on a first tet (entry -1) the fourth, which the owner loads itself
    asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(slots + kCoopSlotGroupBytes * (rank & 3) + 8 * (rank >> 2)),
                 "r"(r.e), "r"(en & 3)
                 : "memory");
    if (en < 0) load_face<kFetchPolicyL1>(P.tets[r.e].d + 12, pol, q3[0], q3[1], q3[2], q3[3]);
  }
  __syncwarp();
  // Lane 8g + piece copies piece `piece` (half piece & 1 of face f) of the records of ranks g, g + 4, ..., g + 28:
  // round j is rank and row 4j + g, whose chunks trade places (coop_chunk) when j is odd.  The copies are issued
  // under predicates, not behind branches, so the warp's copies leave back to back after the four slot reads.
  const int g = lane >> 3, piece = lane & 7, f = piece >> 1;
  int32_t s[16];  // (element, face not to copy) of round j in s[2j], s[2j + 1]
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%16];\n\t"
               "ld.shared.v4.b32 {%4,%5,%6,%7}, [%16+16];\n\t"
               "ld.shared.v4.b32 {%8,%9,%10,%11}, [%16+32];\n\t"
               "ld.shared.v4.b32 {%12,%13,%14,%15}, [%16+48];"
               : "=r"(s[0]), "=r"(s[1]), "=r"(s[2]), "=r"(s[3]), "=r"(s[4]), "=r"(s[5]), "=r"(s[6]), "=r"(s[7]),
                 "=r"(s[8]), "=r"(s[9]), "=r"(s[10]), "=r"(s[11]), "=r"(s[12]), "=r"(s[13]), "=r"(s[14]), "=r"(s[15])
               : "r"(slots + kCoopSlotGroupBytes * g)
               : "memory");
  const char *src = reinterpret_cast<const char *>(P.tets) + 16 * piece;
  const uint32_t dst_even = rows + kCoopRowBytes * g + 32 * f + 16 * (piece & 1);
  const uint32_t dst_odd = rows + kCoopRowBytes * g + 32 * f + 16 * (~piece & 1);
  const int left = n - g;  // round j copies while 4j < left
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    // Warp-uniform: at most 28 active lanes need seven rounds.  The branch also keeps ptxas from repeating the
    // whole fetch on the divergent path of the two __syncwarp()s around it.
    if (j == 7 && n <= 28) break;
    const int skip = s[2 * j + 1];
    // the faces after the skipped one move up one 32-byte slot
    const uint32_t dst = (j & 1 ? dst_odd : dst_even) + 4 * kCoopRowBytes * j - (f > skip ? 32u : 0u);
    asm volatile("{\n\t.reg .pred p;\n\t.reg .b64 a;\n\t"
                 "setp.gt.s32 p, %3, %4;\n\t"
                 "setp.ne.and.s32 p, %5, %6, p;\n\t"
                 "mad.wide.u32 a, %7, 128, %1;\n\t"
                 "@p cp.async.ca.shared.global.L2::cache_hint [%0], [a], 16, %2;\n\t}"
                 ::"r"(dst), "l"(src), "l"(pol), "r"(left), "r"(4 * j), "r"(f), "r"(skip), "r"(s[2 * j])
                 : "memory");
  }
  // (this also waits for gather copies of a particle stage still in flight: issued before, they rarely land later)
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncwarp();
  if (!on) return;
#pragma unroll
  for (int k = 0; k < 3; ++k)
    asm volatile("ld.shared.v2.f64 {%0,%1}, [%4];\n\t"
                 "ld.shared.v2.f64 {%2,%3}, [%5];"
                 : "=d"(q[k][0]), "=d"(q[k][1]), "=d"(q[k][2]), "=d"(q[k][3])
                 : "r"(coop_chunk(rows, rank, 2 * k)), "r"(coop_chunk(rows, rank, 2 * k + 1)));
  plane_exit<false, NS, TM, MO, CU, MU>(P, r, c, q, q3, tgt, id, sl);
}

// Lean crossing step.  The compiler can sink the third record load of plane_step() below the arithmetic on
// the first two, so its latency is paid a second time.  Here the
// three loads are one asm block (issued back to back, before any use), the neighbour is decoded once,
// the parallel-face tolerance is computed once per step, and the ray target is not carried in registers
// (end_ray<true> re-reads it from the caller's array), which makes room for the loads in flight.
template <bool L1ALLOC>
__device__ __forceinline__ void load_faces3(const double *p0, const double *p1, const double *p2, uint64_t pol,
                                            double (&q)[3][4]) {
  if constexpr (L1ALLOC)
    asm volatile(
        "ld.global.nc.L2::cache_hint.v2.f64 {%0,%1}, [%12], %15;\n\t"
        "ld.global.nc.L2::cache_hint.v2.f64 {%2,%3}, [%12+16], %15;\n\t"
        "ld.global.nc.L2::cache_hint.v2.f64 {%4,%5}, [%13], %15;\n\t"
        "ld.global.nc.L2::cache_hint.v2.f64 {%6,%7}, [%13+16], %15;\n\t"
        "ld.global.nc.L2::cache_hint.v2.f64 {%8,%9}, [%14], %15;\n\t"
        "ld.global.nc.L2::cache_hint.v2.f64 {%10,%11}, [%14+16], %15;"
        : "=d"(q[0][0]), "=d"(q[0][1]), "=d"(q[0][2]), "=d"(q[0][3]), "=d"(q[1][0]), "=d"(q[1][1]), "=d"(q[1][2]),
          "=d"(q[1][3]), "=d"(q[2][0]), "=d"(q[2][1]), "=d"(q[2][2]), "=d"(q[2][3])
        : "l"(p0), "l"(p1), "l"(p2), "l"(pol));
  else
    asm volatile(
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%12], %15;\n\t"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%2,%3}, [%12+16], %15;\n\t"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%4,%5}, [%13], %15;\n\t"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%6,%7}, [%13+16], %15;\n\t"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%8,%9}, [%14], %15;\n\t"
        "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%10,%11}, [%14+16], %15;"
        : "=d"(q[0][0]), "=d"(q[0][1]), "=d"(q[0][2]), "=d"(q[0][3]), "=d"(q[1][0]), "=d"(q[1][1]), "=d"(q[1][2]),
          "=d"(q[1][3]), "=d"(q[2][0]), "=d"(q[2][1]), "=d"(q[2][2]), "=d"(q[2][3])
        : "l"(p0), "l"(p1), "l"(p2), "l"(pol));
}

template <int FETCH>
__device__ __forceinline__ void plane_step_lean(const WalkParams &P, int my_i, Ray &r, Counters &c, uint64_t pol) {
  constexpr bool L1 = FETCH == kFetchLeanL1;
  const double *rec = P.tets[r.e].d;
  const int en = r.entry;
  // faces 0,1,2 with the entry face skipped: offsets (en<=0), (en<=1)+1, (en<=2)+2 for en >= 0; 0,1,2 for en < 0
  const int f0 = (en == 0) ? 1 : 0, f1 = (en >= 0 && en <= 1) ? 2 : 1, f2 = (en >= 0 && en <= 2) ? 3 : 2;
  double q[3][4], q3[4];
  load_faces3<L1>(rec + 4 * f0, rec + 4 * f1, rec + 4 * f2, pol, q);
  if (en < 0) load_face<L1 ? kFetchPolicyL1 : kFetchPolicy>(rec + 12, pol, q3[0], q3[1], q3[2], q3[3]);
  const double tol = kParallelTol * (fabs(r.ux) + fabs(r.uy) + fabs(r.uz));
  LeanScan sc;
  scan_face_lean(sc, q[0][0], q[0][1], q[0][2], q[0][3], f0, tol, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
  scan_face_lean(sc, q[1][0], q[1][1], q[1][2], q[1][3], f1, tol, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
  scan_face_lean(sc, q[2][0], q[2][1], q[2][2], q[2][3], f2, tol, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
  if (en < 0) scan_face_lean(sc, q3[0], q3[1], q3[2], q3[3], 3, tol, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
  int32_t nb, bk;
  decode_lean(sc, r.e, nb, bk);
  // The next tet is known here, ~80 instructions (a division, the tally, the loop overhead) before its
  // record is asked for: start the line on its way from DRAM to L2 now.  Once the tet table is larger
  // than the L2 many record fetches miss there, and the prefetch gives such a miss a head start.
  if (nb >= 0 && sc.bnum < sc.bden)
    asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(P.tets + nb));
  advance<true>(P, my_i, r, exit_parameter(sc), nb, bk, c, true);
}

// ---- compact layout (kFetchEdge) ----------------------------------------------------------
constexpr int kPlaneMode = -2;  // EdgeRay::dv of a ray that is finishing on the plane records

__device__ __forceinline__ void ld256_b64(const void *p, uint64_t pol, unsigned long long &a,
                                          unsigned long long &b, unsigned long long &c, unsigned long long &d) {
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0,%1}, [%4], %5;\n\t"
               "ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%2,%3}, [%4+16], %5;"
               : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p), "l"(pol));
}

// First tet of a ray, out of line: its register footprint (four vertices, six edge functions)
// must not set the allocation of the per-crossing path.  The TetStart line has already been
// loaded by the caller (together with the other lanes' per-crossing loads, so the warp waits for
// memory once per iteration); everything crosses the call by value.
struct FirstOut {
  EdgeRay g;
  double texit;
  int32_t next, roles, ok;
};
__device__ __noinline__ FirstOut edge_first_compute(double v0, double v1, double v2, double v3, double v4, double v5,
                                                    double v6, double v7, double v8, double v9, double v10,
                                                    double v11, unsigned long long w0, unsigned long long w1,
                                                    unsigned long long w2, unsigned long long w3, double ox, double oy,
                                                    double oz, double ux, double uy, double uz) {
  const double v[12] = {v0, v1, v2, v3, v4, v5, v6, v7, v8, v9, v10, v11};
  TetLinks L;
  L.nbr[0] = (uint32_t)w0; L.nbr[1] = (uint32_t)(w0 >> 32); L.nbr[2] = (uint32_t)w1; L.nbr[3] = (uint32_t)(w1 >> 32);
  L.opp[0] = (uint32_t)w2; L.opp[1] = (uint32_t)(w2 >> 32); L.opp[2] = (uint32_t)w3; L.opp[3] = (uint32_t)(w3 >> 32);
  Ray r;
  r.ox = ox; r.oy = oy; r.oz = oz; r.ux = ux; r.uy = uy; r.uz = uz;
  FirstOut o;
  o.g.dv = 0;
  o.texit = 0.0;
  o.next = -1;
  o.roles = 0;
  o.ok = edge_first(r, o.g, L, v, o.texit, o.next, o.roles) ? 1 : 0;
  return o;
}

// A ray that met a coplanar edge finishes on the plane records.  Out of line and by value for the
// same reason as edge_first_step: rare, and its registers must not count against the crossing loop.
struct PlaneOut {
  double texit;
  int32_t next, back;
};
__device__ __noinline__ PlaneOut plane_fallback_step(const TetRecord *tets, int32_t e, int32_t en, double ox,
                                                     double oy, double oz, double ux, double uy, double uz) {
  const uint64_t pol = l2_policy_stream_now();
  ExitScan sc;
  const double *rec = tets[e].d;
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    if (f == en) continue;
    double a, b, c, d;
    load_face<kFetchPolicy>(rec + 4 * f, pol, a, b, c, d);
    int32_t nb, bk;
    face_payload(a, b, c, d, e, f, nb, bk);
    scan_face(sc, a, b, c, d, nb, bk, ox, oy, oz, ux, uy, uz);
  }
  PlaneOut o;
  o.texit = exit_parameter(sc);
  o.next = sc.nbr;
  o.back = sc.back;
  return o;
}

// One crossing of the edge-function walk.  Requests first, for every lane at once: the TetLinks
// sector of the current tet + the one new vertex (keep policy; vertices also allocate in L1), or on
// the first tet of a ray the four sectors of its TetStart line (streaming policy).  `tgt` is the
// lane's shared-memory slot holding the ray's target (Ray::tx,ty,tz are not kept in registers).
__device__ __forceinline__ void edge_persist_step(const WalkParams &P, int my_i, Ray &r, EdgeRay &g,
                                                  Counters &c, uint64_t keep, double *tgt) {
  const bool plane = g.dv == kPlaneMode;
  const bool first = r.entry < 0;
  unsigned long long w0 = 0, w1 = 0, w2 = 0, w3 = 0;
  double v[12];
  if (!plane) {
    const TetStart *S = P.starts + r.e;
    const void *pa = first ? (const void *)&S->links : (const void *)(P.links + r.e);
    const double *pb = first ? S->v : reinterpret_cast<const double *>(P.verts + g.dv);
    const uint64_t pol = first ? l2_policy_stream_now() : keep;
    ld256_b64(pa, pol, w0, w1, w2, w3);
    load_face<kFetchPolicyL1>(pb, pol, v[0], v[1], v[2], v[3]);
    if (first) {
      load_face<kFetchPolicy>(S->v + 4, pol, v[4], v[5], v[6], v[7]);
      load_face<kFetchPolicy>(S->v + 8, pol, v[8], v[9], v[10], v[11]);
    }
  }
  double texit;
  int32_t next, roles;
  bool ok = true;
  if (plane) {
    const PlaneOut o = plane_fallback_step(P.tets, r.e, r.entry, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
    texit = o.texit;
    next = o.next;
    roles = o.back;
  } else if (first) {
    const FirstOut o = edge_first_compute(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], v[8], v[9], v[10], v[11],
                                          w0, w1, w2, w3, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
    g = o.g;
    texit = o.texit;
    next = o.next;
    roles = o.roles;
    ok = o.ok != 0;
  } else {
    TetLinks L;
    L.nbr[0] = (uint32_t)w0; L.nbr[1] = (uint32_t)(w0 >> 32); L.nbr[2] = (uint32_t)w1; L.nbr[3] = (uint32_t)(w1 >> 32);
    L.opp[0] = (uint32_t)w2; L.opp[1] = (uint32_t)(w2 >> 32); L.opp[2] = (uint32_t)w3; L.opp[3] = (uint32_t)(w3 >> 32);
    ok = edge_step(r, g, L, v[0], v[1], v[2], texit, next, roles);
  }
  if (ok) {
    // the ray ends in this step (reached / hull / iteration limit): end_ray() needs its target
    if (!(texit < 1.0) || next < 0 || r.iters + 1 >= P.max_iters) {
      r.tx = tgt[0]; r.ty = tgt[1]; r.tz = tgt[2];
    }
    advance(P, my_i, r, texit, next, roles, c, true);
    if (r.iters == 0 && r.stage != kStageDone) {  // a new ray (phase 2 after phase 1)
      tgt[0] = r.tx; tgt[1] = r.ty; tgt[2] = r.tz;
      if (plane) g.dv = 0;  // it starts on the fast path again
    }
  } else {  // coplanar edge: redo this tet, and the rest of the ray, with the planes
    g.dv = kPlaneMode;
    r.entry = -1;
    atomicAdd(&P.stats->fallbacks, 1ull);
  }
}

constexpr int kClaimRun = 4;  // gather mode: a warp takes up to this many consecutive chunks per ticket

// Scheduling state of a persistent warp.  It is warp-uniform and only the refill branch of the kernel uses
// it, once per several crossings, so it lives in a per-warp shared-memory record instead of registers: the
// branch reads it on entry and writes the cursor back on exit, and none of it is live across a crossing.
struct SchedFixed {  // set once per launch
  int total, nchunks, claim_run;
  int own_lo, own_hi, oth_lo, oth_hi;  // die split: chunk ranges of this SM's L2 partition and of the other one
  unsigned int *own_cnt, *oth_cnt;     // die split: their chunk tickets
};
struct SchedCursor {
  int run_base, run_next, run_end, pend_base;  // gather mode: current ticket run, and the next ticket's first chunk
  int tk;                                      // gather mode: the current ticket's ids are ids[tk], the next one's ids[tk ^ 1]
  int split_phase;                             // die split: 0 own chunks, 1 the other partition's, 3 none left, 2 off
  int cur, cursor, cur_count;                  // stage being handed out, its next slot, its particles (0: none)
  int chunk_cur, chunk_next;                   // chunks in the two stages (-1: none)
  uint32_t parity;                             // bit b = phase parity of particle-stage barrier b
};

// REFILL_T: idle lanes are topped up only when at least this many have finished -- the
// refill code then runs with REFILL_T+ active lanes instead of the ~3 that finish per
// iteration, at the price of a few idle lanes in the walk step.
// STAGING: 0 = particle arrays streamed in storage order (TMA bulk copies of the SoA/AoS slices),
// 1 = gather through order[] (binned), 2 = packed rows written by the binning pass (binned, streamed).
// NS: 0 = the plain tally; > 0 = scored walk of up to NS scores (plane-record fetch modes only).  Where the
// scores of a lane live: a shared-memory slot per lane and score (NS * BLOCK doubles per block), written
// once per track, read once per crossing and score -- registers would cost 2 * NS of them, beyond the
// budget of __launch_bounds__(BLOCK, MINB), and re-reading the caller's array per crossing would add NS
// loads to the memory pipe the walk is bound by.
// TM: timed walk (NS > 0): the lane's time state sits in three more slots next to its scores (TimeLane) and its
// current bin in a per-lane int: 3.5 KB more per block of 128 lanes, no register held across the crossing loop.
template <int NS, bool TM = false>
using KernelParams = std::conditional_t<TM, TimedWalkParams, std::conditional_t<NS == 0, WalkParams, ScoredWalkParams>>;

// CU: face currents (NS > 0): the lane's weight sits in one more slot (kCurrentSlot), 1 KB more per block of 128 lanes.
template <int NS, bool TM, bool CU>
using KernelParamsCU = std::conditional_t<CU, CurrentWalkParams, KernelParams<NS, TM>>;

// Shared-memory rows of score_wl: the scores, for the timed walk its three time slots, with currents the weight, with
// cosine bins 1 / |u| and the cosine of the crossing in flight (MU: 2 KB more per block of 128 lanes).
template <int NS, bool TM, bool CU = false, bool MU = false>
constexpr int kLaneSlots = NS > 0 ? NS + (TM ? 3 : 0) + (CU ? 1 : 0) + (MU ? 2 : 0) : 1;

// The lane's ScoreLane, built where it is used from the parameters and the thread index, so that nothing of
// it stays live in registers across the crossing loop.  wl0: slot 0 of lane 0; STEP lanes per score.
template <int NS, int STEP>
__device__ __forceinline__ ScoreLane score_lane(const KernelParams<NS> &P, double *wl0) {
  if constexpr (NS > 0) return ScoreLane{P.sc.responses, wl0 + threadIdx.x, P.sc.nscores, P.sc.stride, STEP};
  else return ScoreLane{};
}

// score_lane() of the timed walk, plus the lane's bin slot (bin0: lane 0's); for TM == false exactly score_lane().
template <int NS, int STEP, bool TM>
__device__ __forceinline__ std::conditional_t<TM, TimeLane, ScoreLane> walk_lane(const KernelParams<NS, TM> &P, double *wl0,
                                                                                 int32_t *bin0) {
  if constexpr (TM) {
    TimeLane tl;
    tl.responses = P.sc.responses;
    tl.wl = wl0 + threadIdx.x;
    tl.n = P.sc.nscores;
    tl.stride = P.sc.stride;
    tl.step = STEP;
    tl.bin = bin0 + threadIdx.x;
    return tl;
  } else {
    return score_lane<NS, STEP>(P, wl0);
  }
}

#define PTB_PERSIST_NAME walk_persist_kernel
#define PTB_PERSIST_PARAMS KernelParams<NS, TM>
#define PTB_PERSIST_CU false
#define PTB_PERSIST_MU false
#include "walk_persist_kernel.cuh"  // (no include guard: it is meant to be included three times)
#undef PTB_PERSIST_NAME
#undef PTB_PERSIST_PARAMS
#undef PTB_PERSIST_CU
#undef PTB_PERSIST_MU
#define PTB_PERSIST_NAME walk_persist_current_kernel
#define PTB_PERSIST_PARAMS CurrentWalkParams
#define PTB_PERSIST_CU true
#define PTB_PERSIST_MU false
#include "walk_persist_kernel.cuh"
#undef PTB_PERSIST_NAME
#undef PTB_PERSIST_PARAMS
#undef PTB_PERSIST_CU
#undef PTB_PERSIST_MU
#define PTB_PERSIST_NAME walk_persist_current_mu_kernel
#define PTB_PERSIST_PARAMS CurrentWalkParams
#define PTB_PERSIST_CU true
#define PTB_PERSIST_MU true
#include "walk_persist_kernel.cuh"
#undef PTB_PERSIST_NAME
#undef PTB_PERSIST_PARAMS
#undef PTB_PERSIST_CU
#undef PTB_PERSIST_MU

// Blocks per SM of the last persistent launch (diagnostics: engine option "walk_blocks_per_sm").
inline int &last_persist_occupancy() {
  static int occ = 0;
  return occ;
}

template <int BLOCK, int FETCH, int MINB, int REFILL_T = 1, int GATHER = 0, int CARVE = -1, int NS = 0, bool TM = false,
          bool MO = false, bool CU = false, bool MU = false>
cudaError_t launch_persist(const KernelParamsCU<NS, TM, CU> &p, long long n, cudaStream_t stream) {
  constexpr auto kernel = [] {
    if constexpr (MU) return walk_persist_current_mu_kernel<BLOCK, FETCH, MINB, REFILL_T, GATHER, NS, TM, MO>;
    else if constexpr (CU) return walk_persist_current_kernel<BLOCK, FETCH, MINB, REFILL_T, GATHER, NS, TM, MO>;
    else return walk_persist_kernel<BLOCK, FETCH, MINB, REFILL_T, GATHER, NS, TM, MO>;
  }();
  static int sms = 0, occ = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int carve = CARVE < 0 ? (int)cudaSharedmemCarveoutMaxShared : CARVE;
    if (CARVE >= 0) {
      // the lane slots (targets, ids, scores) must not cost resident blocks: widen the carveout to what
      // MINB blocks need
      cudaFuncAttributes fa{};
      int per_sm = 0, reserved = 0;
      cudaFuncGetAttributes(&fa, kernel);
      cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
      cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev);
      if (per_sm > 0)
        carve = std::max(carve, (int)((100LL * MINB * ((long long)fa.sharedSizeBytes + reserved) + per_sm - 1) / per_sm));
      carve = std::min(carve, 100);
    }
    // leave as much of the unified L1/smem array to shared memory as the kernel can use
    cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carve);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, BLOCK, 0);
    if (occ < 1) occ = 1;
  }
  last_persist_occupancy() = occ;
  const long long nchunks = (n + kChunk - 1) / kChunk;
  const long long want = (nchunks + BLOCK / 32 - 1) / (BLOCK / 32);
  const unsigned grid = (unsigned)std::min<long long>(want, (long long)sms * occ);
  cudaError_t e = cudaMemsetAsync(p.work_counter, 0, sizeof(unsigned int), stream);
  if (e != cudaSuccess) return e;
  if (GATHER != 0 && p.die0_sms > 0 && p.work_counter2) {
    e = cudaMemsetAsync(p.work_counter2, 0, sizeof(unsigned int), stream);
    if (e != cudaSuccess) return e;
  }
  kernel<<<grid, BLOCK, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace
}  // namespace ptb
