// Launch interface of the sm_90a walk/tally kernels (walk_kernels.cu).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "tet_mesh.hpp"
#include "walk_core.cuh"

namespace ptb {

// Values are stable (options and tests refer to them); the gaps are experiments that were measured,
// lost and removed (9/10 other refill thresholds, 11/12/14 cooperative transposed fetch, 18).
// libpumitally.so contains the four kernels the engine chooses between -- 0, 8, 16, 24; the other
// numbers are measured alternatives compiled only into libpumitally_exp.so
// (experiments/walk_experiments.cu, build flag PTB_EXPERIMENTS).
enum WalkVariant : int {
  kVariantLdg = 0,    // thread per particle, the tet record as 4 sectors of two 128-bit loads (first correct path)
  kVariantBulk = 1,   // thread per particle, record staged in smem by cp.async.bulk + mbarrier
  kVariantQuad = 2,   // 4 lanes per particle (lane per face), coalesced 32 B loads
  kVariantPersist = 3,               // persistent warps, TMA-staged particle chunks, per-lane refill
  kVariantPersistPolicy = 4,         // 3 + L2 evict_last on tets / evict_first on the particle stream
  kVariantPersistPolicy128 = 5,      // 4 + L2::128B prefetch size on tet loads
  kVariantPersistBulk = 6,           // 4 with tet records fetched by cp.async.bulk into smem rows
  kVariantPersistPolicy128Occ8 = 7,  // 5 compiled for 8 resident blocks (64 registers)
  kVariantPersistRefill8 = 8,        // 4, refilling only when >= 8 lanes are idle (default, mesh <~ 2x L2)
  kVariantPersistRefill8Occ8 = 9,    // 8 compiled for 8 resident blocks (64 registers) -- re-test after entry-face elision
  kVariantPersistBulkOcc7 = 13,      // 6 compiled for 7 resident blocks
  kVariantPersistGather = 15,        // 8 on spatially binned particles (order[] from launch_bin_particles)
  kVariantPersistGatherL1 = 16,      // 15 with the cooperative L1-allocating record fetch, 5 blocks/SM (default, mesh >> L2)
  kVariantPersistGatherPlain = 17,   // 15 with plain tet loads (no L2 policy)
  kVariantEdge = 20,        // compact layout + edge-function exit test (walk_compact.cuh), streaming order
  kVariantEdgeGather = 21,  // 20 on spatially binned particles
  kVariantEdgeOcc5 = 22,    // 20 compiled for 5 resident blocks (96 registers, a few spills)
  kVariantEdgeOcc6 = 23,    // 20 compiled for 6 resident blocks (80 registers, more spills)
  kVariantPacked = 24,      // 8 on a packed, spatially sorted copy of the flying particles' inputs (bin + pack pass)
  kVariantPackedL1 = 25,    // 24 with L1-allocating tet loads (neighbouring lanes share records once particles are sorted)
  kVariantPackedL1Occ6 = 26,
  kVariantTwoRays = 27,        // 8 with two rays per lane in flight (software-pipelined walk)
  kVariantPersistAggTally = 28,  // 8 with the warp-aggregated tally (match.any + shuffles)
  kVariantGatherAggTally = 29,   // 16 with the warp-aggregated tally
  kVariantLean = 30,        // 8 with the lean crossing step (three loads as one block, payload decoded once, target re-read)
  kVariantLeanGather = 31,  // 16 with the lean crossing step
  kVariantLeanPacked = 32,  // 24 with the lean crossing step
  kNumVariants = 33
};

// how a variant gets its particles: through order[] from the binning pass / through packed rows
inline bool variant_is_gather(int v) {
  return v == kVariantPersistGather || v == kVariantPersistGatherL1 || v == kVariantPersistGatherPlain ||
         v == kVariantEdgeGather || v == kVariantGatherAggTally || v == kVariantLeanGather;
}
inline bool variant_is_packed(int v) {
  return v == kVariantPacked || v == kVariantPackedL1 || v == kVariantPackedL1Occ6 || v == kVariantLeanPacked;
}


cudaError_t launch_walk(const WalkParams &p, int variant, int block, cudaStream_t stream);
bool walk_variant_available(int variant);  // compiled into this library?
// Tallied walk: the same kernels instantiated for up to kMaxScores scores (walk_core.cuh, ScoreParams; p.flux is
// [element][p.sc.stride]); product variants 0, 8, 16, 24 only.  p.tm is read only when timed.
// timed: the time filter (walk_core.cuh, TimeParams).  p.flux points at time bin 0 of the score bin; time bin j is at
// p.flux + j * p.tm.slice.  p.sc.responses may be nullptr when p.sc.nscores == 1 (every response 1).
// moments: the moment walk (walk_core.cuh, moment_tally): p.sc.stride is kMomentSlots * score_stride(nscores), and
// p.sc.responses may be nullptr when p.sc.nscores == 1 (every response 1: the plain and binned moves).
// currents: face currents (walk_core.cuh, CurrentParams) into p.cu.cur ([E][4] per time bin, p.cu.slice apart); p.cu is
// read only then, and p.sc.responses may be nullptr when p.sc.nscores == 1 here too.  p.cu.nmu > 0 (currents only):
// cosine bins, the MU kernels; cosine bin k of the currents is at p.cu.cur + k * p.cu.mu_stride.
cudaError_t launch_walk_tallied(const CurrentWalkParams &p, bool timed, bool moments, bool currents, int variant,
                                int block, cudaStream_t stream);
// blocks per SM the occupancy calculator gave the last persistent walk kernel launched (0: none yet)
int walk_blocks_per_sm();
// origin == nullptr: the binning key is the stored position (state)
// mid != nullptr: the key is the midpoint of (start, mid[i]) -- pass the dest array
cudaError_t launch_bin_particles(const SeedGrid &g, const double *origin, const ParticleState *state,
                                 const double *mid, const int8_t *flying, int32_t begin, int32_t end, int32_t *pcell, unsigned int *count,
                                 unsigned int *sums, int32_t *order, unsigned int *work_count,
                                 cudaStream_t stream);
// Like launch_bin_particles, but instead of the id list the scatter pass writes one PackedRow per
// flying particle (origin, dest, weight, id, parent element + relocate flag) in cell order.
cudaError_t launch_bin_pack_particles(const SeedGrid &g, const double *origin, const double *dest,
                                      const double *weights, const int8_t *flying, const ParticleState *state,
                                      int32_t begin, int32_t end, int32_t *pcell, unsigned int *count,
                                      unsigned int *sums, PackedRow *rows, unsigned int *work_count,
                                      bool midpoint_key, cudaStream_t stream);
cudaError_t launch_seed_points(const SeedGrid &g, double *xyz, cudaStream_t stream);
cudaError_t launch_seed_finalize(const double *xyz, const ParticleState *state, int32_t *cell_tet,
                                 int32_t ncell, cudaStream_t stream);
cudaError_t launch_init_particles(ParticleState *state, int32_t n, double cx, double cy, double cz,
                                  int32_t elem, cudaStream_t stream);
// origin[3*idx..] = (x,y,z) for every entry of the patch list
cudaError_t launch_patch_origins(double *origin, const PatchEntry *list, int32_t count, cudaStream_t stream);
// Phase 1 of MoveToNextLocation (PumiTallyImpl.cpp:71-112) for the listed particles only: each is
// walked, tally off, from its stored position to (x,y,z) of its entry and its state is updated; an
// entry with a non-finite position makes the particle sit the move out (flying[idx] <- 0, counted as
// lost).  p.origin / p.dest / p.weights are ignored.  For the host path whose mirror is the device's
// own particle positions: every particle not listed is already where its origin says.
cudaError_t launch_relocate_patches(const WalkParams &p, const PatchEntry *list, int32_t count, int8_t *flying,
                                    cudaStream_t stream);
// particle slots [begin, end) <-> (xyz[3k..], elem[k]) with k = slot - begin; elem in the caller's numbering
cudaError_t launch_set_state(ParticleState *state, const double *xyz, const int32_t *elem, const int32_t *elem_map,
                             int32_t begin, int32_t end, cudaStream_t stream);
cudaError_t launch_get_state(const ParticleState *state, double *xyz, int32_t *elem, const int32_t *elem_map,
                             int32_t begin, int32_t end, cudaStream_t stream);
cudaError_t launch_flux_to_caller_order(const double *flux, const int32_t *orig_of_internal, double *out, int64_t n,
                                        cudaStream_t stream);
// scored flux [n][stride] (internal order) -> out[k * n + caller's id], k < nscores
cudaError_t launch_scores_to_caller_order(const double *flux, const int32_t *orig_of_internal, double *out, int64_t n,
                                          int32_t nscores, int32_t stride, cudaStream_t stream);
// scored flux [n][stride] -> out[k * n + e] = flux / volume / per_source (internal order)
cudaError_t launch_normalize_scores(const double *flux, const double *volume, double *out, int64_t n, int32_t nscores,
                                    int32_t stride, double per_source, cudaStream_t stream);
// xyz[3i..3i+2] = position of particle i for i in [begin, end)
cudaError_t launch_export_positions(const ParticleState *state, double *xyz, int32_t begin, int32_t end,
                                    cudaStream_t stream);
// out = flux / volume / per_source (NormalizeFlux, PumiTallyImpl.cpp:393-405; per_source = 1 is the reference)
cudaError_t launch_normalize(const double *flux, const double *volume, double *out, int64_t n,
                             double per_source, cudaStream_t stream);
// *total += sum of weights[i] over flying particles of [begin, end)
// l2_partitions.cu: which SMs share an L2 partition (mask bit s = partition of SM s); 0 = found two clear groups
int probe_l2_partitions(uint32_t mask[8], int *die0_sms, int *nsms, cudaStream_t stream);

// mask[i] = flying[i] && bins[i] == bin  (bin == nbins selects the particles outside [0, nbins))
cudaError_t launch_bin_mask(const int8_t *flying, const int32_t *bins, int32_t bin, int32_t nbins, int8_t *mask,
                            int32_t begin, int32_t end, cudaStream_t stream);
cudaError_t launch_sum_flying_weights(const int8_t *flying, const double *weights, int32_t begin, int32_t end,
                                      double *total, cudaStream_t stream);

// locate_kernels.cu.  Point location of n points (AoS xyz), thread per point (locate_point).  internal[i] <- internal
// element id, out[i] <- caller's id (-1: outside); either may be nullptr.  n < 2^39.
cudaError_t launch_locate(const LocateParams &p, const double *xyz, int64_t n, int32_t *internal, int32_t *out,
                          const int32_t *orig_of_internal, cudaStream_t stream);
// out[r * pitch + i] = vals[r * E + e] (+ grads[(r * E + e) * 3 ..] . (xyz_i - cen[3 e ..]) when grads != nullptr) for
// r < R, e = internal[i]; NaN where e < 0.
cudaError_t launch_evaluate(const double *xyz, const int32_t *internal, int64_t n, const double *vals, const double *grads,
                            const double *cen, int64_t E, int32_t R, double *out, int64_t pitch, cudaStream_t stream);
// Collision estimator (walk_core.cuh, collision_event), thread per event.  Located: event i at xyz[3i..], located as
// launch_locate does.  Particles: event i at particle i's stored position and element, for every i < n with
// collided[i] != 0.  w[i], resp[i * c.nscores + k] (nullptr: every response 1), bins[i] (nullptr: bin 0), times[i]
// (read only when c.nt > 0).  counts[0..2] += events tallied, outside the mesh, rejected.  n < 2^39.
cudaError_t launch_collide_located(const LocateParams &l, const CollisionParams &c, const double *xyz, int64_t n,
                                   const double *w, const double *resp, const int32_t *bins, const double *times,
                                   unsigned long long *counts, cudaStream_t stream);
cudaError_t launch_collide_particles(const ParticleState *state, const int8_t *collided, int32_t n,
                                     const CollisionParams &c, const double *w, const double *resp, const int32_t *bins,
                                     const double *times, unsigned long long *counts, cudaStream_t stream);

// detector_kernels.cu.  Point detectors (walk_core.cuh, detector_event), thread per (event, detector) ray, q = d n + i.
// Located: event i at xyz[3i..], located as launch_locate does (n < 2^39 / D).  Particles: event i at particle i's stored
// position and element, for every i < n with flagged[i] != 0.  w[i], pdf[i D + d] (nullptr: 1 / (4 pi)), resp[i nscores
// + k] (nullptr: every response 1), bins[i] (nullptr: bin 0), times[i] and speeds[i] (read only when p.nt > 0).  The
// scores go to p.tally, the outcomes to counts[kDetCounters].  Up to kDetSmemSlots slots are aggregated in shared memory.
// hull != nullptr: the detector void (walk_core.cuh, detector_ray) with that hull grid, its own kernels, which also
// count the hull entries in counts[kDetCountHullEntries] (counts then holds kDetCountersVoid).
constexpr int kDetCountTraced = 0, kDetCountShadowed = 1, kDetCountLost = 2, kDetCountInsideR0 = 3,
              kDetCountCrossings = 4, kDetCountOutside = 5, kDetCountRejected = 6, kDetCounters = 7,
              kDetCountHullEntries = 7, kDetCountersVoid = 8;
constexpr int64_t kDetSmemSlots = 2048;
cudaError_t launch_detect_located(const LocateParams &l, const DetectorParams &p, const double *xyz, int64_t n,
                                  const double *w, const double *pdf, const double *resp, const int32_t *bins,
                                  const double *times, const double *speeds, unsigned long long *counts,
                                  cudaStream_t stream, const HullGrid *hull = nullptr);
cudaError_t launch_detect_particles(const WalkParams &wp, const DetectorParams &p, const ParticleState *state,
                                    const int8_t *flagged, int32_t n, const double *w, const double *pdf,
                                    const double *resp, const int32_t *bins, const double *times, const double *speeds,
                                    unsigned long long *counts, cudaStream_t stream, const HullGrid *hull = nullptr);

// stats_kernels.cu.  Batch statistics (batch_stats.cuh).  fold: (mean[i], m2[i]) <- welford_fold(x[i] / *divisor, nb)
// for i < n, nb the number of batches including this one; the divisor is read on the device.
cudaError_t launch_batch_fold(const double *x, double *mean, double *m2, int64_t n, const double *divisor, double nb,
                              cudaStream_t stream);
// merge: (mean[i], m2[i]) of na batches <- welford_merge(mean_b[i], m2_b[i], na, nb) for i < n, in place: the statistics
// of the na + nb batches together.
cudaError_t launch_batch_merge(const double *mean_b, const double *m2_b, double *mean, double *m2, int64_t n, double na,
                               double nb, cudaStream_t stream);
// The m0 slots of R result arrays [R][E][stride] of means (and m2, unread for kind 0) of nb batches -> out[(r * nscores
// + k) * E + caller's id of e] = batch_readout(..., volume[e], kind): 0 mean, 1 standard error, 2 relative error.
cudaError_t launch_batch_readout(const double *mean, const double *m2, const double *volume,
                                 const int32_t *orig_of_internal, double *out, int64_t E, int32_t R, int32_t nscores,
                                 int32_t stride, double nb, int kind, cudaStream_t stream);
// Local entries j < n of (mean, m2) are global entries goff + j.  Over the global entries of [base, base + len) that
// are the m0 slot of `score` ((g - base) % stride == score) and have a nonzero mean: red[0] <- the bits of the largest
// relative error (0.0 if none), red[1] <- their number.  red is zeroed first, on the stream.
cudaError_t launch_batch_max_rel_err(const double *mean, const double *m2, int64_t n, int64_t goff, int64_t base,
                                     int64_t len, int32_t stride, int32_t score, double nb, unsigned long long *red,
                                     cudaStream_t stream);
// Region sums (batch_stats.cuh, RegionPlan) of the m0 slots [0, nscores) of narrays result arrays [a][E][stride] at
// flux (array a at flux + a * array_len), over a plan's levels[nlevels] with its elems and starts on the device:
// out[(a * nregions + g) * nscores + k] is the sum of score k of array a over region g.  scratch holds
// region_scratch_len doubles (scratch_len), which may be 0 with one level.
struct RegionLevel;
cudaError_t launch_region_sums(const double *flux, int64_t array_len, int32_t stride, int32_t nscores, int64_t narrays,
                               const int32_t *elems, const int32_t *starts, const RegionLevel *levels, int nlevels,
                               double *scratch, int64_t scratch_len, double *out, cudaStream_t stream);
// Region currents (batch_stats.cuh, RegionCurrentPlan): net[a * P + p] = partial[a * P + p] - partial[a * P + rev[p]]
// (the second term 0 for rev[p] < 0), for the narrays arrays of P partial currents that launch_region_sums formed.
cudaError_t launch_region_net(const double *partial, const int32_t *rev, int64_t P, int64_t narrays, double *net,
                              cudaStream_t stream);
// Face currents (walk_core.cuh, CurrentParams) of R arrays [r][E][4] (internal order), opp [4E] as the engine keeps it
// (4 * neighbour + back, kNoFace on the hull).  out[(r * E + caller's id of e) * 4 + f] is, for direction 0 (outgoing) the
// slot of the neighbour across f (interior) or of (e, f) itself (hull), for direction 1 (incoming) the slot (e, f)
// (interior) or nothing (hull).  kind -1: the value / div (nothing: 0); kind 0-2: batch_readout of mean and m2 at the
// slot with volume 1 (nothing: mean and m2 0).  m2 is read for kinds 1 and 2 only.
constexpr uint32_t kNoFace = 0xffffffffu;
cudaError_t launch_current_readout(const double *mean, const double *m2, const uint32_t *opp, const int32_t *orig_of_internal,
                                   double *out, int64_t E, int32_t R, int direction, int kind, double nb, double div,
                                   cudaStream_t stream);
// out[r] = sum of cur[r * 4E + hull[k]] over k < nhull, for r < R, in a fixed order (the same bits every time)
cudaError_t launch_leakage(const double *cur, int64_t E, int32_t R, const uint32_t *hull, int64_t nhull, double *out,
                           cudaStream_t stream);

// ww_kernels.cu.  Weight windows (weight_windows.cuh).  generate: table[b * E + e] <- ww_generate of the m0 value of
// group b and element e of nb batches, at mean[b * pitch + e * stride] and m2 alike, with phimax the largest eligible
// phi of the group; red [ngroups] is scratch (zeroed first, on the stream).
cudaError_t launch_ww_generate(const double *mean, const double *m2, const double *volume, int64_t E, int32_t ngroups,
                               int64_t pitch, int32_t stride, double nb, double max_rel_err, double c, double ratio,
                               unsigned long long *red, double2 *table, cudaStream_t stream);
// (lower[i], upper[i]) <- the window of group groups[i] (nullptr: 0) in particle i's parent element, for i < n
cudaError_t launch_ww_particles(const ParticleState *state, int32_t n, const int32_t *groups, const double2 *table,
                                int32_t ngroups, int64_t E, double *lower, double *upper, cudaStream_t stream);
// the same at n points (AoS xyz) located as launch_locate locates them; n < 2^39
cudaError_t launch_ww_points(const LocateParams &p, const double *xyz, int64_t n, const int32_t *groups,
                             const double2 *table, int32_t ngroups, int64_t E, double *lower, double *upper,
                             cudaStream_t stream);

// source_kernels.cu.  Mesh source (source_sample.cuh): sample first + j for j < n, with xyz [3n], elem (caller's
// numbering), group and weight each optional; state != nullptr also places sample j as particle j (parent element
// internal_of_orig[elem]), without a walk.
struct SourceTable;
cudaError_t launch_source_sample(const SourceTable &S, uint64_t seed, uint64_t first, int64_t n, double *xyz,
                                 int32_t *elem, int32_t *group, double *weight, ParticleState *state,
                                 const int32_t *internal_of_orig, cudaStream_t stream);

}  // namespace ptb
