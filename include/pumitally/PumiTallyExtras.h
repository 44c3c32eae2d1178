// Additive calls for code that uses pumitally::PumiTally (the reference class, whose header ships
// unchanged because it is the ABI) and wants what the reference left as TODOs: tally reset between
// batches and per-source-particle normalisation (reference: PumiTally.h:93 "Normalized by element
// volumes and total number of particles" vs PumiTallyImpl.cpp:402 which divides by volume only;
// total_initial_weight, PumiTallyImpl.h:170-171, declared and never used).
//
// engine_of() hands out the C-ABI handle behind a PumiTally object; everything in pumitally_c.h can
// be used on it (pumitally_reset_tally, pumitally_set_source_normalization, pumitally_get_flux,
// pumitally_comm_init / pumitally_allreduce_tally for several GPUs, ...).
#ifndef PUMITALLY_PUMITALLYEXTRAS_H
#define PUMITALLY_PUMITALLYEXTRAS_H

#include "pumitally/PumiTally.h"
#include "pumitally_c.h"

namespace pumitally {

// nullptr if `tally` is not a live PumiTally object
pumitally_engine *engine_of(const PumiTally &tally);

// Start a new batch: zero the flux, the statistics and the initial-track weight.
inline int ResetTally(const PumiTally &tally) { return pumitally_reset_tally(engine_of(tally)); }

// mode 0 volume only (reference behaviour), 1 / num_particles, 2 / value, 3 / total weight of the
// batch's first tracks (see pumitally_set_source_normalization).
inline int SetSourceNormalization(const PumiTally &tally, int mode, double value = 1.0) {
  return pumitally_set_source_normalization(engine_of(tally), mode, value);
}

// Score filter: `nbins` flux arrays; MoveToNextLocationBinned scores particle i into array bins[i]
// (see pumitally_set_score_bins in pumitally_c.h).
inline int SetScoreBins(const PumiTally &tally, int32_t nbins) { return pumitally_set_score_bins(engine_of(tally), nbins); }
inline int MoveToNextLocationBinned(const PumiTally &tally, double *particle_origin, double *particle_destinations,
                                    int8_t *flying, double *weights, const int32_t *bins, int32_t size) {
  return pumitally_move_to_next_location_binned(engine_of(tally), particle_origin, particle_destinations, flying,
                                                weights, bins, size);
}

// Scores: `nscores` responses per particle, tallied in one walk; MoveToNextLocationScored adds
// length * weights[i] * responses[i*nscores + k] to score k (see pumitally_set_scores in pumitally_c.h).
// bins may be nullptr (no score filter).
inline int SetScores(const PumiTally &tally, int32_t nscores) { return pumitally_set_scores(engine_of(tally), nscores); }
inline int MoveToNextLocationScored(const PumiTally &tally, double *particle_origin, double *particle_destinations,
                                    int8_t *flying, double *weights, const double *responses, const int32_t *bins,
                                    int32_t size) {
  return pumitally_move_to_next_location_scored(engine_of(tally), particle_origin, particle_destinations, flying,
                                                weights, responses, bins, size);
}

// Time filter: track-length scores split between the time bins [edges[j], edges[j+1]) each flight spans
// (see pumitally_set_time_bins in pumitally_c.h).  times[i] is particle i's time at its origin, speeds[i]
// its speed; responses may be nullptr with one score, bins may be nullptr (no score filter).
inline int SetTimeBins(const PumiTally &tally, const double *edges, int32_t nedges) {
  return pumitally_set_time_bins(engine_of(tally), edges, nedges);
}
inline int MoveToNextLocationTimed(const PumiTally &tally, double *particle_origin, double *particle_destinations,
                                   int8_t *flying, double *weights, const double *times, const double *speeds,
                                   const double *responses, const int32_t *bins, int32_t size) {
  return pumitally_move_to_next_location_timed(engine_of(tally), particle_origin, particle_destinations, flying,
                                               weights, times, speeds, responses, bins, size);
}

// Linear flux moments (see pumitally_set_moments in pumitally_c.h): with order 1 every move, MoveToNextLocation
// included, also tallies the first spatial moment of the flux in each element; pumitally_get_flux_gradient then
// gives the gradient of the flux's linear projection.
inline int SetMoments(const PumiTally &tally, int32_t order) { return pumitally_set_moments(engine_of(tally), order); }

// Face currents (see pumitally_set_face_currents in pumitally_c.h): the weight crossing every element face in the walk,
// per score bin and time bin.  GetFaceCurrentResults: direction 0 outgoing, 1 incoming; kind 0 value, 1 batch mean,
// 2 standard error, 3 relative error; n = ntime * nbins * E * 4, [time][bin][element][face].  GetLeakage: the outgoing
// current summed over the hull faces, n = ntime * nbins.
inline int SetFaceCurrents(const PumiTally &tally, int32_t on) { return pumitally_set_face_currents(engine_of(tally), on); }
inline int32_t GetFaceCurrents(const PumiTally &tally) { return pumitally_get_face_currents(engine_of(tally)); }
inline int GetFaceCurrentResults(const PumiTally &tally, int32_t direction, int32_t kind, double *out, int64_t n) {
  return pumitally_get_face_current_results(engine_of(tally), direction, kind, out, n);
}
inline int GetLeakage(const PumiTally &tally, int32_t kind, double *out, int64_t n) {
  return pumitally_get_leakage(engine_of(tally), kind, out, n);
}

// Cosine bins of the face currents (see pumitally_set_current_cosine_bins in pumitally_c.h): edges mu_0 < ... < mu_C
// in [0, 1] split every crossing by the cosine between its flight and the face normal.  The current results gain a
// cosine axis after the score-bin axis: GetFaceCurrentResults n = ntime * nbins * C * E * 4, GetLeakage n = ntime *
// nbins * C, GetRegionCurrentResults n = ntime * nbins * C * P.  (nullptr, 0) removes them.
inline int SetCurrentCosineBins(const PumiTally &tally, const double *edges, int32_t nedges) {
  return pumitally_set_current_cosine_bins(engine_of(tally), edges, nedges);
}
inline int32_t GetCurrentCosineBins(const PumiTally &tally) { return pumitally_get_current_cosine_bins(engine_of(tally)); }

// Point queries (see pumitally_locate_points in pumitally_c.h): the element containing each of npts points (AoS xyz),
// -1 outside the mesh; and every normalised result at the points, [time][bin][score][point], n = npts or
// ntime * nbins * nscores * npts (the linear reconstruction with moments, NaN outside).  out_elem may be nullptr.
inline int LocatePoints(const PumiTally &tally, const double *xyz, int64_t npts, int32_t *out_elem) {
  return pumitally_locate_points(engine_of(tally), xyz, npts, out_elem);
}
inline int EvaluatePoints(const PumiTally &tally, const double *xyz, int64_t npts, double *out, int64_t n,
                          int32_t *out_elem = nullptr) {
  return pumitally_evaluate_points(engine_of(tally), xyz, npts, out, n, out_elem);
}

// Collision estimator (see pumitally_set_collision_estimator in pumitally_c.h): a collision tally with the track-length
// tally's configuration.  TallyCollisions scores events at arbitrary points (located as LocatePoints does),
// TallyCollisionsAtParticles at the particles' positions after the last move, for every i with collided[i] != 0 (size
// = num_particles).  Event i adds weights[i] * responses[i * nscores + k] to score k; responses may be nullptr with one
// score, bins nullptr (bin 0), times nullptr without time bins.
inline int SetCollisionEstimator(const PumiTally &tally, int32_t on) {
  return pumitally_set_collision_estimator(engine_of(tally), on);
}
inline int TallyCollisions(const PumiTally &tally, const double *xyz, int64_t nevents, const double *weights,
                           const double *responses = nullptr, const int32_t *bins = nullptr,
                           const double *times = nullptr) {
  return pumitally_tally_collisions(engine_of(tally), xyz, nevents, weights, responses, bins, times);
}
inline int TallyCollisionsAtParticles(const PumiTally &tally, const int8_t *collided, const double *weights,
                                      int32_t size, const double *responses = nullptr, const int32_t *bins = nullptr,
                                      const double *times = nullptr) {
  return pumitally_tally_collisions_at_particles(engine_of(tally), collided, weights, responses, bins, times, size);
}

// Point detectors (see pumitally_set_point_detectors in pumitally_c.h): next-event estimates of the flux at fixed
// points.  SetDetectorCrossSections takes Sigma_t [bin][element] (n = nbins * E).  TallyDetectors scores events at
// arbitrary points (located as LocatePoints does), TallyDetectorsAtParticles at the particles' positions after the last
// move, for every i with flagged[i] != 0 (size = num_particles).  pdf [event][detector] may be nullptr (isotropic).
// GetDetectorResults: kind 0 the open tally per source, 1 batch mean, 2 standard error, 3 relative error.
inline int SetPointDetectors(const PumiTally &tally, const double *xyz, int32_t ndet, const double *r0) {
  return pumitally_set_point_detectors(engine_of(tally), xyz, ndet, r0);
}
// Detector void (see pumitally_set_detector_void in pumitally_c.h): on == 1 lets detector rays cross the space outside
// the mesh as a void, so detectors and events may lie outside it and rays re-enter across concave parts of the hull.
inline int SetDetectorVoid(const PumiTally &tally, bool on) {
  return pumitally_set_detector_void(engine_of(tally), on ? 1 : 0);
}
inline bool GetDetectorVoid(const PumiTally &tally) { return pumitally_get_detector_void(engine_of(tally)) != 0; }
inline int SetDetectorCrossSections(const PumiTally &tally, const double *sigma_t, int64_t n) {
  return pumitally_set_detector_cross_sections(engine_of(tally), sigma_t, n);
}
inline int TallyDetectors(const PumiTally &tally, const double *xyz, int64_t nevents, const double *weights,
                          const double *pdf = nullptr, const double *responses = nullptr, const int32_t *bins = nullptr,
                          const double *times = nullptr, const double *speeds = nullptr) {
  return pumitally_tally_detectors(engine_of(tally), xyz, nevents, weights, pdf, responses, bins, times, speeds);
}
inline int TallyDetectorsAtParticles(const PumiTally &tally, const int8_t *flagged, const double *weights, int32_t size,
                                     const double *pdf = nullptr, const double *responses = nullptr,
                                     const int32_t *bins = nullptr, const double *times = nullptr,
                                     const double *speeds = nullptr) {
  return pumitally_tally_detectors_at_particles(engine_of(tally), flagged, weights, pdf, responses, bins, times, speeds,
                                                size);
}
inline int GetDetectorResults(const PumiTally &tally, int32_t kind, double *out, int64_t n) {
  return pumitally_get_detector_results(engine_of(tally), kind, out, n);
}

// Batch statistics (see pumitally_set_batch_statistics in pumitally_c.h): EndBatch folds the batch's per-source results
// into a running mean and variance on the device and starts the next batch.  GetBatchResults: tally 0 track length, 1
// collision; kind 0 mean, 1 standard error, 2 relative error, 3 gradient of the mean (n as pumitally_get_normalized_flux
// / pumitally_get_flux_gradient take it).  GetBatchMaxRelErr: the largest relative error of one score and how many
// results have a nonzero mean, for tally triggers.
inline int SetBatchStatistics(const PumiTally &tally, int32_t on) {
  return pumitally_set_batch_statistics(engine_of(tally), on);
}
inline int EndBatch(const PumiTally &tally) { return pumitally_end_batch(engine_of(tally)); }
inline int GetBatchResults(const PumiTally &tally, int32_t which, int32_t kind, double *out, int64_t n) {
  return pumitally_get_batch_results(engine_of(tally), which, kind, out, n);
}
inline int GetBatchMaxRelErr(const PumiTally &tally, int32_t which, int32_t score, double *out_max,
                             int64_t *out_nonzero) {
  return pumitally_get_batch_max_rel_err(engine_of(tally), which, score, out_max, out_nonzero);
}

// Region tallies (see pumitally_set_regions in pumitally_c.h): SetRegions groups the elements into nregions regions
// (one id per element in [-1, nregions), -1 for none; nullptr with 0 removes them).  GetRegionResults: tally 0 track
// length, 1 collision; kind 0 the raw sum over each region, 1 sum / volume / the per-source divisor.
// GetRegionBatchResults: kind 0 mean, 1 standard error, 2 relative error of the region sums over the batches.  n is
// nregions (time bin 0, bin 0, score 0) or ntime * nbins * nscores * nregions, [time][bin][score][region].
inline int SetRegions(const PumiTally &tally, const int32_t *region_of_element, int64_t n, int32_t nregions) {
  return pumitally_set_regions(engine_of(tally), region_of_element, n, nregions);
}
inline int GetRegionVolumes(const PumiTally &tally, double *out, int64_t n) {
  return pumitally_get_region_volumes(engine_of(tally), out, n);
}
inline int GetRegionResults(const PumiTally &tally, int32_t which, int32_t kind, double *out, int64_t n) {
  return pumitally_get_region_results(engine_of(tally), which, kind, out, n);
}
inline int GetRegionBatchResults(const PumiTally &tally, int32_t which, int32_t kind, double *out, int64_t n) {
  return pumitally_get_region_batch_results(engine_of(tally), which, kind, out, n);
}

// Region currents (see pumitally_set_region_currents in pumitally_c.h): with regions set and face currents on, the
// partial and net current of every ordered pair of adjacent regions (-1: no region, -2: outside the mesh).
// GetRegionCurrentPairs: the pairs (n = pair count); GetRegionCurrentAreas: each pair's face area.
// GetRegionCurrentResults: which 0 partial, 1 net; kind 0 value, 1 batch mean, 2 standard error, 3 relative error;
// n = ntime * nbins * pair count, [time][bin][pair].
inline int SetRegionCurrents(const PumiTally &tally, int32_t on) {
  return pumitally_set_region_currents(engine_of(tally), on);
}
inline int64_t GetRegionCurrentPairCount(const PumiTally &tally) {
  return pumitally_get_region_current_pair_count(engine_of(tally));
}
inline int GetRegionCurrentPairs(const PumiTally &tally, int32_t *from, int32_t *to, int64_t n) {
  return pumitally_get_region_current_pairs(engine_of(tally), from, to, n);
}
inline int GetRegionCurrentAreas(const PumiTally &tally, double *out, int64_t n) {
  return pumitally_get_region_current_areas(engine_of(tally), out, n);
}
inline int GetRegionCurrentResults(const PumiTally &tally, int32_t which, int32_t kind, double *out, int64_t n) {
  return pumitally_get_region_current_results(engine_of(tally), which, kind, out, n);
}

// Checkpoints (see pumitally_save_checkpoint in pumitally_c.h): SaveCheckpoint writes the tally state and the batch
// statistics to a file atomically; LoadCheckpoint restores them into an engine set up with the same configuration;
// MergeCheckpoint adds another run's folded batches.  No particle state is saved: after LoadCheckpoint, call
// CopyInitialPosition before the next move.  A refusal returns 1 and changes nothing.
inline int SaveCheckpoint(const PumiTally &tally, const char *path) {
  return pumitally_save_checkpoint(engine_of(tally), path);
}
inline int LoadCheckpoint(const PumiTally &tally, const char *path) {
  return pumitally_load_checkpoint(engine_of(tally), path);
}
inline int MergeCheckpoint(const PumiTally &tally, const char *path) {
  return pumitally_merge_checkpoint(engine_of(tally), path);
}

// Weight windows (see pumitally_set_weight_windows in pumitally_c.h): ngroups (lower, upper) pairs per element,
// [group][element] in the caller's numbering; lower <= 0 is no window, read back as (-1, -1).  GenerateWeightWindows
// makes them from the batch statistics of one result by the MAGIC method, the score bins as groups.
// WeightWindowsAtParticles gives the window of each particle's parent element (size = num_particles), WeightWindowsAtPoints
// the window at located points; groups may be nullptr (group 0).
inline int SetWeightWindows(const PumiTally &tally, const double *lower, const double *upper, int64_t n,
                            int32_t ngroups) {
  return pumitally_set_weight_windows(engine_of(tally), lower, upper, n, ngroups);
}
inline int GetWeightWindows(const PumiTally &tally, double *lower, double *upper, int64_t n) {
  return pumitally_get_weight_windows(engine_of(tally), lower, upper, n);
}
inline int GenerateWeightWindows(const PumiTally &tally, int32_t which, int32_t score, int32_t time_bin, double ratio,
                                 double max_rel_err) {
  return pumitally_generate_weight_windows(engine_of(tally), which, score, time_bin, ratio, max_rel_err);
}
inline int WeightWindowsAtParticles(const PumiTally &tally, const int32_t *groups, double *lower, double *upper,
                                    int32_t size) {
  return pumitally_get_weight_windows_at_particles(engine_of(tally), groups, lower, upper, size);
}
inline int WeightWindowsAtPoints(const PumiTally &tally, const double *xyz, int64_t npts, const int32_t *groups,
                                 double *lower, double *upper) {
  return pumitally_get_weight_windows_at_points(engine_of(tally), xyz, npts, groups, lower, upper);
}

// Mesh source (see pumitally_set_source in pumitally_c.h): strengths [group][element] in the caller's numbering, bias
// optional (nullptr), per_volume multiplies each by its element's volume.  SampleSource draws samples first .. first +
// n - 1 of seed (outputs may be nullptr); place != 0 (n == num_particles) puts sample j at particle j without a walk.
// GetSourceStrength gives Q, the unbiased total the caller normalises by.
inline int SetSource(const PumiTally &tally, const double *strength, const double *bias, int64_t n, int32_t ngroups,
                     int32_t per_volume) {
  return pumitally_set_source(engine_of(tally), strength, bias, n, ngroups, per_volume);
}
inline int32_t GetSourceGroups(const PumiTally &tally) { return pumitally_get_source_groups(engine_of(tally)); }
inline int GetSourceStrength(const PumiTally &tally, double *total) {
  return pumitally_get_source_strength(engine_of(tally), total);
}
inline int SampleSource(const PumiTally &tally, uint64_t seed, int64_t first, int64_t n, double *xyz, int32_t *elem,
                        int32_t *group, double *weight, int32_t place) {
  return pumitally_sample_source(engine_of(tally), seed, first, n, xyz, elem, group, weight, place);
}

}  // namespace pumitally

#endif  // PUMITALLY_PUMITALLYEXTRAS_H
