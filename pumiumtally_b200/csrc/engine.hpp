// Batch orchestration of the tally engine: owns the device-resident mesh
// tables, particle state, staging buffers, streams and the optional NCCL
// communicator.  Plays the role of the reference's PumiTallyImpl
// (reference: src/pumitally/PumiTallyImpl.h:154-221) minus everything Kokkos /
// pumi-pic / Omega_h.
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include <cuda_runtime.h>

#include "batch_stats.cuh"
#include "checkpoint.hpp"
#include "host_stage.hpp"
#include "source_sample.cuh"
#include "tet_mesh.hpp"
#include "walk_kernels.hpp"

namespace ptb {

struct EngineStats {
  uint64_t segments = 0, tracks = 0, relocations = 0, lost = 0, moves = 0;
  double kernel_ms = 0.0;
  double h2d_bytes = 0.0;
  uint64_t plane_fallbacks = 0;
};

// What a move tallies besides the track length, and the per-particle arrays that takes (nullptr: absent).
struct MoveTally {
  enum Kind { kPlain, kScored, kTimed };
  Kind kind = kPlain;                  // kPlain includes the binned moves
  const int32_t *bins = nullptr;       // [N] score bin per particle; counts only while the engine has several
  const double *responses = nullptr;   // [N * nscores] (scored; timed with one score: optional, every response 1)
  const double *times = nullptr;       // [N] time at the origin (timed)
  const double *speeds = nullptr;      // [N] (timed)
};

// One call of a move entry point: host or device pointers, as the entry point taking it says.
struct Move {
  const double *origin = nullptr, *dest = nullptr;
  int8_t *flying = nullptr;  // zeroed by a host move once consumed; a device move never writes it
  const double *weights = nullptr;
  int32_t size = 0;          // 3 * num_particles
  MoveTally tally;
};

class Engine {
 public:
  // Throws std::runtime_error when no CUDA device is usable: there is no CPU path.
  Engine(HostMesh &&mesh, int32_t num_particles, int device);
  ~Engine();
  Engine(const Engine &) = delete;
  Engine &operator=(const Engine &) = delete;

  int64_t num_elements() const { return mesh_.ntets; }
  int32_t num_particles() const { return n_; }
  const HostMesh &mesh() const { return mesh_; }

  // Host-pointer entry points (reference semantics; block until inputs are consumed).
  int copy_initial_position(const double *xyz, int32_t size);
  int move_to_next_location(const Move &m);
  // Device-pointer entry points (enqueue only).
  int copy_initial_position_device(const double *d_xyz, int32_t size, cudaStream_t stream);
  int move_to_next_location_device(const Move &m, cudaStream_t stream);

  // Score filter: nbins flux arrays; a move with bins tallies particle i into array bins[i] (outside
  // [0, nbins): the particle flies unscored).  Resets the tally.  Before comm_init on multi-GPU runs.
  int set_score_bins(int32_t nbins);
  int32_t score_bins() const { return nbins_; }
  // Scores: nscores responses per particle and move, tallied in one walk (walk_core.cuh, ScoreParams).  A scored
  // move adds l * w[i] * r[i*nscores + k] to score k of the particle's bin for every segment of length l.
  // Resets the tally; before comm_init.  With nscores > 1 only the scored and timed moves are accepted.
  int set_scores(int32_t nscores);
  int32_t scores() const { return nscores_; }
  // Time filter: edges T_0 < ... < T_nt (nt = nedges - 1, 1..kMaxTimeBins); a timed move splits every segment
  // between the time bins [T_j, T_j+1) it spans, by the time spent in each (walk_core.cuh, TimeParams).  edges ==
  // nullptr with nedges == 0 removes the filter.  Resets the tally; before comm_init.  While time bins are set only
  // the timed moves are accepted.
  int set_time_bins(const double *edges, int32_t nedges);
  int32_t time_bins() const { return ntime_; }
  // Linear flux moments (walk_core.cuh, moment_tally): order 1 makes every move also tally the first spatial moment
  // of every score, order 0 stops it.  Resets the tally; before comm_init.  Combines with bins, scores and time bins.
  int set_moments(int32_t order);
  int32_t moments() const { return moments_; }
  // n == 3E: time bin 0, bin 0, score 0; n == 3 * ntime * nbins * nscores * E: everything,
  // [time][bin][score][element][3].  m1 about each element's centroid (raw), or g = M^-1 m1 (normalised).
  int get_flux_moments(double *out, int64_t n);
  int get_flux_gradient(double *out, int64_t n);
  // Point queries (walk_core.cuh, locate_point).  locate: the element (caller's numbering) containing each of npts
  // points (AoS xyz), -1 outside the mesh or for a non-finite coordinate.  evaluate: every normalised result at each
  // point, [time][bin][score][point] (n == npts: time bin 0, bin 0, score 0; n == ntime * nbins * nscores * npts:
  // everything), get_normalized_flux's value of the element plus g . (x - c_e) with moments, NaN outside; out_elem may be
  // nullptr.  Host calls work through chunk-sized device buffers.  A query changes no particle, tally or statistic.
  int locate_points(const double *xyz, int64_t npts, int32_t *out_elem);
  int locate_points_device(const double *d_xyz, int64_t npts, int32_t *d_elem, cudaStream_t stream);  // enqueue only
  int evaluate_points(const double *xyz, int64_t npts, double *out, int64_t n, int32_t *out_elem);
  // Collision estimator (walk_core.cuh, collision_event): on == 1 adds a collision tally of the track-length tally's
  // configuration, in its own region of d_flux_.  Resets the tally; before comm_init.  Event i adds weights[i] *
  // responses[i * nscores + k] to score k of its element, bin bins[i] and time bin of times[i]; responses may be
  // nullptr with one score, bins nullptr (bin 0), times is required while time bins are set.  tally_collisions: events
  // at nevents points (AoS xyz), located as locate_points does; host calls work through chunk-sized buffers.
  // tally_collisions_at_particles: the particles i with collided[i] != 0, at their stored positions and elements
  // (n == num_particles).  Neither touches the particles, the track-length tally or the move statistics.
  int set_collision_estimator(int32_t on);
  int32_t collision_estimator() const { return collision_ ? 1 : 0; }
  int tally_collisions(const double *xyz, int64_t nevents, const double *weights, const double *responses,
                       const int32_t *bins, const double *times);
  int tally_collisions_device(const double *d_xyz, int64_t nevents, const double *d_weights, const double *d_responses,
                              const int32_t *d_bins, const double *d_times, cudaStream_t stream);  // enqueue only
  int tally_collisions_at_particles(const int8_t *collided, const double *weights, const double *responses,
                                    const int32_t *bins, const double *times, int32_t n);
  int tally_collisions_at_particles_device(const int8_t *d_collided, const double *d_weights, const double *d_responses,
                                           const int32_t *d_bins, const double *d_times, int32_t n, cudaStream_t stream);
  // kind 0 raw, 1 normalised, 2 first moments, 3 gradient: get_flux, get_normalized_flux, get_flux_moments and
  // get_flux_gradient of the collision tally (n as they take it)
  int get_collision_results(int32_t kind, double *out, int64_t n);
  // Face currents (walk_core.cuh, CurrentParams): on == 1 makes every move also tally the weight crossing each face,
  // per score bin and time bin, and the leakage through the hull; 0 stops it.  Resets the tally, discards the folded
  // batches; before comm_init.  Combines with everything else and changes none of its results.
  int set_face_currents(int32_t on);
  int32_t face_currents() const { return currents_ ? 1 : 0; }
  // Cosine bins of the face currents (walk_core.cuh, CurrentParams, MU): edges mu_0 < ... < mu_C in [0, 1] (C = nedges
  // - 1, 1..kMaxCosineBins) split every crossing by the cosine between its flight and the face normal; the current
  // results gain a cosine axis after the score-bin axis (C arrays where there was one).  edges == nullptr with nedges
  // == 0 removes them.  Resets the tally, discards the folded batches; before comm_init.  Takes effect while face
  // currents are on.
  int set_current_cosine_bins(const double *edges, int32_t nedges);
  int32_t current_cosine_bins() const { return nmu_; }
  // direction 0 outgoing, 1 incoming partial current of face f (opposite the caller's local vertex f) of every element;
  // kind 0 the open tally / the per-source divisor, 1 batch mean, 2 standard error, 3 relative error (neither divided
  // by an area or volume).  n == ntime * nbins * C * E * 4, [time][bin][cosine][element][face] in the caller's
  // numbering (C = 1 without cosine bins).
  int get_face_current_results(int32_t direction, int32_t kind, double *out, int64_t n);
  // the outgoing current summed over every hull face, kinds as above; n == ntime * nbins * C, [time][bin][cosine]
  int get_leakage(int32_t kind, double *out, int64_t n);
  // Point detectors (walk_core.cuh, detector_event): D = ndet detectors at xyz[3D] (AoS, each inside the mesh, or
// anywhere finite with the detector void on) with
  // exclusion radii r0[D] (finite, >= 0), 1 <= D <= kMaxDetectors; xyz == r0 == nullptr with ndet == 0 removes them.
  // Resets the tally, discards the folded batches; before comm_init.  Anything else is refused and changes nothing.
  int set_point_detectors(const double *xyz, int32_t ndet, const double *r0);
  int32_t point_detectors() const { return ndet_; }
  // Detector void (walk_core.cuh, detector_ray): on == 1 treats the space outside the mesh as a void the rays cross, so
  // detectors may lie anywhere, events outside the mesh are traced and rays re-enter across concave parts of the hull.
  // Setting the current mode changes nothing; switching resets the tally and discards the folded batches; switching
  // off while a detector lies outside the mesh is refused; before comm_init.
  int set_detector_void(int32_t on);
  int32_t detector_void() const { return det_void_ ? 1 : 0; }
  // Sigma_t [bin][element] in the caller's numbering, n == nbins * E, finite and >= 0; kept until set_score_bins changes
  // nbins.  Resets nothing.  Detector calls are refused without it.
  int set_detector_cross_sections(const double *sigma_t, int64_t n);
  // Next-event estimates of every (event, detector) ray into [time][bin][score][detector].  pdf[i * D + d] is the
  // angular density toward detector d per steradian (nullptr: 1 / (4 pi)); responses may be nullptr with one score, bins
  // nullptr (bin 0); times and speeds are required while time bins are set.  tally_detectors: events at nevents points,
  // located as locate_points does; host calls work through chunk-sized buffers.  tally_detectors_at_particles: the
  // particles i with flagged[i] != 0, at their stored positions and elements (n == num_particles).  Neither touches the
  // particles, any other tally or the move statistics.
  int tally_detectors(const double *xyz, int64_t nevents, const double *weights, const double *pdf,
                      const double *responses, const int32_t *bins, const double *times, const double *speeds);
  int tally_detectors_device(const double *d_xyz, int64_t nevents, const double *d_weights, const double *d_pdf,
                             const double *d_responses, const int32_t *d_bins, const double *d_times,
                             const double *d_speeds, cudaStream_t stream);  // enqueue only
  int tally_detectors_at_particles(const int8_t *flagged, const double *weights, const double *pdf,
                                   const double *responses, const int32_t *bins, const double *times,
                                   const double *speeds, int32_t n);
  int tally_detectors_at_particles_device(const int8_t *d_flagged, const double *d_weights, const double *d_pdf,
                                          const double *d_responses, const int32_t *d_bins, const double *d_times,
                                          const double *d_speeds, int32_t n, cudaStream_t stream);
  // kind 0 the open tally / the per-source divisor (the sum over ranks after an exchange), 1 batch mean, 2 standard
  // error, 3 relative error; n == ntime * nbins * nscores * D, [time][bin][score][detector].
  int get_detector_results(int32_t kind, double *out, int64_t n);
  // Batch statistics (batch_stats.cuh): on == 1 keeps a running mean and sum of squared deviations of every reported
  // double (both tallies), folded by end_batch from the batch's results divided by its source-normalisation divisor;
  // 0 frees them.  Resets the tally; before comm_init.  Any later set_* call discards the folded batches.
  int set_batch_statistics(int32_t on);
  // Collective with several ranks: the batch tally is reduce-scattered and each rank folds its share.  Then reset_tally.
  int end_batch();
  // tally 0 track length, 1 collision; kind 0 mean, 1 standard error (both / volume), 2 relative error, 3 gradient of
  // the mean (n as get_normalized_flux / get_flux_gradient take it).  Collective with several ranks.
  int get_batch_results(int32_t tally, int32_t kind, double *out, int64_t n);
  // Largest relative error of score `score` over the results with a nonzero mean, and their number (device reduction).
  int get_batch_max_rel_err(int32_t tally, int32_t score, double *out_max, int64_t *out_nonzero);
  // Region tallies (batch_stats.cuh, RegionPlan): region_of_element[n == E] in [-1, nregions) in the caller's numbering
  // (-1: in no region), 1 <= nregions <= E; nullptr with nregions == 0 removes the regions.  Resets the tally, discards
  // the folded batches; before comm_init.  Anything else is refused and changes nothing.
  int set_regions(const int32_t *region_of_element, int64_t n, int32_t nregions);
  int32_t regions() const { return nregions_; }
  int get_region_volumes(double *out, int64_t n);  // n == nregions
  // tally 0 track length, 1 collision; kind 0 the raw sum over each region, 1 sum / V_G / the per-source divisor;
  // [time][bin][score][region] (n == nregions: time bin 0, bin 0, score 0).  Collective with several ranks, as get_flux.
  int get_region_results(int32_t tally, int32_t kind, double *out, int64_t n);
  // kinds 0-2 of get_batch_results for the region sums, folded by end_batch while regions are set; not collective
  int get_region_batch_results(int32_t tally, int32_t kind, double *out, int64_t n);
  // Region currents (batch_stats.cuh, RegionCurrentPlan): on == 1 (regions set, face currents on, 4E <= INT32_MAX) also
  // reports the partial and net current of every ordered pair of adjacent regions (-1: no region, -2: outside the
  // mesh), summed from the face-current slots, with batch statistics folded next to the region sums.  Resets the
  // tally, discards the folded batches; before comm_init.  Anything else is refused and changes nothing.
  int set_region_currents(int32_t on);
  int32_t region_currents() const { return rc_on() ? 1 : 0; }
  int64_t region_current_pair_count() const { return int64_t(rc_plan_.from.size()); }
  int get_region_current_pairs(int32_t *from, int32_t *to, int64_t n);
  int get_region_current_areas(double *out, int64_t n);
  // which 0 partial, 1 net; kind 0 the open tally / the per-source divisor (collective as get_region_results), 1 batch
  // mean, 2 standard error, 3 relative error (not collective).  n == ntime * nbins * C * P, [time][bin][cosine][pair].
  int get_region_current_results(int32_t which, int32_t kind, double *out, int64_t n);
  // Checkpoints (checkpoint.hpp): the tally state -- the open batch, if anything was tallied since the last reset, and
  // the batch statistics (element and region) -- with a fingerprint of the configuration.  No particle state: after a
  // load the caller places the particles (CopyInitialPosition) before the next move.  Save changes nothing in the
  // engine and writes path + ".tmp", then renames it over path.  Load replaces the tally state after the same
  // configuration was set up (and comm_init, with several ranks); merge adds the file's folded batches to this
  // engine's (batch statistics on, no open batch in the file) and leaves the open batch alone.  Both refuse a
  // different fingerprint, a corrupt or truncated file, or too little device memory for a second copy of what they
  // read (up to 2 stats_len() + reported_len() doubles), and then change nothing.  Not collective.
  int save_checkpoint(const std::string &path);
  int load_checkpoint(const std::string &path);
  int merge_checkpoint(const std::string &path);
  // Weight windows (weight_windows.cuh): ngroups (lower, upper) pairs per element, not tally state (no reset, set_*,
  // end_batch, comm_init or checkpoint touches them).  set: host arrays [group][element] in the caller's numbering,
  // n == ngroups * E; lower <= 0 is no window, stored (-1, -1); any other entry must be finite with upper > lower, or the
  // call is refused and changes nothing.  lower == nullptr with ngroups == 0 removes them.  get: what set stored.
  int set_weight_windows(const double *lower, const double *upper, int64_t n, int32_t ngroups);
  int32_t weight_window_groups() const { return ww_groups_; }
  int get_weight_windows(double *lower, double *upper, int64_t n);
  // The MAGIC step over the batch statistics of (tally, score, time_bin), the score bins as groups: replaces the table.
  // Collective with several ranks (stats_view).
  int generate_weight_windows(int32_t tally, int32_t score, int32_t time_bin, double ratio, double max_rel_err);
  // The window of group groups[i] (nullptr: 0) in particle i's parent element (n == num_particles) or at point i (located
  // as locate_points does); (-1, -1) for a group outside [0, ngroups), an element without a window or a point outside.
  // Nothing changes.  Host calls work through chunk-sized device buffers; the device calls are enqueued only.
  int weight_windows_at_particles(const int32_t *groups, double *lower, double *upper, int32_t n);
  int weight_windows_at_particles_device(const int32_t *d_groups, double *d_lower, double *d_upper, int32_t n,
                                         cudaStream_t stream);
  int weight_windows_at_points(const double *xyz, int64_t npts, const int32_t *groups, double *lower, double *upper);
  int weight_windows_at_points_device(const double *d_xyz, int64_t npts, const int32_t *d_groups, double *d_lower,
                                      double *d_upper, cudaStream_t stream);
  // Mesh source (source_sample.cuh): strength [group][element] in the caller's numbering (n == ngroups * E), times
  // each element's volume with per_volume, times bias [same layout] when bias != nullptr, sampled by a CDF over the
  // entries.  Not tally state (no reset, set_*, end_batch, comm_init or checkpoint touches it).  A negative or
  // non-finite strength or bias, a zero bias where the strength is > 0, or a zero or non-finite total is refused and
  // changes nothing; strength == nullptr with ngroups == 0 removes the source.
  int set_source(const double *strength, const double *bias, int64_t n, int32_t ngroups, int32_t per_volume);
  int32_t source_groups() const { return src_groups_; }
  int get_source_strength(double *total);  // Q: the sum of the unbiased strengths (times the volumes with per_volume)
  // Samples first .. first + n - 1 of `seed`: AoS xyz, element (caller's numbering), group and birth weight, each
  // optional.  place != 0 (n == num_particles) makes sample j particle j's position and parent element, without a walk,
  // as the initial placement.  Without place nothing in the engine changes.  The host call works through chunk-sized
  // device buffers and synchronises; the device call is enqueued behind the last work on the particle state.
  int sample_source(uint64_t seed, int64_t first, int64_t n, double *xyz, int32_t *elem, int32_t *group,
                    double *weight, int32_t place);
  int sample_source_device(uint64_t seed, int64_t first, int64_t n, double *d_xyz, int32_t *d_elem, int32_t *d_group,
                           double *d_weight, int32_t place, cudaStream_t stream);
  // n == E: time bin 0, bin 0, score 0; n == ntime * nbins * nscores * E: everything, [time][bin][score][element]
  int get_flux(double *out, int64_t n);
  // Device-side accessors, caller's element numbering, enqueued on `stream` (no synchronisation).
  int set_state_device(const double *d_xyz, const int32_t *d_elem, int32_t first, int32_t count, cudaStream_t stream);
  int get_state_device(double *d_xyz, int32_t *d_elem, int32_t first, int32_t count, cudaStream_t stream);
  int get_flux_device(double *d_out, cudaStream_t stream);
  int get_normalized_flux(double *out_flux, double *out_volume, int64_t n);
  int get_element_ids(int32_t *out, int64_t n);
  int get_positions(double *out, int64_t n3);
  int reset_tally();
  // Per-source normalisation of the *normalised* flux (get_normalized_flux, WriteTallyResults); the raw
  // flux is never touched.  0 = none (reference behaviour: flux / volume, PumiTallyImpl.cpp:402),
  // 1 = also divide by the number of particles (what PumiTally.h:93 documents), 2 = by `value`
  // (a total source weight the caller knows), 3 = by the total weight of the first tracks after
  // CopyInitialPosition / reset_tally (the reference's total_initial_weight, PumiTallyImpl.h:170-171).
  int set_source_normalization(int mode, double value);
  double source_normalization();  // the divisor currently in effect (1 for mode 0)
  int get_stats(EngineStats *out);
  int synchronize();
  double *flux_device_ptr() { return gather_shares() ? nullptr : flux_view(); }
  int set_option(const std::string &name, int64_t value);
  int64_t get_option(const std::string &name) const;
  void set_output_name(const std::string &s) { output_name_ = s; }
  int write_tally_results();
  int64_t debug_order(int32_t *out, int64_t n);

  // multi-GPU exchange step
  int comm_init(int rank, int nranks, const uint8_t id[128]);
  int allreduce_tally();
  // The cheaper batch-end exchange: every rank ends up with the sum over ranks of ITS share of the
  // elements only (ncclReduceScatter: half the traffic of the all-reduce); the shares are gathered
  // (ncclAllGather, collective) the first time a flux accessor or WriteTallyResults needs the whole array.
  int reduce_tally_to_owners();
  // whichever of the two comm_init measured to be quicker on this mesh (same choice on every rank)
  int exchange_tally();

 private:
  // t: the move's tally with device arrays (bins only with several score bins); the default is a plain move
  int launch_range(const double *d_origin, const double *d_dest, const int8_t *d_flying,
                   const double *d_weights, int32_t begin, int32_t end, cudaStream_t stream,
                   const MoveTally &t = {});
  int move_host(const double *origin, const double *dest, int8_t *flying, const double *weights, int32_t size,
                const MoveTally &dev, int32_t chunk);
  // slice: doubles between time bins of d_flux; variant, tag: the kernel and its auto-tuner slot (-1: none)
  // d_cur, cur_slice: the face currents of the score bin and the doubles between their time bins (read with currents);
  // mu_stride: the doubles between their cosine bins (0: every cosine bin into one array)
  int launch_range_into(double *d_flux, const double *d_origin, const double *d_dest, const int8_t *d_flying,
                        const double *d_weights, int32_t begin, int32_t end, cudaStream_t stream, const MoveTally &t,
                        int64_t slice, int variant, int tag, double *d_cur = nullptr, int64_t cur_slice = 0,
                        int64_t mu_stride = 0);
  // scored and timed moves, and every move with moments or face currents: a tallied walk kernel, never one of the
  // auto-tuner's samples
  bool scored_move(const MoveTally &t) const { return t.kind != MoveTally::kPlain || moments_ > 0 || currents_; }
  bool move_refused(const Move &m, bool device) const;  // with a message; checked before anything is uploaded
  // L2 partition of every SM (l2_partitions.cu), probed when option die_split is switched on; die0_sms_ == 0: no usable map
  uint32_t die_mask_[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  int die0_sms_ = 0, nsms_ = 0;
  bool die_split_ = false;
  int32_t nbins_ = 1;
  int32_t nscores_ = 1, stride_ = 1;  // scores, and doubles per element of d_flux_ (score_stride(nscores_), times
                                      // kMomentSlots with moments)
  int32_t ntime_ = 0;                 // time bins (0: no time filter)
  int32_t moments_ = 0;               // moment order (0: none, 1: linear; walk_core.cuh, moment_tally)
  bool collision_ = false;            // the collision tally follows the track-length one in d_flux_
  bool currents_ = false;             // face currents and leakage follow both tallies in d_flux_
  int32_t nmu_ = 0;                   // cosine bins of the face currents (0: none)
  size_t flux_alloc_ = 0;             // doubles allocated at d_flux_
  // d_flux_: the track-length tally [time][bin][element][stride_] (flux_len()), with the collision estimator the
  // collision tally of the same layout, then the unreported array of a binned move's unmatched particles and padding
  size_t nslices() const { return ntime_ > 0 ? size_t(ntime_) : 1; }
  size_t flux_len() const { return nslices() * size_t(nbins_) * size_t(mesh_.ntets) * size_t(stride_); }
  // With face currents the reported part goes on: the current slots [time][bin][cosine][element][4] (walk_core.cuh,
  // CurrentParams) from current_base(), then one leakage slot per [time][bin][cosine], filled by end_batch.  The
  // (time, bin) arrays of the tallies stay result_arrays(); the currents have cur_arrays() = C times as many.
  size_t current_base() const { return flux_len() * (collision_ ? 2 : 1); }
  size_t ncos() const { return nmu_ > 0 ? size_t(nmu_) : 1; }
  int32_t cur_arrays() const { return result_arrays() * int32_t(ncos()); }  // [time][bin][cosine] arrays of 4E doubles
  size_t current_len() const { return size_t(cur_arrays()) * size_t(mesh_.ntets) * 4; }
  size_t leak_base() const { return current_base() + current_len(); }
  size_t reported_len_for(bool currents) const {
    return current_base() + (currents ? current_len() + size_t(cur_arrays()) : 0);
  }
  size_t reported_len() const { return reported_len_for(currents_); }  // what the exchange moves
  size_t bin_len() const { return size_t(mesh_.ntets) * size_t(stride_); }
  int32_t result_arrays() const { return int32_t(nslices()) * nbins_; }  // (time, bin) arrays of bin_len() doubles
  // results laid out [time][bin][score][element] (and read through the score-stride kernels)
  bool multi_results() const { return nscores_ > 1 || ntime_ > 0 || moments_ > 0; }
  int resize_flux(int32_t nbins, int32_t nscores, int32_t ntime, int32_t moments, bool collision, bool currents,
                  int32_t nmu);
  // base: doubles from d_flux_ (or the exchanged array) to the tally read, 0 (track length) or flux_len() (collision)
  // [time][bin][score][element][3]; src != nullptr: the records at src + base, gradients not divided by a source divisor
  int copy_moments(std::vector<double> &out, bool gradient, size_t base = 0, const double *src = nullptr);
  int get_moments_entry(double *out, int64_t n, bool gradient, size_t base = 0);
  bool per_source_divisor(double *out);  // of the normalised results; false, with a message, while there is none
  int copy_results(std::vector<double> &out, bool normalized, size_t base = 0);
  // ---- point queries (locate_kernels.cu) ----
  LocateParams locate_params() const;
  int ensure_candidates();  // non-convex hull: the cells' candidate lists, built and uploaded at the first query
  int64_t *d_cand_off_ = nullptr;
  int32_t *d_cand_ = nullptr;
  size_t cand_entries_ = 0;
  bool candidates_ready_ = false;
  // The query, event and sampling calls: each has a setup its host and device forms share (refusal, device, lazy tables,
  // `arena` bytes for the host form, stream order, flags; 1 refused or failed, -1 nothing to enqueue, 0 go on) and an
  // enqueue of its kernels from device pointers, which the host form runs through staged().
  int locate_setup(const double *xyz, int64_t npts, const int32_t *elem, size_t arena);
  cudaError_t enqueue_locate(const double *xyz, int64_t npts, int32_t *elem, cudaStream_t stream);
  // n items in chunks of min(chunk_, n) through the arena (Staged arrays, engine.cu): setup(arena bytes), then per chunk
  // the uploads, enqueue(first item, count, device arrays...) and the copies back on compute_; one sync at the end
  template <class Setup, class Enqueue, class... A> int staged(int64_t n, Setup &&setup, Enqueue &&enqueue, A... a);
  void *d_arena_ = nullptr;  // grow-only device scratch of the host forms, carved into 256-byte aligned slices
  size_t arena_bytes_ = 0;
  int ensure_arena(size_t bytes);
  // evaluation table, internal element order: vals [R][E] normalised results, with moments grads [R][E][3] (the
  // normalised gradient) and cen [E][3] (vertex-average centroids); valid until the next move, reset, exchange or change
  // of the source normalisation or of the configuration
  bool eval_valid_ = false;
  double *d_eval_vals_ = nullptr, *d_eval_grads_ = nullptr, *d_eval_cen_ = nullptr;
  int build_eval_table();
  // named cell arrays of the VTK output; data owns them (a moved vector keeps its storage)
  struct VtkArrays {
    std::vector<std::vector<double>> data;
    std::vector<std::pair<std::string, const double *>> named;
    std::vector<int> ncomp;
  };
  // The arrays write_scored_results writes for the tally at `base`, every name prefixed.  main != nullptr: the sum of
  // score 0 over the bins and time bins is returned there instead of being named prefix + "flux".
  int scored_arrays(size_t base, const std::string &prefix, VtkArrays &a, std::vector<double> *main);
  int write_scored_results(VtkArrays &a);  // everything, [time][bin][score][element], caller's order
  // ---- collision estimator (locate_kernels.cu) ----
  CollisionParams collision_params() const;
  bool collision_refused(const double *responses, const double *times) const;  // with a message
  int follow_last_stream(cudaStream_t stream);  // order work on the particle state behind the last such work
  unsigned long long *d_coll_counts_ = nullptr;  // [3] events tallied, outside the mesh, rejected since the last reset
  int collide_located_setup(const double *xyz, int64_t n, const double *w, const double *r, const double *t,
                            size_t arena);
  cudaError_t enqueue_collide_located(const double *xyz, int64_t n, const double *w, const double *r,
                                      const int32_t *bins, const double *t, cudaStream_t stream);
  int collide_particles_setup(const int8_t *collided, const double *w, const double *r, const double *t, int32_t n,
                              size_t arena, cudaStream_t stream);
  cudaError_t enqueue_collide_particles(int32_t first, int32_t n, const int8_t *collided, const double *w,
                                        const double *r, const int32_t *bins, const double *t, cudaStream_t stream);
  // ---- point detectors (detector_kernels.cu) ----
  int32_t ndet_ = 0;                               // 0: no detectors
  std::vector<double> det_xyz_, det_r0_;           // as set_point_detectors took them
  std::vector<int32_t> det_elem_;                  // internal element of each detector
  double *d_det_pos_ = nullptr, *d_det_r0_ = nullptr;
  double *d_sigma_ = nullptr;                      // [nbins][E] internal order; nullptr: no table
  int32_t sigma_bins_ = 0;                         // nbins of the table
  uint32_t sigma_crc_ = 0;                         // CRC-32 of the table as uploaded
  // [2 * det_len()]: the open tally and the sum over ranks of the last exchange; then, with batch statistics,
  // [2 * det_len()]: the batch mean and M2
  double *d_det_ = nullptr;
  bool det_global_valid_ = false;                  // the second block holds the exchanged sum of the first
  unsigned long long *d_det_counts_ = nullptr;     // [kDetCountersVoid] since the last reset
  bool det_void_ = false;                          // the detector void (set_detector_void)
  // the hull grid of the detector void: hull-tet lists of the seed-grid cells, uploaded at the mode's first use
  HullGrid hull_{};
  int64_t *d_hull_off_ = nullptr;
  int32_t *d_hull_tets_ = nullptr;
  size_t hull_entries_ = 0;                        // entries of the hull-tet lists
  bool hull_ready_ = false;
  int ensure_hull_grid();
  const HullGrid *hull_grid_params() const { return det_void_ ? &hull_ : nullptr; }  // nullptr: the mode is off
  size_t det_len() const { return nslices() * size_t(nbins_) * size_t(nscores_) * size_t(ndet_); }
  int alloc_detectors(size_t len, bool stats, double **out);  // len doubles per block, zeroed; nothing changes on failure
  DetectorParams detector_params() const;
  bool detector_refused(const double *responses, const double *times, const double *speeds) const;  // with a message
  int detect_located_setup(const double *xyz, int64_t n, const double *w, const double *r, const double *t,
                           const double *v, size_t arena);
  cudaError_t enqueue_detect_located(const double *xyz, int64_t n, const double *w, const double *pdf, const double *r,
                                     const int32_t *bins, const double *t, const double *v, cudaStream_t stream);
  int detect_particles_setup(const int8_t *flagged, const double *w, const double *r, const double *t, const double *v,
                             int32_t n, size_t arena, cudaStream_t stream);
  int exchange_detectors();  // the detector block summed over the ranks into its second block (collective)
  // ---- batch statistics (stats_kernels.cu) ----
  bool batch_stats_ = false;
  int64_t batches_ = 0;                            // batches folded
  double *d_mean_ = nullptr, *d_m2_ = nullptr;     // [stats_len()] running mean and sum of squared deviations
  double *d_batch_div_ = nullptr;                  // [2] divisor of the batch being folded, scratch of the exchange
  unsigned long long *d_stats_red_ = nullptr;      // [2] result of the max-relative-error reduction
  bool sharded() const { return nccl_comm_ && nranks_ > 1; }
  // entries this rank keeps: the whole reported tally, or its share of it after comm_init with several ranks
  size_t stats_len() const { return sharded() ? share_ : reported_len(); }
  int alloc_stats(size_t len);  // zeroed, batches_ = 0; nothing changes when the allocation fails
  void free_stats();
  // the statistics of the whole reported tally: this rank's, or gathered from every rank's share into *tmp (collective,
  // the caller frees *tmp)
  int stats_view(const double **mean, const double **m2, double **tmp);
  // [time][bin][score][element] of tally `tally`, kinds 0-2 of get_batch_results, caller's numbering
  int copy_batch_results(std::vector<double> &out, int32_t tally, int32_t kind);
  bool batch_refused(int32_t tally, int32_t kind) const;  // with a message
  // the "<name>_mean" / "<name>_rel_err" arrays of the tally at `tally`, names prefixed
  int batch_arrays(int32_t tally, const std::string &prefix, VtkArrays &a);
  // ---- region tallies (stats_kernels.cu, launch_region_sums) ----
  int32_t nregions_ = 0;                           // 0: no regions
  std::vector<RegionLevel> region_levels_;         // of the plan set_regions built
  std::vector<double> region_volume_;              // [nregions_], summed in the plan's order
  std::vector<int32_t> region_of_internal_;        // [E] the map set_regions took, internal order (the pair plan's)
  int32_t *d_region_elems_ = nullptr, *d_region_starts_ = nullptr;  // the plan's elems and starts
  int32_t *d_region_ident_ = nullptr;              // [nregions_] 0, 1, ...: the readout's order map
  double *d_region_volume_ = nullptr;              // [nregions_]
  double *d_region_work_ = nullptr;                // scratch of launch_region_sums, then one tally's region sums
  int64_t region_scratch_ = 0;                     // doubles of that scratch
  size_t region_work_len_ = 0;                     // doubles at d_region_work_
  double *d_region_stats_ = nullptr;               // [3 * region_len()]: the batch's sums, running mean, M2
  // region results of every reported tally: [tally][time][bin][region][score], then with region currents the partials
  // and the nets [time][bin][cosine][pair] from rc_base()
  size_t rc_base() const { return (collision_ ? 2 : 1) * size_t(result_arrays()) * size_t(nregions_) * size_t(nscores_); }
  size_t region_len_for(bool rcur) const {
    return rc_base() + (rcur ? 2 * size_t(cur_arrays()) * rc_plan_.from.size() : 0);
  }
  size_t region_len() const { return region_len_for(rc_on()); }
  void free_regions();
  int ensure_region_work();   // d_region_work_ for the current layout
  int ensure_region_stats();  // d_region_stats_ (zeroed when allocated: it is freed whenever the batches are discarded)
  // the region sums of `narrays` result arrays from `flux` (the arrays of one or both tallies) into out, on compute_
  int region_sums(const double *flux, int64_t narrays, double *out);
  bool region_refused(int32_t tally, int32_t kind, int32_t max_kind, int64_t n) const;  // with a message
  uint64_t region_hash_ = 0;                       // of the map set_regions took (caller's numbering), 0 without
  // ---- region currents (stats_kernels.cu, launch_region_sums / launch_region_net) ----
  RegionCurrentPlan rc_plan_;                      // empty while region currents are off
  int32_t *d_rc_slots_ = nullptr, *d_rc_starts_ = nullptr, *d_rc_rev_ = nullptr;  // the plan's slots, starts and rev
  int32_t *d_rc_ident_ = nullptr;                  // [P] 0, 1, ...: the readout's order map
  double *d_rc_ones_ = nullptr;                    // [P] 1.0: the readout's volumes
  bool rc_on() const { return !rc_plan_.from.empty(); }
  void free_region_currents();
  // the plan of region_of_internal on the device into *fresh (nothing changes in the engine), with a message on failure
  int build_region_currents(const int32_t *region_of_internal, RegionCurrentPlan *plan, int32_t *dev[4], double **ones);
  void install_region_currents(RegionCurrentPlan &&plan, int32_t *dev[4], double *ones);
  // partials then nets of the R current arrays at cur (R * 4E doubles) into out[2 R P], on compute_
  int region_current_sums(const double *cur, double *out);
  // ---- checkpoints (checkpoint.hpp) ----
  bool tallied_ = false;  // a move, collision or localisation since the last reset: a checkpoint holds the open batch
  bool mesh_hashed_ = false;
  uint64_t mesh_hash_ = 0, order_hash_ = 0;  // coordinates and t2v (caller's numbering); orig_of_internal
  ckpt::Fingerprint fingerprint();
  // load (merge == false) or merge the checkpoint at path, with a message on refusal
  int read_checkpoint(const std::string &path, bool merge);
  // ---- face currents (stats_kernels.cu, launch_current_readout / launch_leakage) ----
  // [4E] per internal element and face: 4 * neighbour + back, kNoFace on the hull; the hull slots 4 e + f, ascending
  // (30-bit element ids: every slot index fits 32 bits).  Built and uploaded at the first use.
  uint32_t *d_face_opp_ = nullptr, *d_hull_slots_ = nullptr;
  int64_t nhull_ = 0;
  int ensure_face_maps();
  // leakage of the R = result_arrays() current arrays at cur (R * 4E doubles) into out[R], on compute_
  int leakage_sums(const double *cur, double *out);
  // the "current_out" / "current_in" arrays (4 components, summed over time and score bins, per source)
  int current_arrays(VtkArrays &a);
  // ---- weight windows (ww_kernels.cu) ----
  int32_t ww_groups_ = 0;     // 0: no windows
  double2 *d_ww_ = nullptr;   // [ww_groups_][internal element] (lower, upper), (-1, -1) where there is none
  void free_weight_windows();
  int alloc_weight_windows(int32_t ngroups, double2 **out);  // 16 ngroups E bytes; nothing changes when it fails
  int ww_particles_setup(int32_t n, const double *lower, const double *upper, size_t arena, cudaStream_t stream);
  cudaError_t enqueue_ww_particles(int32_t first, int32_t n, const int32_t *groups, double *lower, double *upper,
                                   cudaStream_t stream);
  int ww_points_setup(const double *xyz, int64_t npts, const double *lower, const double *upper, size_t arena);
  cudaError_t enqueue_ww_points(const double *xyz, int64_t npts, const int32_t *groups, double *lower, double *upper,
                                cudaStream_t stream);
  // the "ww_lower" / "ww_upper" arrays (with several groups "_g<g>" after each name), caller's numbering
  int ww_arrays(VtkArrays &a);
  // ---- mesh source (source_kernels.cu) ----
  int32_t src_groups_ = 0;                 // 0: no source
  double *d_src_cdf_ = nullptr;            // [ngroups * E] C[k], caller's numbering
  double *d_src_bias_ = nullptr;           // [ngroups * E] b[k], nullptr without bias
  double *d_src_verts_ = nullptr;          // [E][4][3] vertices in the caller's numbering and local order (first use)
  double src_total_ = 0.0, src_strength_ = 0.0;  // T and Q
  int64_t src_last_ = -1;                  // the last entry with p > 0
  std::vector<double> src_given_;          // the strengths as the caller gave them (VTK "source")
  void free_source();
  SourceTable source_table() const;
  int source_setup(int64_t first, int64_t n, bool outputs, int32_t place, size_t arena, cudaStream_t stream);
  // samples first + b .. first + b + n - 1, with place into particles b .. b + n - 1
  cudaError_t enqueue_source(uint64_t seed, int64_t first, int64_t b, int64_t n, double *xyz, int32_t *elem,
                             int32_t *group, double *weight, bool place, cudaStream_t stream);
  int source_arrays(VtkArrays &a);  // "source" (with several groups "source_g<g>"), caller's numbering
  // per-particle side arrays of a host-pointer move on their way to the device (upload_aux)
  struct AuxUpload {
    void *d = nullptr;    // device copy
    void *h = nullptr;    // pinned copy of pageable caller arrays
    size_t cap = 0;       // bytes allocated at d / h
    cudaEvent_t ev = nullptr;
  };
  int upload_aux(AuxUpload &u, const void *a, const void *b, size_t bytes);
  void pool_copy(void *dst, const void *src, size_t bytes);  // on the staging workers once they exist
  AuxUpload time_up_;                 // [2N] times, then speeds, of a host-pointer timed move
  AuxUpload resp_up_;                 // [N * nscores_] responses of a host-pointer scored or timed move
  AuxUpload bins_up_;                 // [N] bins of a host-pointer move
  double *d_edges_ = nullptr;         // [ntime_ + 1] time bin edges
  double *d_mu_edges_ = nullptr;      // [nmu_ + 1] cosine bin edges
  std::vector<double> mu_edges_;      // the same on the host (checkpoint fingerprint)
  uint64_t scored_moves_ = 0;         // scored_move() moves since the last reset (not the auto-tuner's samples)
  int8_t *d_mask_ = nullptr;          // [N] flying flags of one bin
  bool host_is_pinned(const void *p) const;
  void maybe_register(const void *p, size_t bytes);
  void collect_timers(bool wait);
  void build_seed_grid();
  bool upload_compact();

  HostMesh mesh_;
  int32_t n_ = 0;
  int device_ = 0;
  bool initialized_ = false;  // is_pumipic_initialized (PumiTallyImpl.h:168)
  uint64_t moves_ = 0;        // iter_count (PumiTallyImpl.h:169)
  std::string output_name_ = "fluxresult.vtk";

  // options
  int variant_ = kVariantPersistRefill8;  // chosen in the constructor from mesh size vs L2 (choose_variant)
  int choose_variant() const;
  // Auto-tuner (only while the engine picks the kernel itself and the mesh is in the streaming regime):
  // whether processing the particles in spatial order pays depends on the particle data (it does for
  // collimated long tracks, config c4; it ties for isotropic ones), so the first four moves of every
  // kTuneEpoch alternate between the streaming kernel and the packed/sorted one, and the rest of the
  // epoch uses whichever had the lower kernel time.
  static constexpr uint64_t kTuneEpoch = 64;
  bool auto_variant_ = true, autotune_ = true;
  int tuned_variant_ = kVariantPersistRefill8;
  int move_variant_ = kVariantPersistRefill8, move_tag_ = -1;
  double explore_ms_[2] = {0.0, 0.0};
  int explore_pending_ = 0;
  bool explore_complete_ = false;
  uint64_t launches_ = 0;  // kernels launched by the move / localisation entry points
  void begin_move(bool scored);
  int block_ = 128;
  bool chunk_user_set_ = false;
  int32_t chunk_ = 1 << 19;  // particles per H2D/compute pipeline stage (a host move may raise its own, unless user-set)
  // Seed grid for relocation / localisation.  The reference walks straight from the particle's old
  // position to the new one and stops at the hull if that segment leaves the mesh -- on a mesh with
  // concavities or voids even when the new position is inside.  Starting from a seed cell instead
  // reaches it, which is a different (better, but different) answer, so by default the shortcut is
  // used only when the hull is convex (seed_grid_mode_ 1); 0 = never, 2 = always.
  bool use_seed_grid_ = true;
  int seed_grid_mode_ = 1;
  int32_t max_iters_ = 0;  // crossing limit per walk; 0 = ntets + 16
  bool morton_ = true;    // binning key: Morton rank of the cell (matches the tet storage order) instead of its z-major index
  int claim_run_ = 4;     // chunks per ticket in gather mode
  bool bin_midpoint_ = false;  // binning key: cell of the track's midpoint instead of its start (experiment, c5)

  // device memory
  TetRecord *d_tets_ = nullptr;
  TetLinks *d_links_ = nullptr;    // compact layout (walk_compact.cuh); null when the mesh exceeds its id ranges
  VertexRec *d_verts_ = nullptr;
  TetStart *d_starts_ = nullptr;
  double *d_flux_ = nullptr, *d_volume_ = nullptr, *d_scratch_ = nullptr;
  int norm_mode_ = 0;
  double norm_value_ = 1.0;
  double *d_initial_weight_ = nullptr;  // total weight of the first tracks of the batch
  bool initial_weight_pending_ = true;  // the next move is the batch's first
  ParticleState *d_state_ = nullptr;  // persistent position + parent element, 32 B per particle
  double *d_origin_ = nullptr, *d_dest_ = nullptr, *d_weights_ = nullptr;  // staging
  int8_t *d_flying_ = nullptr;
  DeviceStats *d_stats_ = nullptr;
  unsigned int *d_tickets_ = nullptr;  // ring of chunk counters for the persistent kernel
  unsigned ticket_next_ = 0;
  SeedGrid grid_{};              // relocation seed grid (grid_.cell_tet lives in d_grid_)
  int32_t *d_grid_ = nullptr;
  int32_t *d_orig_of_internal_ = nullptr, *d_internal_of_orig_ = nullptr;  // element renumbering maps (device accessors)
  int ensure_element_maps();
  int32_t *d_cell_rank_ = nullptr;
  // spatial binning of the flying particles (gather-mode kernels)
  int32_t *d_pcell_ = nullptr, *d_order_ = nullptr;
  PackedRow *d_rows_ = nullptr;  // packed variant: one 64-byte row per flying particle, allocated at first use
  unsigned int *last_work_count_ = nullptr;
  unsigned int *d_cell_count_ = nullptr, *d_cell_sums_ = nullptr, *d_work_count_ = nullptr;

  cudaStream_t compute_ = nullptr, copy_ = nullptr;
  cudaStream_t last_stream_ = nullptr;  // stream of the previous kernel launch that touched the particle state
  bool last_stream_set_ = false;
  cudaEvent_t ev_order_ = nullptr;
  struct TimerPair { cudaEvent_t a, b; int tag; };  // tag: auto-tuner slot the time belongs to, -1 = none
  std::vector<TimerPair> timers_free_, timers_busy_;
  std::vector<cudaEvent_t> chunk_events_;
  // caller buffers pinned with cudaHostRegister (option "register_host"): base -> bytes
  std::vector<std::pair<const void *, size_t>> registered_;
  bool register_host_ = false;
  double kernel_ms_ = 0.0, h2d_bytes_ = 0.0;

  // Host-pointer path, staged (host_stage.hpp): pinned per-particle slots for dest / weight / flying
  // that are both the DMA source of a move and the mirror the next move's origins are compared
  // against; only origins that changed travel, as a patch list applied to the device's copy of the
  // previous destinations.  Invariant between moves (mirror_valid_): h_dest_ == the device array
  // d_dest_, bit for bit.
  int host_path_ = 2;                 // 2 automatic (default), 1 staged, 0 direct copies from the caller's arrays
  uint64_t host_moves_ = 0;           // host-pointer moves so far (schedule of the staged-vs-direct probe)
  double span_ms_[2] = {0.0, 0.0};    // upload span per path: [0] staged, [1] direct
  int span_n_[2] = {0, 0};
  int span_tag_ = -1;                 // path of the move whose span has not been collected yet
  int span_choice_ = -1;              // this epoch's decision: 0 staged, 1 direct, -1 still probing
  void collect_upload_span();
  int mark_move_done();
  cudaEvent_t ev_done_ = nullptr;     // after the last kernel of the latest host move
  int host_threads_ = 0;              // 0 = default_host_threads() - 1
  std::unique_ptr<HostStager> stager_;  // worker pool + per-chunk stage pass
  void *stage_base_ = nullptr;
  double *h_dest_ = nullptr, *h_w_ = nullptr;
  int8_t *h_fly_ = nullptr;
  bool stage_ready_ = false, stage_failed_ = false, stage_registered_ = false;
  bool mirror_valid_ = false;
  int32_t staged_chunk_ = 0;          // chunking of the last staged move (its chunk_events_ are still meaningful)
  int staged_chunks_ = 0;
  PatchEntry *h_patch_ = nullptr;     // pinned ring of kPatchSlots chunk-sized lists
  PatchEntry *d_patch_ = nullptr;     // one list per chunk of a move
  size_t patch_cap_ = 0;              // entries per chunk
  int patch_chunks_ = 0;              // lists d_patch_ has room for
  double stage_host_s_ = 0.0, stage_sent_bytes_ = 0.0;
  cudaEvent_t ev_copy0_ = nullptr, ev_copy1_ = nullptr;  // span of the last staged move's uploads
  int pool_node_ = -1;
  int ensure_stage_buffers(const void *caller_mem, size_t caller_bytes);
  void follow_caller_memory(const void *p, size_t bytes);
  int ensure_patch_buffers(int nchunks, int32_t chunk);
  int move_direct(const double *origin, const double *dest, int8_t *flying, const double *weights, int nchunks,
                  const MoveTally &dev, int32_t chunk);
  // Page-locked caller arrays (pinned by the caller, or by option register_host): see move_pinned().
  // Off by default: the positions travelling back (24 B per particle, device->host) can slow the uploads
  // down more than the saved host work buys.
  bool pinned_path_ = false;
  double *h_pos_ = nullptr;            // pinned mirror of the device's particle positions [3N]
  bool pos_mirror_valid_ = false;
  cudaStream_t d2h_ = nullptr;
  std::vector<cudaEvent_t> pos_events_, walk_events_;  // per chunk: positions back on the host / walk + export done
  double d2h_bytes_ = 0.0;
  int ensure_position_mirror(int nchunks);
  int move_pinned(const double *origin, const double *dest, int8_t *flying, const double *weights, int nchunks,
                  int32_t chunk);
  int relocate_patches(const PatchEntry *d_list, int32_t count, cudaStream_t stream);

  // NCCL (resolved with dlopen at comm_init time)
  void *nccl_comm_ = nullptr;
  int rank_ = 0, nranks_ = 1;
  // Result of the last batch-end exchange.  This rank's own tally keeps accumulating in d_flux_
  // across moves (reference semantics: raw flux summed over all moves); the exchange writes the
  // sum over ranks here, so it can be repeated after every batch without counting earlier batches
  // twice.  The accessors return this array until the next move or reset changes the local tally.
  double *d_flux_global_ = nullptr;
  bool flux_global_valid_ = false;
  int exchange_choice_ = 0;           // 0 all-reduce, 1 reduce-scatter to owners
  double exchange_ms_[2] = {0, 0};    // comm_init's measurement of both (mean over ranks)
  bool flux_owned_only_ = false;  // d_flux_global_ holds only this rank's share (after reduce_tally_to_owners)
  size_t share_ = 0;              // elements per rank in the scattered layout = ceil(E / nranks)
  int gather_shares();
  double *flux_view() { return flux_global_valid_ ? d_flux_global_ : d_flux_; }
  double allreduce_ms_ = 0.0;  // device time of the last exchange
  cudaEvent_t ev_ar0_ = nullptr, ev_ar1_ = nullptr;
};

// NCCL entry points resolved with dlopen at run time (nccl_dl.cpp)
int nccl_get_unique_id(uint8_t out[128]);
int nccl_comm_init_rank(void **comm, int nranks, const uint8_t id[128], int rank);
int nccl_allreduce_sum_f64(void *comm, const double *send, double *recv, size_t count, cudaStream_t stream);
int nccl_reduce_scatter_sum_f64(void *comm, const double *send, double *recv, size_t count, cudaStream_t stream);
int nccl_all_gather_f64(void *comm, const double *send, double *recv, size_t count, cudaStream_t stream);
void nccl_comm_destroy(void *comm);

}  // namespace ptb
