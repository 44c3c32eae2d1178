// extern "C" layer of libpumitally.so (declarations and reference citations in
// include/pumitally_c.h).  No exceptions cross this boundary.
#include "pumitally_c.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <string>

#include "engine.hpp"

struct pumitally_engine {
  ptb::Engine *impl;
};

namespace {

int device_from_args(int *argc, char ***argv) {
  int dev = -1;
  if (const char *env = std::getenv("PUMITALLY_DEVICE")) dev = std::atoi(env);
  if (argc && argv && *argv)
    for (int i = 0; i < *argc; ++i) {
      const char *a = (*argv)[i];
      if (a && std::strncmp(a, "--pumitally-device=", 19) == 0) dev = std::atoi(a + 19);
    }
  return dev;
}

pumitally_engine *make_engine(ptb::HostMesh &&mesh, int32_t num_particles, int device) {
  try {
    auto *h = new pumitally_engine{nullptr};
    h->impl = new ptb::Engine(std::move(mesh), num_particles, device);
    return h;
  } catch (const std::exception &ex) {
    fprintf(stderr, "%s\n", ex.what());
    return nullptr;
  }
}

template <typename F>
int guarded(pumitally_engine *e, F &&f) {
  if (!e || !e->impl) {
    fprintf(stderr, "[pumitally] ERROR: null engine handle\n");
    return 1;
  }
  try {
    return f(*e->impl);
  } catch (const std::exception &ex) {
    fprintf(stderr, "[pumitally] ERROR: %s\n", ex.what());
    return 1;
  }
}

// The particle data of a move; a device move never writes `flying`.
ptb::Move move_of(const double *origin, const double *dest, const int8_t *flying, const double *weights, int32_t size,
                  const ptb::MoveTally &tally = {}) {
  return ptb::Move{origin, dest, const_cast<int8_t *>(flying), weights, size, tally};
}

int host_move(pumitally_engine *e, const char *what, const ptb::Move &m) {
  if (m.size > 0 && (!m.origin || !m.dest || !m.flying || !m.weights)) {
    fprintf(stderr, "[pumitally] ERROR: %s: null input array\n", what);
    return 1;
  }
  return guarded(e, [&](ptb::Engine &g) { return g.move_to_next_location(m); });
}

int device_move(pumitally_engine *e, const ptb::Move &m, void *stream) {
  return guarded(e, [&](ptb::Engine &g) { return g.move_to_next_location_device(m, static_cast<cudaStream_t>(stream)); });
}

}  // namespace

extern "C" {

pumitally_engine *pumitally_create(const char *mesh_filename, int32_t num_particles, int *argc,
                                   char ***argv) {
  // reference prints the same banner (PumiTallyImpl.cpp:554-555)
  printf("Reading the Omega_h mesh %s to tally with tracklength estimator\n",
         mesh_filename ? mesh_filename : "");
  ptb::HostMesh mesh;
  std::string err;
  if (!mesh.load(mesh_filename ? mesh_filename : "", &err)) {
    fprintf(stderr, "[ERROR] %s\n", err.c_str());
    return nullptr;
  }
  printf("PumiPIC Loaded mesh %s with %lld elements\n", mesh_filename, (long long)mesh.ntets);
  return make_engine(std::move(mesh), num_particles, device_from_args(argc, argv));
}

pumitally_engine *pumitally_create_from_arrays(const double *coords, int64_t nverts,
                                               const int32_t *tet2vert, int64_t ntets,
                                               int32_t num_particles, int32_t device) {
  ptb::HostMesh mesh;
  std::string err;
  if (!mesh.from_arrays(coords, nverts, tet2vert, ntets, &err)) {
    fprintf(stderr, "[ERROR] %s\n", err.c_str());
    return nullptr;
  }
  if (device < 0) device = device_from_args(nullptr, nullptr);
  return make_engine(std::move(mesh), num_particles, device);
}

int pumitally_copy_initial_position(pumitally_engine *e, const double *xyz, int32_t size) {
  if (size > 0 && !xyz) {
    fprintf(stderr, "[pumitally] ERROR: CopyInitialPosition: null position array\n");
    return 1;
  }
  return guarded(e, [&](ptb::Engine &g) { return g.copy_initial_position(xyz, size); });
}

int pumitally_move_to_next_location(pumitally_engine *e, const double *origin, const double *dest,
                                    int8_t *flying, const double *weights, int32_t size) {
  return host_move(e, "MoveToNextLocation", move_of(origin, dest, flying, weights, size));
}

int pumitally_write_tally_results(pumitally_engine *e) {
  return guarded(e, [&](ptb::Engine &g) { return g.write_tally_results(); });
}

void pumitally_destroy(pumitally_engine *e) {
  if (!e) return;
  delete e->impl;
  delete e;
}

int64_t pumitally_num_elements(const pumitally_engine *e) {
  return (e && e->impl) ? e->impl->num_elements() : -1;
}
int32_t pumitally_num_particles(const pumitally_engine *e) {
  return (e && e->impl) ? e->impl->num_particles() : -1;
}
int pumitally_get_flux(pumitally_engine *e, double *out, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_flux(out, n); });
}
int pumitally_get_normalized_flux(pumitally_engine *e, double *out_flux, double *out_volume,
                                  int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_normalized_flux(out_flux, out_volume, n); });
}
int pumitally_get_element_ids(pumitally_engine *e, int32_t *out, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_element_ids(out, n); });
}
int pumitally_get_positions(pumitally_engine *e, double *out, int64_t n3) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_positions(out, n3); });
}
int pumitally_get_adjacency(const pumitally_engine *e, int32_t *out, int64_t n4) {
  if (!e || !e->impl || n4 != 4 * e->impl->num_elements()) return 1;
  const std::vector<int32_t> adj = e->impl->mesh().adjacency_original();
  std::memcpy(out, adj.data(), size_t(n4) * sizeof(int32_t));
  return 0;
}
int pumitally_set_score_bins(pumitally_engine *e, int32_t nbins) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_score_bins(nbins); });
}
int32_t pumitally_get_score_bins(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "score_bins")) : 0;
}
int pumitally_move_to_next_location_binned(pumitally_engine *e, const double *origin, const double *dest,
                                           int8_t *flying, const double *weights, const int32_t *bins, int32_t size) {
  return host_move(e, "MoveToNextLocation", move_of(origin, dest, flying, weights, size, {ptb::MoveTally::kPlain, bins}));
}
int pumitally_move_to_next_location_device_binned(pumitally_engine *e, const double *d_origin, const double *d_dest,
                                                  const int8_t *d_flying, const double *d_weights, const int32_t *d_bins,
                                                  int32_t size, void *stream) {
  return device_move(e, move_of(d_origin, d_dest, d_flying, d_weights, size, {ptb::MoveTally::kPlain, d_bins}), stream);
}

int pumitally_set_scores(pumitally_engine *e, int32_t nscores) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_scores(nscores); });
}
int32_t pumitally_get_scores(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "scores")) : 0;
}
int pumitally_move_to_next_location_scored(pumitally_engine *e, const double *origin, const double *dest, int8_t *flying,
                                           const double *weights, const double *responses, const int32_t *bins,
                                           int32_t size) {
  return host_move(e, "MoveToNextLocationScored",
                   move_of(origin, dest, flying, weights, size, {ptb::MoveTally::kScored, bins, responses}));
}
int pumitally_move_to_next_location_device_scored(pumitally_engine *e, const double *d_origin, const double *d_dest,
                                                  const int8_t *d_flying, const double *d_weights,
                                                  const double *d_responses, const int32_t *d_bins, int32_t size,
                                                  void *stream) {
  return device_move(
      e, move_of(d_origin, d_dest, d_flying, d_weights, size, {ptb::MoveTally::kScored, d_bins, d_responses}), stream);
}

int pumitally_set_time_bins(pumitally_engine *e, const double *edges, int32_t nedges) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_time_bins(edges, nedges); });
}
int32_t pumitally_get_time_bins(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "time_bins")) : 0;
}
int pumitally_move_to_next_location_timed(pumitally_engine *e, const double *origin, const double *dest, int8_t *flying,
                                          const double *weights, const double *times, const double *speeds,
                                          const double *responses, const int32_t *bins, int32_t size) {
  return host_move(e, "MoveToNextLocationTimed",
                   move_of(origin, dest, flying, weights, size, {ptb::MoveTally::kTimed, bins, responses, times, speeds}));
}
int pumitally_move_to_next_location_device_timed(pumitally_engine *e, const double *d_origin, const double *d_dest,
                                                 const int8_t *d_flying, const double *d_weights, const double *d_times,
                                                 const double *d_speeds, const double *d_responses,
                                                 const int32_t *d_bins, int32_t size, void *stream) {
  return device_move(e, move_of(d_origin, d_dest, d_flying, d_weights, size,
                                {ptb::MoveTally::kTimed, d_bins, d_responses, d_times, d_speeds}), stream);
}

int pumitally_set_moments(pumitally_engine *e, int32_t order) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_moments(order); });
}
int32_t pumitally_get_moments(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "moments")) : 0;
}
int pumitally_get_flux_moments(pumitally_engine *e, double *out, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_flux_moments(out, n); });
}
int pumitally_get_flux_gradient(pumitally_engine *e, double *out, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_flux_gradient(out, n); });
}

int pumitally_locate_points(pumitally_engine *e, const double *xyz, int64_t npts, int32_t *out_elem) {
  return guarded(e, [&](ptb::Engine &g) { return g.locate_points(xyz, npts, out_elem); });
}
int pumitally_locate_points_device(pumitally_engine *e, const double *d_xyz, int64_t npts, int32_t *d_elem,
                                   void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.locate_points_device(d_xyz, npts, d_elem, static_cast<cudaStream_t>(stream));
  });
}
int pumitally_evaluate_points(pumitally_engine *e, const double *xyz, int64_t npts, double *out, int64_t n,
                              int32_t *out_elem) {
  return guarded(e, [&](ptb::Engine &g) { return g.evaluate_points(xyz, npts, out, n, out_elem); });
}

int pumitally_set_collision_estimator(pumitally_engine *e, int32_t on) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_collision_estimator(on); });
}
int32_t pumitally_get_collision_estimator(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "collision_estimator")) : 0;
}
int pumitally_tally_collisions(pumitally_engine *e, const double *xyz, int64_t nevents, const double *weights,
                               const double *responses, const int32_t *bins, const double *times) {
  return guarded(e, [&](ptb::Engine &g) { return g.tally_collisions(xyz, nevents, weights, responses, bins, times); });
}
int pumitally_tally_collisions_device(pumitally_engine *e, const double *d_xyz, int64_t nevents, const double *d_weights,
                                      const double *d_responses, const int32_t *d_bins, const double *d_times,
                                      void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.tally_collisions_device(d_xyz, nevents, d_weights, d_responses, d_bins, d_times,
                                     static_cast<cudaStream_t>(stream));
  });
}
int pumitally_tally_collisions_at_particles(pumitally_engine *e, const int8_t *collided, const double *weights,
                                            const double *responses, const int32_t *bins, const double *times,
                                            int32_t n) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.tally_collisions_at_particles(collided, weights, responses, bins, times, n);
  });
}
int pumitally_tally_collisions_at_particles_device(pumitally_engine *e, const int8_t *d_collided,
                                                   const double *d_weights, const double *d_responses,
                                                   const int32_t *d_bins, const double *d_times, int32_t n,
                                                   void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.tally_collisions_at_particles_device(d_collided, d_weights, d_responses, d_bins, d_times, n,
                                                  static_cast<cudaStream_t>(stream));
  });
}
int pumitally_get_collision_results(pumitally_engine *e, int32_t kind, double *out, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_collision_results(kind, out, n); });
}

int pumitally_set_point_detectors(pumitally_engine *e, const double *xyz, int32_t ndet, const double *r0) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_point_detectors(xyz, ndet, r0); });
}
int32_t pumitally_get_point_detectors(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "point_detectors")) : 0;
}
int pumitally_set_detector_void(pumitally_engine *e, int32_t on) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_detector_void(on); });
}
int32_t pumitally_get_detector_void(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "detector_void")) : 0;
}
int pumitally_set_detector_cross_sections(pumitally_engine *e, const double *sigma_t, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_detector_cross_sections(sigma_t, n); });
}
int pumitally_tally_detectors(pumitally_engine *e, const double *xyz, int64_t nevents, const double *weights,
                              const double *pdf, const double *responses, const int32_t *bins, const double *times,
                              const double *speeds) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.tally_detectors(xyz, nevents, weights, pdf, responses, bins, times, speeds);
  });
}
int pumitally_tally_detectors_device(pumitally_engine *e, const double *d_xyz, int64_t nevents, const double *d_weights,
                                     const double *d_pdf, const double *d_responses, const int32_t *d_bins,
                                     const double *d_times, const double *d_speeds, void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.tally_detectors_device(d_xyz, nevents, d_weights, d_pdf, d_responses, d_bins, d_times, d_speeds,
                                    static_cast<cudaStream_t>(stream));
  });
}
int pumitally_tally_detectors_at_particles(pumitally_engine *e, const int8_t *flagged, const double *weights,
                                           const double *pdf, const double *responses, const int32_t *bins,
                                           const double *times, const double *speeds, int32_t n) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.tally_detectors_at_particles(flagged, weights, pdf, responses, bins, times, speeds, n);
  });
}
int pumitally_tally_detectors_at_particles_device(pumitally_engine *e, const int8_t *d_flagged, const double *d_weights,
                                                  const double *d_pdf, const double *d_responses, const int32_t *d_bins,
                                                  const double *d_times, const double *d_speeds, int32_t n,
                                                  void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.tally_detectors_at_particles_device(d_flagged, d_weights, d_pdf, d_responses, d_bins, d_times, d_speeds, n,
                                                 static_cast<cudaStream_t>(stream));
  });
}
int pumitally_get_detector_results(pumitally_engine *e, int32_t kind, double *out, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_detector_results(kind, out, n); });
}

int pumitally_set_face_currents(pumitally_engine *e, int32_t on) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_face_currents(on); });
}
int32_t pumitally_get_face_currents(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "face_currents")) : 0;
}
int pumitally_get_face_current_results(pumitally_engine *e, int32_t direction, int32_t kind, double *out, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_face_current_results(direction, kind, out, n); });
}
int pumitally_get_leakage(pumitally_engine *e, int32_t kind, double *out, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_leakage(kind, out, n); });
}
int pumitally_set_current_cosine_bins(pumitally_engine *e, const double *edges, int32_t nedges) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_current_cosine_bins(edges, nedges); });
}
int32_t pumitally_get_current_cosine_bins(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "current_cosine_bins")) : 0;
}

int pumitally_set_batch_statistics(pumitally_engine *e, int32_t on) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_batch_statistics(on); });
}
int pumitally_end_batch(pumitally_engine *e) {
  return guarded(e, [&](ptb::Engine &g) { return g.end_batch(); });
}
int pumitally_get_batch_results(pumitally_engine *e, int32_t tally, int32_t kind, double *out, int64_t n) {
  if (n > 0 && !out) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.get_batch_results(tally, kind, out, n); });
}
int pumitally_get_batch_max_rel_err(pumitally_engine *e, int32_t tally, int32_t score, double *out_max,
                                    int64_t *out_nonzero) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_batch_max_rel_err(tally, score, out_max, out_nonzero); });
}

int pumitally_set_regions(pumitally_engine *e, const int32_t *region_of_element, int64_t n, int32_t nregions) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_regions(region_of_element, n, nregions); });
}
int32_t pumitally_get_regions(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "regions")) : 0;
}
int pumitally_get_region_volumes(pumitally_engine *e, double *out, int64_t n) {
  if (n > 0 && !out) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.get_region_volumes(out, n); });
}
int pumitally_get_region_results(pumitally_engine *e, int32_t tally, int32_t kind, double *out, int64_t n) {
  if (n > 0 && !out) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.get_region_results(tally, kind, out, n); });
}
int pumitally_get_region_batch_results(pumitally_engine *e, int32_t tally, int32_t kind, double *out, int64_t n) {
  if (n > 0 && !out) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.get_region_batch_results(tally, kind, out, n); });
}

int pumitally_set_region_currents(pumitally_engine *e, int32_t on) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_region_currents(on); });
}
int32_t pumitally_get_region_currents(const pumitally_engine *e) {
  return e ? int32_t(pumitally_get_option(e, "region_currents")) : 0;
}
int64_t pumitally_get_region_current_pair_count(const pumitally_engine *e) {
  return e ? pumitally_get_option(e, "region_current_pairs") : 0;
}
int pumitally_get_region_current_pairs(pumitally_engine *e, int32_t *from, int32_t *to, int64_t n) {
  if (n > 0 && (!from || !to)) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.get_region_current_pairs(from, to, n); });
}
int pumitally_get_region_current_areas(pumitally_engine *e, double *out, int64_t n) {
  if (n > 0 && !out) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.get_region_current_areas(out, n); });
}
int pumitally_get_region_current_results(pumitally_engine *e, int32_t which, int32_t kind, double *out, int64_t n) {
  if (n > 0 && !out) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.get_region_current_results(which, kind, out, n); });
}

int pumitally_save_checkpoint(pumitally_engine *e, const char *path) {
  if (!path) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.save_checkpoint(path); });
}
int pumitally_load_checkpoint(pumitally_engine *e, const char *path) {
  if (!path) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.load_checkpoint(path); });
}
int pumitally_merge_checkpoint(pumitally_engine *e, const char *path) {
  if (!path) return 1;
  return guarded(e, [&](ptb::Engine &g) { return g.merge_checkpoint(path); });
}

int pumitally_set_weight_windows(pumitally_engine *e, const double *lower, const double *upper, int64_t n,
                                 int32_t ngroups) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_weight_windows(lower, upper, n, ngroups); });
}
int32_t pumitally_get_weight_window_groups(const pumitally_engine *e) {
  return (e && e->impl) ? e->impl->weight_window_groups() : 0;
}
int pumitally_get_weight_windows(pumitally_engine *e, double *lower, double *upper, int64_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_weight_windows(lower, upper, n); });
}
int pumitally_generate_weight_windows(pumitally_engine *e, int32_t tally, int32_t score, int32_t time_bin, double ratio,
                                      double max_rel_err) {
  return guarded(e, [&](ptb::Engine &g) { return g.generate_weight_windows(tally, score, time_bin, ratio, max_rel_err); });
}
int pumitally_get_weight_windows_at_particles(pumitally_engine *e, const int32_t *groups, double *lower, double *upper,
                                              int32_t n) {
  return guarded(e, [&](ptb::Engine &g) { return g.weight_windows_at_particles(groups, lower, upper, n); });
}
int pumitally_get_weight_windows_at_particles_device(pumitally_engine *e, const int32_t *d_groups, double *d_lower,
                                                     double *d_upper, int32_t n, void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.weight_windows_at_particles_device(d_groups, d_lower, d_upper, n, static_cast<cudaStream_t>(stream));
  });
}
int pumitally_get_weight_windows_at_points(pumitally_engine *e, const double *xyz, int64_t npts, const int32_t *groups,
                                           double *lower, double *upper) {
  return guarded(e, [&](ptb::Engine &g) { return g.weight_windows_at_points(xyz, npts, groups, lower, upper); });
}
int pumitally_get_weight_windows_at_points_device(pumitally_engine *e, const double *d_xyz, int64_t npts,
                                                  const int32_t *d_groups, double *d_lower, double *d_upper,
                                                  void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.weight_windows_at_points_device(d_xyz, npts, d_groups, d_lower, d_upper, static_cast<cudaStream_t>(stream));
  });
}

int pumitally_set_source(pumitally_engine *e, const double *strength, const double *bias, int64_t n, int32_t ngroups,
                         int32_t per_volume) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_source(strength, bias, n, ngroups, per_volume); });
}
int32_t pumitally_get_source_groups(const pumitally_engine *e) {
  return (e && e->impl) ? e->impl->source_groups() : 0;
}
int pumitally_get_source_strength(pumitally_engine *e, double *total) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_source_strength(total); });
}
int pumitally_sample_source(pumitally_engine *e, uint64_t seed, int64_t first, int64_t n, double *xyz, int32_t *elem,
                            int32_t *group, double *weight, int32_t place) {
  return guarded(e, [&](ptb::Engine &g) { return g.sample_source(seed, first, n, xyz, elem, group, weight, place); });
}
int pumitally_sample_source_device(pumitally_engine *e, uint64_t seed, int64_t first, int64_t n, double *d_xyz,
                                   int32_t *d_elem, int32_t *d_group, double *d_weight, int32_t place, void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.sample_source_device(seed, first, n, d_xyz, d_elem, d_group, d_weight, place,
                                  static_cast<cudaStream_t>(stream));
  });
}

int pumitally_reset_tally(pumitally_engine *e) {
  return guarded(e, [&](ptb::Engine &g) { return g.reset_tally(); });
}

int pumitally_set_source_normalization(pumitally_engine *e, int32_t mode, double value) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_source_normalization(mode, value); });
}
double pumitally_get_source_normalization(pumitally_engine *e) {
  return (e && e->impl) ? e->impl->source_normalization() : 0.0;
}

int pumitally_get_stats(pumitally_engine *e, pumitally_stats *out) {
  return guarded(e, [&](ptb::Engine &g) {
    ptb::EngineStats s;
    if (g.get_stats(&s)) return 1;
    out->segments = s.segments;
    out->tracks = s.tracks;
    out->relocations = s.relocations;
    out->lost = s.lost;
    out->moves = s.moves;
    out->kernel_ms = s.kernel_ms;
    out->h2d_bytes = s.h2d_bytes;
    out->plane_fallbacks = s.plane_fallbacks;
    return 0;
  });
}

int pumitally_set_output_name(pumitally_engine *e, const char *filename) {
  return guarded(e, [&](ptb::Engine &g) {
    g.set_output_name(filename ? filename : "fluxresult.vtk");
    return 0;
  });
}
int pumitally_set_option(pumitally_engine *e, const char *name, int64_t value) {
  return guarded(e, [&](ptb::Engine &g) { return g.set_option(name ? name : "", value); });
}

int64_t pumitally_get_option(const pumitally_engine *e, const char *name) {
  return (e && e->impl && name) ? e->impl->get_option(name) : -1;
}

int pumitally_copy_initial_position_device(pumitally_engine *e, const double *d_xyz, int32_t size,
                                           void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.copy_initial_position_device(d_xyz, size, static_cast<cudaStream_t>(stream));
  });
}
int pumitally_move_to_next_location_device(pumitally_engine *e, const double *d_origin,
                                           const double *d_dest, const int8_t *d_flying,
                                           const double *d_weights, int32_t size, void *stream) {
  return device_move(e, move_of(d_origin, d_dest, d_flying, d_weights, size), stream);
}
int pumitally_set_state_device(pumitally_engine *e, const double *d_xyz, const int32_t *d_elem, int32_t first,
                               int32_t count, void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.set_state_device(d_xyz, d_elem, first, count, static_cast<cudaStream_t>(stream));
  });
}
int pumitally_get_state_device(pumitally_engine *e, double *d_xyz, int32_t *d_elem, int32_t first, int32_t count,
                               void *stream) {
  return guarded(e, [&](ptb::Engine &g) {
    return g.get_state_device(d_xyz, d_elem, first, count, static_cast<cudaStream_t>(stream));
  });
}
int pumitally_get_flux_device(pumitally_engine *e, double *d_out, void *stream) {
  return guarded(e, [&](ptb::Engine &g) { return g.get_flux_device(d_out, static_cast<cudaStream_t>(stream)); });
}
double *pumitally_flux_device_ptr(pumitally_engine *e) {
  return (e && e->impl) ? e->impl->flux_device_ptr() : nullptr;
}
int pumitally_synchronize(pumitally_engine *e) {
  return guarded(e, [&](ptb::Engine &g) { return g.synchronize(); });
}

int pumitally_nccl_unique_id(uint8_t out_id[128]) { return ptb::nccl_get_unique_id(out_id); }
int pumitally_comm_init(pumitally_engine *e, int32_t rank, int32_t nranks, const uint8_t id[128]) {
  return guarded(e, [&](ptb::Engine &g) { return g.comm_init(rank, nranks, id); });
}
int pumitally_allreduce_tally(pumitally_engine *e) {
  return guarded(e, [&](ptb::Engine &g) { return g.allreduce_tally(); });
}
int pumitally_exchange_tally(pumitally_engine *e) {
  return guarded(e, [&](ptb::Engine &g) { return g.exchange_tally(); });
}
int pumitally_reduce_tally_to_owners(pumitally_engine *e) {
  return guarded(e, [&](ptb::Engine &g) { return g.reduce_tally_to_owners(); });
}

int64_t pumitally_debug_order(pumitally_engine *e, int32_t *out, int64_t n) {
  if (!e || !e->impl) return -1;
  return e->impl->debug_order(out, n);
}

int64_t pumitally_debug_stage(const double *origin, const double *dest, int8_t *flying, const double *weights,
                              double *b_dest, double *b_w, int8_t *b_fly, int64_t n, int32_t compare,
                              int32_t threads, void *out_patches, int64_t cap) {
  try {
    ptb::HostStager st(threads, {});
    st.set_buffers(b_dest, b_w, b_fly);
    st.reserve(size_t(cap));
    st.begin(origin, dest, flying, weights, 0, n, compare != 0, static_cast<ptb::PatchEntry *>(out_patches));
    return st.end();
  } catch (const std::exception &ex) {
    fprintf(stderr, "[pumitally] ERROR: %s\n", ex.what());
    return -2;
  }
}

const char *pumitally_version(void) { return "pumitally-b200 0.2 (sm_90a)"; }

}  // extern "C"
