// Engine: device state + batch orchestration (see engine.hpp).
#include "engine.hpp"

#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cerrno>
#include <cfloat>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <type_traits>

#include "host_stage.hpp"
#include "seed_grid.hpp"
#include "vtk_writer.hpp"
#include "weight_windows.cuh"

namespace ptb {

namespace {

#define PTB_CUDA_OK(expr)                                                                  \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      fprintf(stderr, "[pumitally] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e),    \
              __FILE__, __LINE__, cudaGetErrorString(_e));                                 \
      return 1;                                                                            \
    }                                                                                      \
  } while (0)

void cuda_or_throw(cudaError_t e, const char *what) {
  if (e != cudaSuccess)
    throw std::runtime_error(std::string("[pumitally] ") + what + ": " + cudaGetErrorString(e) +
                             " (this library has no CPU fallback; a CUDA device is required)");
}

constexpr unsigned kTicketRing = 256;
constexpr size_t kFluxPad = 1024;  // most ranks a communicator may have (padding of the flux arrays)

template <typename T>
void dev_alloc(T **p, size_t count, const char *what) {
  cuda_or_throw(cudaMalloc(reinterpret_cast<void **>(p), std::max<size_t>(count, 1) * sizeof(T)), what);
}

}  // namespace

Engine::Engine(HostMesh &&mesh, int32_t num_particles, int device)
    : mesh_(std::move(mesh)), n_(num_particles) {
  if (n_ < 0) throw std::runtime_error("[pumitally] num_particles must be >= 0");
  int ndev = 0;
  cuda_or_throw(cudaGetDeviceCount(&ndev), "cudaGetDeviceCount");
  if (ndev <= 0) cuda_or_throw(cudaErrorNoDevice, "no CUDA device");
  if (device >= 0) {
    cuda_or_throw(cudaSetDevice(device), "cudaSetDevice");
    device_ = device;
  } else {
    cuda_or_throw(cudaGetDevice(&device_), "cudaGetDevice");
  }
  cuda_or_throw(cudaStreamCreateWithFlags(&compute_, cudaStreamNonBlocking), "stream");
  cuda_or_throw(cudaStreamCreateWithFlags(&copy_, cudaStreamNonBlocking), "stream");

  const size_t E = size_t(mesh_.ntets), N = size_t(n_);
  dev_alloc(&d_tets_, E, "tet records");
  flux_alloc_ = E + kFluxPad;
  dev_alloc(&d_flux_, E + kFluxPad, "flux");  // padded: the reduce-scatter exchange sends nranks equal shares
  dev_alloc(&d_volume_, E, "volume");
  dev_alloc(&d_scratch_, E, "scratch");
  dev_alloc(&d_state_, N, "particle state");
  // staging buffers (PumiTallyImpl.cpp:36-41; origin and dest get their own so one
  // upload per array suffices instead of re-using one position buffer twice)
  dev_alloc(&d_origin_, 3 * N, "origin staging");
  dev_alloc(&d_dest_, 3 * N, "dest staging");
  dev_alloc(&d_weights_, N, "weights staging");
  dev_alloc(&d_flying_, N, "flying staging");
  dev_alloc(&d_stats_, 1, "stats");
  dev_alloc(&d_coll_counts_, 3, "collision counters");
  cuda_or_throw(cudaMemset(d_coll_counts_, 0, 3 * sizeof(unsigned long long)), "memset");
  dev_alloc(&d_det_counts_, kDetCountersVoid, "detector counters");
  cuda_or_throw(cudaMemset(d_det_counts_, 0, kDetCountersVoid * sizeof(unsigned long long)), "memset");
  dev_alloc(&d_initial_weight_, 1, "initial weight");
  cuda_or_throw(cudaMemset(d_initial_weight_, 0, sizeof(double)), "memset");
  dev_alloc(&d_batch_div_, 2, "batch divisor");
  dev_alloc(&d_stats_red_, 2, "batch statistics reduction");
  dev_alloc(&d_tickets_, 2 * kTicketRing, "tickets");  // second half: the other L2 partition's tickets (die split)
  dev_alloc(&d_pcell_, N, "particle cells");
  dev_alloc(&d_order_, N, "processing order");
  dev_alloc(&d_work_count_, kTicketRing, "work counts");

  cuda_or_throw(cudaMemcpy(d_tets_, mesh_.records.data(), E * sizeof(TetRecord), cudaMemcpyHostToDevice), "upload tets");
  cuda_or_throw(cudaMemcpy(d_volume_, mesh_.volume.data(), E * sizeof(double), cudaMemcpyHostToDevice), "upload volume");
  cuda_or_throw(cudaMemset(d_flux_, 0, (E + kFluxPad) * sizeof(double)), "memset");
  cuda_or_throw(cudaMemset(d_stats_, 0, sizeof(DeviceStats)), "memset");
  // InitializeParticlesInElement0 (PumiTallyImpl.cpp:492-528)
  cuda_or_throw(launch_init_particles(d_state_, n_, mesh_.centroid0[0], mesh_.centroid0[1],
                                      mesh_.centroid0[2], mesh_.start_elem, compute_), "init particles");
  cuda_or_throw(cudaStreamSynchronize(compute_), "init sync");
  build_seed_grid();
  use_seed_grid_ = mesh_.hull_convex;  // seed_grid_mode_ 1: only where it is equivalent to the reference's walk
  if (!mesh_.hull_convex)
    printf("[INFO] pumitally-b200: the mesh hull is not convex: relocation walks go the reference's way (no seed-grid "
           "shortcut; option seed_grid=2 forces it)\n");
  variant_ = choose_variant();
  if (const char *env = std::getenv("PUMITALLY_REGISTER_HOST")) register_host_ = std::atoi(env) != 0;
  if (const char *env = std::getenv("PUMITALLY_DIE_SPLIT")) {
    if (std::atoi(env) != 0) set_option("die_split", 1);
  }
  // the packed records are only needed on the device from here on
  std::vector<TetRecord>().swap(mesh_.records);
  printf("[INFO] pumitally-b200: %lld elements, %d particles on CUDA device %d\n",
         (long long)mesh_.ntets, n_, device_);
}

// Compact layout: TetLinks (32 B per tet) + vertices (32 B each) are what the edge-function walk
// reads per crossing; TetStart lines (128 B per tet) are read once per ray.  Built and uploaded the
// first time one of the edge-walk variants is selected (the default kernels never touch it).
bool Engine::upload_compact() {
#ifndef PTB_EXPERIMENTS
  return false;  // the edge-walk variants are not part of this library
#endif
  if (d_links_) return true;
  std::string err;
  if (!mesh_.build_compact(&err)) {
    printf("[INFO] pumitally-b200: compact layout not built (%s); plane records only\n", err.c_str());
    return false;
  }
  const size_t E = size_t(mesh_.ntets), V = size_t(mesh_.nverts);
  std::vector<TetLinks> links(E);
  for (size_t e = 0; e < E; ++e) links[e] = mesh_.starts[e].links;
  dev_alloc(&d_links_, E, "tet links");
  dev_alloc(&d_verts_, V, "vertices");
  dev_alloc(&d_starts_, E, "tet start lines");
  cuda_or_throw(cudaMemcpy(d_links_, links.data(), E * sizeof(TetLinks), cudaMemcpyHostToDevice), "upload links");
  cuda_or_throw(cudaMemcpy(d_verts_, mesh_.cverts.data(), V * sizeof(VertexRec), cudaMemcpyHostToDevice), "upload vertices");
  cuda_or_throw(cudaMemcpy(d_starts_, mesh_.starts.data(), E * sizeof(TetStart), cudaMemcpyHostToDevice), "upload start lines");
  std::vector<TetStart>().swap(mesh_.starts);
  std::vector<VertexRec>().swap(mesh_.cverts);
  return true;
}

Engine::~Engine() {
  cudaSetDevice(device_);
  cudaDeviceSynchronize();
  if (nccl_comm_) nccl_comm_destroy(nccl_comm_);
  cudaFree(d_flux_global_);
  if (ev_order_) cudaEventDestroy(ev_order_);
  if (ev_done_) cudaEventDestroy(ev_done_);
  cudaFree(d_mask_);
  for (AuxUpload *u : {&time_up_, &resp_up_, &bins_up_}) {
    cudaFree(u->d);
    if (u->h) cudaFreeHost(u->h);
    if (u->ev) cudaEventDestroy(u->ev);
  }
  cudaFree(d_edges_);
  cudaFree(d_mu_edges_);
  cudaFree(d_face_opp_);
  cudaFree(d_hull_slots_);
  if (ev_copy0_) cudaEventDestroy(ev_copy0_);
  if (ev_copy1_) cudaEventDestroy(ev_copy1_);
  if (ev_ar0_) cudaEventDestroy(ev_ar0_);
  if (ev_ar1_) cudaEventDestroy(ev_ar1_);
  for (auto &r : registered_) cudaHostUnregister(const_cast<void *>(r.first));
  for (auto &t : timers_free_) { cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
  for (auto &t : timers_busy_) { cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
  for (auto &e : chunk_events_) cudaEventDestroy(e);
  stager_.reset();
  if (h_pos_) { cudaHostUnregister(h_pos_); free(h_pos_); }
  if (d2h_) cudaStreamDestroy(d2h_);
  for (auto &e : pos_events_) cudaEventDestroy(e);
  for (auto &e : walk_events_) cudaEventDestroy(e);
  if (stage_base_) {
    if (stage_registered_) { cudaHostUnregister(stage_base_); free(stage_base_); }
    else cudaFreeHost(stage_base_);
  }
  cudaFree(d_rows_);
  if (h_patch_) cudaFreeHost(h_patch_);
  cudaFree(d_patch_);
  cudaFree(d_links_); cudaFree(d_verts_); cudaFree(d_starts_);
  cudaFree(d_tets_); cudaFree(d_flux_); cudaFree(d_volume_); cudaFree(d_scratch_);
  cudaFree(d_state_);
  cudaFree(d_origin_); cudaFree(d_dest_); cudaFree(d_weights_); cudaFree(d_flying_);
  cudaFree(d_stats_);
  cudaFree(d_initial_weight_);
  cudaFree(d_tickets_);
  cudaFree(d_grid_);
  cudaFree(d_orig_of_internal_); cudaFree(d_internal_of_orig_);
  cudaFree(d_cell_rank_);
  cudaFree(d_pcell_); cudaFree(d_order_); cudaFree(d_cell_count_); cudaFree(d_cell_sums_);
  cudaFree(d_work_count_);
  cudaFree(d_cand_off_); cudaFree(d_cand_);
  cudaFree(d_hull_off_); cudaFree(d_hull_tets_);
  cudaFree(d_arena_);
  cudaFree(d_eval_vals_); cudaFree(d_eval_grads_); cudaFree(d_eval_cen_);
  cudaFree(d_coll_counts_);
  cudaFree(d_det_counts_);
  cudaFree(d_det_); cudaFree(d_det_pos_); cudaFree(d_det_r0_); cudaFree(d_sigma_);
  free_stats();
  free_regions();
  free_region_currents();
  free_weight_windows();
  free_source();
  cudaFree(d_src_verts_);
  cudaFree(d_batch_div_); cudaFree(d_stats_red_);
  if (compute_) cudaStreamDestroy(compute_);
  if (copy_) cudaStreamDestroy(copy_);
}

// Localise the seed point of every grid cell with the walk kernel itself (from the centroid of
// element 0, like any particle) and keep the tet for cells whose seed point lies in the mesh.
void Engine::build_seed_grid() {
  grid_ = choose_seed_grid(mesh_);
  const int32_t ncell = grid_.nx * grid_.ny * grid_.nz;
  double *xyz = nullptr;
  ParticleState *ts = nullptr;
  dev_alloc(&d_grid_, size_t(ncell), "seed grid");
  dev_alloc(&xyz, 3 * size_t(ncell), "seed points");
  dev_alloc(&ts, size_t(ncell), "seed tmp");
  cuda_or_throw(launch_seed_points(grid_, xyz, compute_), "seed points");
  cuda_or_throw(launch_init_particles(ts, ncell, mesh_.centroid0[0], mesh_.centroid0[1],
                                      mesh_.centroid0[2], mesh_.start_elem, compute_), "seed init");
  WalkParams p{};
  p.tets = d_tets_;
  p.flux = d_flux_;
  p.state = ts;
  p.origin = xyz;
  p.begin = 0;
  p.end = ncell;
  p.max_iters = int32_t(std::min<int64_t>(mesh_.ntets + 16, INT_MAX));
  p.bulk_ok = 1;
  p.work_counter = d_tickets_;
  p.stats = d_stats_;
  p.cx = mesh_.center[0]; p.cy = mesh_.center[1]; p.cz = mesh_.center[2];
  cuda_or_throw(launch_walk(p, kVariantPersistRefill8, 128, compute_), "seed walk");
  cuda_or_throw(launch_seed_finalize(xyz, ts, d_grid_, ncell, compute_), "seed finalize");
  cuda_or_throw(cudaStreamSynchronize(compute_), "seed sync");
  cuda_or_throw(cudaMemset(d_stats_, 0, sizeof(DeviceStats)), "memset");
  cudaFree(xyz); cudaFree(ts);
  grid_.cell_tet = d_grid_;
  {
    const std::vector<int32_t> rank = morton_cell_ranks(grid_);
    dev_alloc(&d_cell_rank_, size_t(ncell), "cell ranks");
    cuda_or_throw(cudaMemcpy(d_cell_rank_, rank.data(), size_t(ncell) * sizeof(int32_t), cudaMemcpyHostToDevice), "upload cell ranks");
    grid_.cell_rank = d_cell_rank_;
  }
  dev_alloc(&d_cell_count_, size_t(ncell), "cell histogram");
  dev_alloc(&d_cell_sums_, size_t(ncell) / 1024 + 2, "cell block sums");
}

void Engine::collect_timers(bool wait) {
  for (size_t k = 0; k < timers_busy_.size();) {
    TimerPair t = timers_busy_[k];
    if (wait) cudaEventSynchronize(t.b);
    if (cudaEventQuery(t.b) == cudaSuccess) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) kernel_ms_ += ms;
      if (t.tag >= 0) {
        explore_ms_[t.tag] += ms;
        if (--explore_pending_ == 0 && explore_complete_) {  // all four exploration moves measured
          // the streaming kernel keeps the job unless sorting buys more than 3 %
          tuned_variant_ = (explore_ms_[1] > 0.0 && explore_ms_[1] < 0.97 * explore_ms_[0]) ? kVariantPacked : kVariantPersistRefill8;
          explore_complete_ = false;
        }
      }
      timers_free_.push_back(t);
      timers_busy_[k] = timers_busy_.back();
      timers_busy_.pop_back();
    } else {
      ++k;
    }
  }
}

// Picks the kernel for the move that is about to be launched (see the auto-tuner note in engine.hpp).
void Engine::begin_move(bool scored) {
  collect_timers(false);
  move_variant_ = variant_;
  move_tag_ = -1;
  if (!auto_variant_ || !autotune_ || variant_ != kVariantPersistRefill8) return;
  // sorting costs per particle, walking per crossing: with thousands of particles per tet (config c3) the
  // sorted variant cannot win and two exploration moves would cost more than an epoch can pay back
  if (int64_t(n_) > 16 * mesh_.ntets) return;
  // a scored, timed or moment move runs the kernel a plain move would run outside the exploration, and is never
  // timed for it (its walk costs more per crossing): the tuner's clock counts plain moves only
  if (scored) {
    move_variant_ = tuned_variant_;
    return;
  }
  // exploration moves 1..4 of every epoch in the order streaming, packed, packed, streaming (move 0 of a
  // run is atypical: nothing has been re-sourced yet); decision when all four have been timed
  const uint64_t k = (moves_ - scored_moves_) % kTuneEpoch;
  if (k >= 1 && k <= 4) {
    if (k == 1) { explore_ms_[0] = explore_ms_[1] = 0.0; explore_complete_ = false; }
    move_tag_ = (k == 2 || k == 3) ? 1 : 0;
    move_variant_ = move_tag_ ? kVariantPacked : kVariantPersistRefill8;
  } else {
    if (k == 5) {
      explore_complete_ = true;  // every exploration launch has been issued
      // a caller that queues moves back to back has not let the four timed moves finish yet: wait for
      // them once per epoch (a bubble of at most one move) rather than decide an epoch late
      for (auto &t : timers_busy_)
        if (t.tag >= 0) cudaEventSynchronize(t.b);
      collect_timers(false);
      if (explore_complete_ && explore_pending_ == 0) {
        tuned_variant_ = (explore_ms_[1] > 0.0 && explore_ms_[1] < 0.97 * explore_ms_[0]) ? kVariantPacked : kVariantPersistRefill8;
        explore_complete_ = false;
      }
    }
    move_variant_ = tuned_variant_;
  }
}

// Re-sourced particles of the pinned-caller host path: phase 1 for the listed particles only.
int Engine::relocate_patches(const PatchEntry *d_list, int32_t count, cudaStream_t stream) {
  if (count <= 0) return 0;
  WalkParams p{};
  p.tets = d_tets_;
  p.flux = d_flux_;
  p.state = d_state_;
  p.begin = 0;
  p.end = n_;
  p.max_iters = max_iters_ > 0 ? max_iters_ : int32_t(std::min<int64_t>(mesh_.ntets + 16, INT_MAX));
  p.stats = d_stats_;
  p.grid = grid_;
  p.cx = mesh_.center[0]; p.cy = mesh_.center[1]; p.cz = mesh_.center[2];
  if (!use_seed_grid_) p.grid.cell_tet = nullptr;
  PTB_CUDA_OK(launch_relocate_patches(p, d_list, count, d_flying_, stream));
  ++launches_;
  return 0;
}

// Particle state, binning scratch and the ticket ring are shared by every launch: work enqueued on
// another stream than the previous launch's (a device-pointer move on the caller's stream after a
// host-pointer move on the engine's own, or the other way round) is ordered behind it by an event.
int Engine::follow_last_stream(cudaStream_t stream) {
  if (last_stream_set_ && stream != last_stream_) {
    if (!ev_order_) PTB_CUDA_OK(cudaEventCreateWithFlags(&ev_order_, cudaEventDisableTiming));
    PTB_CUDA_OK(cudaEventRecord(ev_order_, last_stream_));
    PTB_CUDA_OK(cudaStreamWaitEvent(stream, ev_order_, 0));
  }
  last_stream_ = stream;
  last_stream_set_ = true;
  return 0;
}

int Engine::launch_range(const double *d_origin, const double *d_dest, const int8_t *d_flying,
                         const double *d_weights, int32_t begin, int32_t end, cudaStream_t stream,
                         const MoveTally &t) {
  if (end <= begin) return 0;
  if (follow_last_stream(stream)) return 1;
  if (d_dest) flux_global_valid_ = flux_owned_only_ = eval_valid_ = false;  // the local tally moves on; the last exchange no longer describes it
  const int64_t slice = int64_t(nbins_) * int64_t(bin_len());  // time filter: from one time bin of an array to the next
  // face currents: [time][bin][cosine][element][4] after the tallies; a binned move's unmatched particles cross into the
  // scratch array after the unreported flux array (every cosine bin into it)
  const int64_t E4 = 4 * int64_t(mesh_.ntets), cur_bin = int64_t(ncos()) * E4, cur_slice = int64_t(nbins_) * cur_bin;
  double *cur = currents_ ? d_flux_ + current_base() : nullptr;
  if (!(t.bins && d_dest))
    return launch_range_into(d_flux_, d_origin, d_dest, d_flying, d_weights, begin, end, stream, t, slice, move_variant_,
                             move_tag_, cur, cur_slice, E4);
  // Score filter: particles are independent and a particle that does not fly is not touched, so the range
  // is walked once per bin with the flying flags masked down to that bin's particles and the tally pointed
  // at that bin's flux array -- the walk kernels themselves are the unfiltered ones.  One more pass (array
  // nbins_, never reported) flies the particles whose bin is outside [0, nbins_): they move, unscored.
  // The streaming kernel pays for every particle of the range in every pass, flying or not; the packed kernel's
  // sort pass keeps only the flying
  // ones, so its passes cost what their members cost.  Unless the caller has fixed the kernel, binned moves use it,
  // and are not one of the auto-tuner's exploration moves.
  const bool packed = auto_variant_ && d_weights;
  const int variant = packed ? int(kVariantPacked) : move_variant_, tag = packed ? -1 : move_tag_;
  for (int32_t b = 0; b <= nbins_; ++b) {
    if (launch_bin_mask(d_flying, t.bins, b, nbins_, d_mask_, begin, end, stream) != cudaSuccess) return 1;
    ++launches_;
    // the unreported array follows every reported one (with a time filter, all time bins of a bin-b pass go to it)
    if (launch_range_into(d_flux_ + (b < nbins_ ? size_t(b) * bin_len() : reported_len()), d_origin, d_dest, d_mask_,
                          d_weights, begin, end, stream, t, b < nbins_ ? slice : 0, variant, tag,
                          cur ? (b < nbins_ ? cur + b * cur_bin : d_flux_ + reported_len() + bin_len()) : nullptr,
                          b < nbins_ ? cur_slice : 0, b < nbins_ ? E4 : 0))
      return 1;
  }
  return 0;
}

int Engine::launch_range_into(double *d_flux, const double *d_origin, const double *d_dest, const int8_t *d_flying,
                              const double *d_weights, int32_t begin, int32_t end, cudaStream_t stream,
                              const MoveTally &t, int64_t slice, int variant, int tag, double *d_cur,
                              int64_t cur_slice, int64_t mu_stride) {
  if (d_dest && d_weights && initial_weight_pending_)  // first tracks of the batch: their total weight
    PTB_CUDA_OK(launch_sum_flying_weights(d_flying, d_weights, begin, end, d_initial_weight_, stream));
  CurrentWalkParams tp{};
  WalkParams &p = tp;
  const bool timed_walk = t.kind == MoveTally::kTimed && d_dest;
  // with moments every tallying move is a scored one; the plain and binned moves have one score and no responses
  const bool scored = scored_move(t) && d_dest;
  if (scored) tp.sc = ScoreParams{t.responses, nscores_, stride_};
  if (timed_walk) tp.tm = TimeParams{d_edges_, t.times, t.speeds, ntime_, slice};
  if (scored && currents_) tp.cu = CurrentParams{d_cur, cur_slice, d_mu_edges_, nmu_, mu_stride};
  p.tets = d_tets_;
  p.links = d_links_;
  p.verts = d_verts_;
  p.starts = d_starts_;
  p.flux = d_flux;
  p.state = d_state_;
  p.origin = d_origin;
  p.dest = d_dest;
  p.flying = d_flying;
  p.weights = d_weights;
  p.begin = begin;
  p.end = end;
  p.max_iters = max_iters_ > 0 ? max_iters_ : int32_t(std::min<int64_t>(mesh_.ntets + 16, INT_MAX));
  p.stats = d_stats_;
  p.grid = grid_;
  p.cx = mesh_.center[0]; p.cy = mesh_.center[1]; p.cz = mesh_.center[2];
  if (!use_seed_grid_) p.grid.cell_tet = nullptr;
  p.work_counter = d_tickets_ + (ticket_next_++ % kTicketRing);
  if (die_split_ && die0_sms_ > 0) {  // sorted kernels: each L2 partition's SMs on their own end of the sequence
    for (int i = 0; i < 8; ++i) p.die_mask[i] = die_mask_[i];
    p.die0_sms = die0_sms_;
    p.nsms = nsms_;
    p.work_counter2 = p.work_counter + kTicketRing;
  }
  auto aligned16 = [](const void *q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
  p.bulk_ok = (begin % 16 == 0) && aligned16(d_origin) && aligned16(d_dest) && aligned16(d_flying) &&
              aligned16(d_weights);
  TimerPair timer{};
  if (timers_free_.empty()) {
    PTB_CUDA_OK(cudaEventCreate(&timer.a));
    PTB_CUDA_OK(cudaEventCreate(&timer.b));
  } else {
    timer = timers_free_.back();
    timers_free_.pop_back();
  }
  timer.tag = tag;
  if (timer.tag >= 0) ++explore_pending_;
  PTB_CUDA_OK(cudaEventRecord(timer.a, stream));
  bool use_packed = variant_is_packed(variant);
  if (use_packed && !(d_dest && d_weights)) {  // localisation
    variant = kVariantPersistRefill8;
    use_packed = false;
  }
  if (use_packed && !d_rows_ &&
      cudaMalloc(reinterpret_cast<void **>(&d_rows_), std::max<size_t>(size_t(n_), 1) * sizeof(PackedRow)) != cudaSuccess) {
    cudaGetLastError();
    d_rows_ = nullptr;
    if (auto_variant_) {  // the auto-tuner wanted to try it: carry on with the streaming kernel for good
      autotune_ = false;
      tuned_variant_ = variant = move_variant_ = kVariantPersistRefill8;
      use_packed = false;
    } else {
      fprintf(stderr, "[pumitally] ERROR: no device memory for the packed particle rows\n");
      return 1;
    }
  }
  if (use_packed) {
    // counting sort by seed-grid cell, the scatter pass writing one 64-byte row per flying particle
    unsigned int *wc = d_work_count_ + (ticket_next_ % kTicketRing);
    SeedGrid bin_grid = grid_;
    if (!morton_) bin_grid.cell_rank = nullptr;
    PTB_CUDA_OK(launch_bin_pack_particles(bin_grid, d_origin, d_dest, d_weights, d_flying, d_state_, begin, end,
                                          d_pcell_, d_cell_count_, d_cell_sums_, d_rows_ + begin, wc, bin_midpoint_, stream));
    p.rows = d_rows_ + begin;
    p.work_count = wc;
    last_work_count_ = wc;
    p.flying = nullptr;  // only flying particles have rows
    launches_ += 5;  // count, 3-kernel scan, pack
  }
  if (variant_is_gather(variant)) {
    // counting sort of the range's flying particles by seed-grid cell of their origin
    unsigned int *wc = d_work_count_ + (ticket_next_ % kTicketRing);
    const double *key = d_origin;  // no origin array (pinned-caller host path): the stored position
    SeedGrid bin_grid = grid_;
    if (!morton_) bin_grid.cell_rank = nullptr;
    p.claim_run = claim_run_;
    PTB_CUDA_OK(launch_bin_particles(bin_grid, key, d_state_, (bin_midpoint_ && d_dest) ? d_dest : nullptr, d_flying, begin, end, d_pcell_, d_cell_count_,
                                     d_cell_sums_, d_order_ + begin, wc, stream));
    p.order = d_order_ + begin;
    p.work_count = wc;
    last_work_count_ = wc;
    launches_ += 5;  // count, 3-kernel scan, scatter
    p.flying = nullptr;  // order[] holds flying particles only
  }
  const cudaError_t err = scored ? launch_walk_tallied(tp, timed_walk, moments_ > 0, currents_, variant, block_, stream)
                                 : launch_walk(p, variant, block_, stream);
  if (err != cudaSuccess) {
    fprintf(stderr, "[pumitally] ERROR: walk kernel %d: %s (scored, timed and moment moves run on the kernels 0, 8, 16 "
                    "and 24 only)\n", variant, cudaGetErrorString(err));
    return 1;
  }
  ++launches_;
  PTB_CUDA_OK(cudaEventRecord(timer.b, stream));
  timers_busy_.push_back(timer);
  return 0;
}

// OpenMC hands over ordinary (pageable) std::vector storage and reuses the same buffers for every
// call.  Pageable cudaMemcpyAsync is staged by the driver at a fraction of the PCIe rate, so with
// option register_host=1 (or PUMITALLY_REGISTER_HOST=1) each new caller buffer is page-locked once
// with cudaHostRegister and stays registered until the engine is destroyed.  Off by default: the
// caller must then keep those buffers alive (or at least not free them) for the engine's lifetime.
void Engine::maybe_register(const void *p, size_t bytes) {
  if (!register_host_ || !p || bytes == 0 || host_is_pinned(p)) return;
  for (auto &r : registered_)
    if (r.first == p && r.second >= bytes) return;
  if (cudaHostRegister(const_cast<void *>(p), bytes, cudaHostRegisterDefault) == cudaSuccess)
    registered_.emplace_back(p, bytes);
  else
    cudaGetLastError();  // overlapping/foreign registration: fall back to the pageable path
}

bool Engine::host_is_pinned(const void *p) const {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

// CopyInitialPositionToBuffer + MoveToInitialLocation (PumiTallyImpl.cpp:54-64, 195-221)
int Engine::copy_initial_position(const double *xyz, int32_t size) {
  if (int64_t(size) != 3 * int64_t(n_)) {
    fprintf(stderr, "[pumitally] ERROR: CopyInitialPosition size %d != 3 * num_particles (%d)\n", size, n_);
    return 1;
  }
  if (initialized_) {
    fprintf(stderr, "[pumitally] ERROR: CopyInitialPosition may only be called once\n");
    return 1;
  }
  PTB_CUDA_OK(cudaSetDevice(device_));
  // Through the staging slots when they can be had: the pool copies xyz into the pinned dest slots
  // (pageable cudaMemcpy runs at a fifth of the PCIe rate) and the device copy goes to d_dest_, so
  // that "pinned dest slots == device dest array == where every particle is" already holds for the
  // first move and its origins need not travel either.
  const double *src = xyz;
  double *d_xyz = d_origin_;
  if (host_path_ != 0 && n_ > 0 && ensure_stage_buffers(xyz, size_t(size) * sizeof(double)) == 0) {
    pool_copy(h_dest_, xyz, size_t(size) * sizeof(double));
    src = h_dest_;
    d_xyz = d_dest_;
    mirror_valid_ = true;
  }
  PTB_CUDA_OK(cudaMemcpyAsync(d_xyz, src, size_t(size) * sizeof(double), cudaMemcpyHostToDevice, compute_));
  h2d_bytes_ += double(size) * sizeof(double);
  tallied_ = true;  // the localisation walk counts relocations and lost walks
  move_variant_ = variant_;
  move_tag_ = -1;
  if (launch_range(d_xyz, nullptr, nullptr, nullptr, 0, n_, compute_)) return 1;
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  initialized_ = true;
  return 0;
}

int Engine::copy_initial_position_device(const double *d_xyz, int32_t size, cudaStream_t stream) {
  if (int64_t(size) != 3 * int64_t(n_) || initialized_) {
    fprintf(stderr, "[pumitally] ERROR: CopyInitialPosition: bad size or called twice\n");
    return 1;
  }
  PTB_CUDA_OK(cudaSetDevice(device_));
  tallied_ = true;  // the localisation walk counts relocations and lost walks
  move_variant_ = variant_;
  move_tag_ = -1;
  if (launch_range(d_xyz, nullptr, nullptr, nullptr, 0, n_, stream)) return 1;
  initialized_ = true;
  return 0;
}

constexpr int kPatchSlots = 4;             // pinned patch lists in flight
constexpr double kPatchMaxFraction = 0.4;  // above this share of changed origins a chunk is sent whole

// Pinned staging ("bounce") buffers of the host-pointer path, allocated at the first host call:
// one slot per particle for dest, weight and flying.  They are the DMA source of every move AND the
// mirror the next move's origins are compared against (host_stage.hpp).  Ordinary page-aligned
// memory, first touched by the pool's workers (which run on the GPU's NUMA node) and then
// page-locked with cudaHostRegister -- an order of magnitude faster than cudaHostAlloc for
// hundreds of MB; cudaHostAlloc is the fallback.
// The workers follow the caller's memory: if the arrays of this call live on another NUMA node than
// the one the pool runs on, the workers move there (a few microseconds, once per change).
void Engine::follow_caller_memory(const void *p, size_t bytes) {
  if (!stager_) return;
  const int node = numa_node_of(p, bytes);
  if (node < 0 || node == pool_node_) return;
  const std::vector<int> cpus = numa_node_cpus(node);
  if (cpus.empty()) return;
  stager_->pool().repin(cpus);
  pool_node_ = node;
}

int Engine::ensure_stage_buffers(const void *caller_mem, size_t caller_bytes) {
  if (stage_ready_) return 0;
  if (stage_failed_) return 1;
  const size_t N = std::max<size_t>(size_t(n_), 1);
  if (!stager_) {
    // workers (and, by first touch, the staging slots) on the NUMA node of the caller's arrays; when
    // that cannot be determined, on the GPU's node
    std::vector<int> cpus;
    pool_node_ = numa_node_of(caller_mem, caller_bytes);
    if (pool_node_ >= 0) cpus = numa_node_cpus(pool_node_);
    if (cpus.empty()) {
      char bus[64] = {0};
      pool_node_ = -1;
      if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device_) == cudaSuccess) cpus = gpu_local_cpus(bus);
      else cudaGetLastError();
    }
    // one of the CPUs the quota allows is left to the calling thread, which enqueues copies and kernels
    stager_.reset(new HostStager(host_threads_ > 0 ? host_threads_ : std::max(1, default_host_threads() - 1), cpus));
  }
  HostPool *pool_ = &stager_->pool();
  const size_t bytes_dest = (3 * N * sizeof(double) + 4095) & ~size_t(4095);
  const size_t bytes_w = (N * sizeof(double) + 4095) & ~size_t(4095);
  const size_t bytes_fly = (N + 4095) & ~size_t(4095);
  const size_t total = bytes_dest + bytes_w + bytes_fly;
  void *base = nullptr;
  if (posix_memalign(&base, size_t(2) << 20, total) == 0) {
    madvise(base, total, MADV_HUGEPAGE);  // 2 MB pages where the kernel offers them: three streams of TLB misses less
    const int T = pool_->size();
    // Where the staging slots live.  Default: on the workers' node (= the caller's arrays' node).
    // PUMITALLY_STAGE_NODE=<n> puts them on another node: on a two-socket host the pass then draws on
    // both sockets' memory controllers (caller arrays on one, slots + DMA reads on the other).
    const char *env_node = std::getenv("PUMITALLY_STAGE_NODE");
    const std::vector<int> there;  // (placement is done with mbind below: the other node's CPUs may not be in the mask)
    if (env_node) {
      unsigned long mask[16] = {0};
      const int node = std::atoi(env_node);
      if (node >= 0 && node < 1024) {
        mask[node / 64] = 1ul << (node % 64);
        if (syscall(SYS_mbind, base, total, 2 /* MPOL_BIND */, mask, 1024ul, 0u) != 0)
          fprintf(stderr, "[pumitally] WARNING: mbind of the staging slots to node %d failed\n", node);
      }
    }
    pool_->run([&](int t) {  // first touch on the workers' NUMA node
      const size_t lo = (total * size_t(t) / size_t(T)) & ~size_t(4095);
      const size_t hi = t == T - 1 ? total : (total * size_t(t + 1) / size_t(T)) & ~size_t(4095);
      std::memset(static_cast<char *>(base) + lo, 0, hi - lo);
    });
    if (!there.empty() && pool_node_ >= 0) pool_->repin(numa_node_cpus(pool_node_));
    if (cudaHostRegister(base, total, cudaHostRegisterDefault) == cudaSuccess) {
      stage_registered_ = true;
    } else {
      cudaGetLastError();
      free(base);
      base = nullptr;
    }
  }
  if (!base) {
    if (cudaHostAlloc(&base, total, cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      stage_failed_ = true;  // the direct path (plain copies from the caller's memory) still works
      fprintf(stderr, "[pumitally] WARNING: no pinned host memory for the staging buffers (%zu MB); "
                      "uploads fall back to direct copies from the caller's arrays\n", total >> 20);
      return 1;
    }
    stage_registered_ = false;
  }
  stage_base_ = base;
  h_dest_ = static_cast<double *>(base);
  h_w_ = reinterpret_cast<double *>(static_cast<char *>(base) + bytes_dest);
  h_fly_ = reinterpret_cast<int8_t *>(static_cast<char *>(base) + bytes_dest + bytes_w);
  stager_->set_buffers(h_dest_, h_w_, h_fly_);
  stage_ready_ = true;
  return 0;
}

int Engine::ensure_patch_buffers(int nchunks, int32_t chunk) {
  size_t cap = size_t(double(std::min<int64_t>(chunk, n_)) * kPatchMaxFraction) + 64;
  if (h_patch_ && patch_cap_ >= cap && patch_chunks_ >= nchunks) return 0;
  // (grow only, in both dimensions: moves with different stage sizes -- binned and plain -- may alternate)
  cap = std::max(cap, patch_cap_);
  nchunks = std::max(nchunks, patch_chunks_);
  PTB_CUDA_OK(cudaDeviceSynchronize());
  if (h_patch_) cudaFreeHost(h_patch_);
  if (d_patch_) cudaFree(d_patch_);
  h_patch_ = nullptr;
  d_patch_ = nullptr;
  patch_cap_ = cap;
  patch_chunks_ = nchunks;
  PTB_CUDA_OK(cudaHostAlloc(reinterpret_cast<void **>(&h_patch_), cap * kPatchSlots * sizeof(PatchEntry), cudaHostAllocDefault));
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_patch_), cap * size_t(nchunks) * sizeof(PatchEntry)));
  stager_->reserve(cap);
  return 0;
}

// MoveToNextLocation (PumiTallyImpl.cpp:66-149), host pointers.
//
// Staged path (default): the particle range is cut into chunks; for each chunk the pool refills the
// pinned staging slots from the caller's arrays and finds the origins that differ from the previous
// destinations (stage_chunk), then flying + patch list + dest + weights of the chunk are enqueued on
// the copy stream and the walk kernel of the chunk behind them on the compute stream -- chunk k is
// on the wire and chunk k-1 is being walked while the pool stages chunk k+1.  The device's copy of
// the previous destinations becomes this move's origin array (buffer swap) and only the changed
// origins are patched in, so 32 B + a few patch bytes per particle cross PCIe instead of 57 B.  The
// call returns as soon as the caller's arrays have been consumed (they are in the staging buffers
// by then; reference: blocking deep_copy); copies and kernels may still be in flight.
//
// Direct path (option host_path=0, or no pinned memory to be had): plain cudaMemcpyAsync of all
// four arrays from the caller's memory, optionally page-locked first (option register_host).
//
// Binned, scored and timed moves: the side arrays travel ahead of the particle data on the copy stream (times and
// speeds, then responses, then bins), through a pinned copy made by the worker pool when a caller's array is pageable
// (upload_aux), and are on the device before the call returns.  Everything else is the ordinary host path, except the
// pinned-caller variant (move_pinned), whose relocation pass knows nothing of bins or scores.
int Engine::move_to_next_location(const Move &m) {
  if (move_refused(m, false)) return 1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  tallied_ = true;
  const MoveTally &t = m.tally;
  const size_t N = size_t(n_);
  MoveTally dev;  // t with the device copies of its arrays
  dev.kind = t.kind;
  cudaEvent_t sent[3];
  int nsent = 0, rc = 0;
  auto send = [&](AuxUpload &u, const void *a, const void *b, size_t bytes) {
    if (rc == 0) rc = upload_aux(u, a, b, bytes);
    if (rc == 0) sent[nsent++] = u.ev;
    return rc == 0;
  };
  if (t.kind == MoveTally::kTimed && send(time_up_, t.times, t.speeds, N * sizeof(double))) {
    dev.times = static_cast<const double *>(time_up_.d);
    dev.speeds = dev.times + N;
  }
  if (t.responses && send(resp_up_, t.responses, nullptr, N * size_t(nscores_) * sizeof(double)))
    dev.responses = static_cast<const double *>(resp_up_.d);
  if (t.bins && nbins_ > 1 && send(bins_up_, t.bins, nullptr, N * sizeof(int32_t)))
    dev.bins = static_cast<const int32_t *>(bins_up_.d);
  if (rc == 0) {
    begin_move(scored_move(t));
    // Pipeline stage size, unless the caller set it: 512 Ki particles for the streaming kernel (shortest tail); the
    // sorted kernels pay a fixed price per launch (a scan over all seed-grid cells), so their stages are 2 Mi.  A
    // binned move walks every stage nbins + 1 times, seven small launches each, all enqueued by this thread between
    // two stage passes: its stages are 2 Mi too.
    int32_t chunk = chunk_;
    if (!chunk_user_set_ && dev.bins) chunk = std::max(chunk, int32_t(1) << 21);
    // The auto-tuner compares kernel times; in a host move the sorted kernel it may prefer would also need the
    // larger stages, whose longer tail can cost more than the kernel wins.  So a host move of more than one stage keeps the engine's base kernel and does not take
    // part in the exploration; the tuner works for device-pointer moves and single-stage host moves (c4's 1 M tracks).
    if (auto_variant_ && variant_is_packed(move_variant_) && !variant_is_packed(variant_) && n_ > chunk) {
      move_variant_ = variant_;
      move_tag_ = -1;
    }
    if (!chunk_user_set_ && (variant_is_gather(move_variant_) || variant_is_packed(move_variant_)))
      chunk = std::max(chunk, int32_t(1) << 21);
    rc = move_host(m.origin, m.dest, m.flying, m.weights, m.size, dev, chunk);
  }
  while (nsent > 0) PTB_CUDA_OK(cudaEventSynchronize(sent[--nsent]));  // the caller gets them back with the others
  if (rc == 0 && scored_move(t)) ++scored_moves_;
  return rc;
}

int Engine::move_host(const double *origin, const double *dest, int8_t *flying, const double *weights, int32_t size,
                      const MoveTally &dev, int32_t chunk) {
  const int nchunks = n_ ? (n_ + chunk - 1) / chunk : 0;
  while (int(chunk_events_.size()) < nchunks + 2) {
    cudaEvent_t e;
    PTB_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    chunk_events_.push_back(e);
  }
  if (register_host_) {  // opt-in: page-lock the caller's arrays the first time they are seen
    maybe_register(origin, 3 * size_t(n_) * sizeof(double));
    maybe_register(dest, 3 * size_t(n_) * sizeof(double));
    maybe_register(weights, size_t(n_) * sizeof(double));
    maybe_register(flying, size_t(n_));
  }
  // host_path 2 (default): staged, except that page-locked caller arrays (which the direct path can DMA
  // at the full PCIe rate without any host work) get the faster of the two, measured: moves 2-3 of every
  // 256 go direct, the others staged until the upload spans of both are known.  Where the host is the
  // scarce resource -- several ranks sharing one socket's memory system -- direct wins; with cores and
  // bandwidth to spare, staged does (DESIGN.md section 5).
  bool want_staged = host_path_ != 0;
  int probe = -1;
  if (host_path_ == 2 && host_is_pinned(origin) && host_is_pinned(dest) && host_is_pinned(weights) && host_is_pinned(flying)) {
    collect_upload_span();
    const uint64_t k = host_moves_ % 256;
    if (k == 0) { span_ms_[0] = span_ms_[1] = 0.0; span_n_[0] = span_n_[1] = 0; span_choice_ = -1; }
    if (k >= 2 && k <= 3) {
      probe = 1;
    } else if (k <= 1 || span_n_[0] == 0 || span_n_[1] == 0) {
      probe = 0;
    } else {
      // decided once per epoch, from the probe moves only: changing paths is not free (the first staged move
      // after a direct one has no mirror and sends every origin)
      if (span_choice_ < 0) {
        span_choice_ = (span_ms_[1] / span_n_[1] < 0.9 * span_ms_[0] / span_n_[0]) ? 1 : 0;
        if (std::getenv("PUMITALLY_DEBUG_SPANS"))
          fprintf(stderr, "[pumitally] staged %.3f ms, direct %.3f ms per move -> %s\n", span_ms_[0] / span_n_[0],
                  span_ms_[1] / span_n_[1], span_choice_ ? "direct" : "staged");
      }
      probe = span_choice_;
    }
    want_staged = probe == 0;
  }
  ++host_moves_;
  span_tag_ = probe;
  const bool staged = want_staged && n_ > 0 && ensure_stage_buffers(dest, size_t(size) * sizeof(double)) == 0 &&
                      ensure_patch_buffers(nchunks, chunk) == 0;
  if (!staged) return move_direct(origin, dest, flying, weights, nchunks, dev, chunk);
  follow_caller_memory(dest, size_t(size) * sizeof(double));
  // Caller arrays that are page-locked (by the caller, or just above) need no copy into the staging
  // slots: dest and weights go to the device straight from them, and the origins are compared with
  // the device's own particle positions, which each move sends back (move_pinned).  Plain moves only.
  const bool plain = dev.kind == MoveTally::kPlain && !dev.bins;
  if (pinned_path_ && plain && host_is_pinned(origin) && host_is_pinned(dest) && host_is_pinned(weights) &&
      ensure_position_mirror(nchunks) == 0)
    return move_pinned(origin, dest, flying, weights, nchunks, chunk);
  pos_mirror_valid_ = false;  // the move below does not send positions back

  // a chunk's staging slots may be refilled once the previous move's copies out of them are done;
  // with an unchanged chunking that is chunk_events_[k], otherwise wait for the whole copy stream
  if (staged_chunk_ != chunk || staged_chunks_ != nchunks) {
    PTB_CUDA_OK(cudaStreamSynchronize(copy_));
    staged_chunks_ = 0;
  }
  const bool compare = mirror_valid_;
  mirror_valid_ = false;  // until this move has gone through completely
  stager_->set_buffers(h_dest_, h_w_, h_fly_);
  cudaEvent_t ev_prev_done = chunk_events_[nchunks];
  // the device staging arrays are free once the previous move's kernels have finished
  PTB_CUDA_OK(cudaEventRecord(ev_prev_done, compute_));
  PTB_CUDA_OK(cudaStreamWaitEvent(copy_, ev_prev_done, 0));
  // the previous destinations, still on the device, are this move's origins before patching
  if (compare) std::swap(d_origin_, d_dest_);
  double sent = 0.0;
  bool caller_memory_on_the_wire = false;
  const auto t_begin = std::chrono::steady_clock::now();
  auto range_of = [&](int k, int32_t &b, int32_t &e) {
    b = int32_t(int64_t(k) * chunk);
    e = int32_t(std::min<int64_t>(n_, int64_t(b) + chunk));
  };
  // the staging slots of chunk k may be refilled once the previous move's copies out of them are done,
  // its pinned patch slot once the copies of chunk k - kPatchSlots of this move are done
  auto start_stage = [&](int k) -> int {
    if (k < staged_chunks_) PTB_CUDA_OK(cudaEventSynchronize(chunk_events_[k]));
    if (k >= kPatchSlots) PTB_CUDA_OK(cudaEventSynchronize(chunk_events_[k - kPatchSlots]));
    int32_t b, e;
    range_of(k, b, e);
    stager_->begin(origin, dest, flying, weights, b, e, compare, h_patch_ + size_t(k % kPatchSlots) * patch_cap_);
    return 0;
  };
  if (!ev_copy0_) {
    PTB_CUDA_OK(cudaEventCreate(&ev_copy0_));
    PTB_CUDA_OK(cudaEventCreate(&ev_copy1_));
  }
  PTB_CUDA_OK(cudaEventRecord(ev_copy0_, copy_));
  if (nchunks > 0 && start_stage(0)) return 1;
  for (int k = 0; k < nchunks; ++k) {
    int32_t b, e;
    range_of(k, b, e);
    const size_t cnt = size_t(e - b);
    const int64_t npatch = stager_->end();  // chunk k is staged
    // the workers stage chunk k+1 while this thread enqueues the copies and kernels of chunk k
    if (k + 1 < nchunks && start_stage(k + 1)) return 1;
    PatchEntry *hp = h_patch_ + size_t(k % kPatchSlots) * patch_cap_, *dp = d_patch_ + size_t(k) * patch_cap_;
    PTB_CUDA_OK(cudaMemcpyAsync(d_flying_ + b, h_fly_ + b, cnt, cudaMemcpyHostToDevice, copy_));
    if (!compare || npatch < 0) {  // no usable mirror, or too many changed origins: the slice travels whole
      PTB_CUDA_OK(cudaMemcpyAsync(d_origin_ + 3 * size_t(b), origin + 3 * size_t(b), 3 * cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
      sent += 24.0 * double(cnt);
      caller_memory_on_the_wire = true;
    } else if (npatch > 0) {
      PTB_CUDA_OK(cudaMemcpyAsync(dp, hp, size_t(npatch) * sizeof(PatchEntry), cudaMemcpyHostToDevice, copy_));
      sent += double(npatch) * sizeof(PatchEntry);
    }
    PTB_CUDA_OK(cudaMemcpyAsync(d_dest_ + 3 * size_t(b), h_dest_ + 3 * size_t(b), 3 * cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
    PTB_CUDA_OK(cudaMemcpyAsync(d_weights_ + b, h_w_ + b, cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
    sent += 33.0 * double(cnt);
    PTB_CUDA_OK(cudaEventRecord(chunk_events_[k], copy_));
    PTB_CUDA_OK(cudaStreamWaitEvent(compute_, chunk_events_[k], 0));
    if (compare && npatch > 0) {
      PTB_CUDA_OK(launch_patch_origins(d_origin_, dp, int32_t(npatch), compute_));
      ++launches_;
    }
    if (launch_range(d_origin_, d_dest_, d_flying_, d_weights_, b, e, compute_, dev)) return 1;
  }
  PTB_CUDA_OK(cudaEventRecord(ev_copy1_, copy_));
  if (mark_move_done()) return 1;
  // origin slices that went whole were read from the caller's own memory (asynchronously, if it is
  // pinned): they must be on the device before the caller gets its arrays back
  if (caller_memory_on_the_wire) PTB_CUDA_OK(cudaStreamSynchronize(copy_));
  stage_host_s_ = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  stage_sent_bytes_ = sent;
  h2d_bytes_ += sent;
  staged_chunk_ = chunk;
  staged_chunks_ = nchunks;
  mirror_valid_ = true;
  initial_weight_pending_ = false;
  ++moves_;
  return 0;
}

// Pinned mirror of the particle positions as the device holds them (x,y,z per particle, the layout of
// the caller's origin array), refreshed by every move of the pinned-caller path.
int Engine::ensure_position_mirror(int nchunks) {
  if (!h_pos_) {
    const size_t bytes = (3 * std::max<size_t>(size_t(n_), 1) * sizeof(double) + 4095) & ~size_t(4095);
    void *base = nullptr;
    if (posix_memalign(&base, 4096, bytes) == 0) {
      HostPool &pool = stager_->pool();
      const int T = pool.size();
      pool.run([&](int t) {
        const size_t lo = (bytes * size_t(t) / size_t(T)) & ~size_t(4095);
        const size_t hi = t == T - 1 ? bytes : (bytes * size_t(t + 1) / size_t(T)) & ~size_t(4095);
        std::memset(static_cast<char *>(base) + lo, 0, hi - lo);
      });
      if (cudaHostRegister(base, bytes, cudaHostRegisterDefault) != cudaSuccess) {
        cudaGetLastError();
        free(base);
        base = nullptr;
      }
    }
    if (!base) {
      pinned_path_ = false;  // no pinned memory for the mirror: the staged path serves pinned callers too
      return 1;
    }
    h_pos_ = static_cast<double *>(base);
    PTB_CUDA_OK(cudaStreamCreateWithFlags(&d2h_, cudaStreamNonBlocking));
  }
  while (int(pos_events_.size()) < nchunks) {
    cudaEvent_t a, b;
    PTB_CUDA_OK(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
    PTB_CUDA_OK(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
    pos_events_.push_back(a);
    walk_events_.push_back(b);
  }
  return 0;
}

// Host-pointer move when the caller's origin / dest / weights arrays are page-locked.
//
// Nothing is copied on the host except flying[] (1 byte per particle, so that it can be zeroed at
// once): dest and weights are DMA'd from the caller's arrays, chunk by chunk.  The origins are not
// sent at all; the pool compares them with h_pos_, the device's own particle positions as of the end
// of the previous move (exact bit patterns, hull clip points included), and only particles that fly
// from somewhere else are listed.  On the device the listed particles are relocated first (phase 1,
// tally off: relocate_patches), then the walk kernel runs with "origin == stored position" for every
// particle, then the chunk's new positions are exported and sent back on the otherwise idle
// device->host direction of the link.  Host memory traffic per particle: 24 B origin + 24 B mirror
// read by the pool, 33 B read and 24 B written by the DMA engines -- half of the staged path's.
int Engine::move_pinned(const double *origin, const double *dest, int8_t *flying, const double *weights,
                        int nchunks, int32_t chunk) {
  mirror_valid_ = false;  // the staged path's mirror does not see this move
  if (!ev_copy0_) {
    PTB_CUDA_OK(cudaEventCreate(&ev_copy0_));
    PTB_CUDA_OK(cudaEventCreate(&ev_copy1_));
  }
  if (staged_chunk_ != chunk || staged_chunks_ != nchunks || !pos_mirror_valid_) {
    PTB_CUDA_OK(cudaStreamSynchronize(copy_));
    PTB_CUDA_OK(cudaStreamSynchronize(d2h_));
    staged_chunks_ = 0;
  }
  if (!pos_mirror_valid_) {  // first move on this path, or moves in between that sent nothing back
    PTB_CUDA_OK(launch_export_positions(d_state_, d_origin_, 0, n_, compute_));
    PTB_CUDA_OK(cudaMemcpyAsync(h_pos_, d_origin_, 3 * size_t(n_) * sizeof(double), cudaMemcpyDeviceToHost, compute_));
    PTB_CUDA_OK(cudaStreamSynchronize(compute_));
    ++launches_;
  }
  pos_mirror_valid_ = false;  // until this move has gone through completely
  stager_->set_buffers(nullptr, nullptr, h_fly_, h_pos_);
  cudaEvent_t ev_prev_done = chunk_events_[nchunks];
  PTB_CUDA_OK(cudaEventRecord(ev_prev_done, compute_));
  PTB_CUDA_OK(cudaStreamWaitEvent(copy_, ev_prev_done, 0));
  double sent = 0.0;
  const auto t_begin = std::chrono::steady_clock::now();
  auto range_of = [&](int k, int32_t &b, int32_t &e) {
    b = int32_t(int64_t(k) * chunk);
    e = int32_t(std::min<int64_t>(n_, int64_t(b) + chunk));
  };
  auto start_stage = [&](int k) -> int {
    if (k < staged_chunks_) {
      PTB_CUDA_OK(cudaEventSynchronize(chunk_events_[k]));  // previous move's upload of the chunk's flying slots
      PTB_CUDA_OK(cudaEventSynchronize(pos_events_[k]));    // its positions are back
    }
    if (k >= kPatchSlots) PTB_CUDA_OK(cudaEventSynchronize(chunk_events_[k - kPatchSlots]));
    int32_t b, e;
    range_of(k, b, e);
    stager_->begin(origin, dest, flying, weights, b, e, true, h_patch_ + size_t(k % kPatchSlots) * patch_cap_);
    return 0;
  };
  PTB_CUDA_OK(cudaEventRecord(ev_copy0_, copy_));
  if (nchunks > 0 && start_stage(0)) return 1;
  for (int k = 0; k < nchunks; ++k) {
    int32_t b, e;
    range_of(k, b, e);
    const size_t cnt = size_t(e - b);
    const int64_t npatch = stager_->end();
    if (k + 1 < nchunks && start_stage(k + 1)) return 1;
    PatchEntry *hp = h_patch_ + size_t(k % kPatchSlots) * patch_cap_, *dp = d_patch_ + size_t(k) * patch_cap_;
    PTB_CUDA_OK(cudaMemcpyAsync(d_flying_ + b, h_fly_ + b, cnt, cudaMemcpyHostToDevice, copy_));
    if (npatch < 0) {  // most of the chunk was re-sourced: its origins travel whole, the kernel sorts them out
      PTB_CUDA_OK(cudaStreamWaitEvent(copy_, walk_events_[k], 0));  // d_origin_ doubles as the export buffer
      PTB_CUDA_OK(cudaMemcpyAsync(d_origin_ + 3 * size_t(b), origin + 3 * size_t(b), 3 * cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
      sent += 24.0 * double(cnt);
    } else if (npatch > 0) {
      PTB_CUDA_OK(cudaMemcpyAsync(dp, hp, size_t(npatch) * sizeof(PatchEntry), cudaMemcpyHostToDevice, copy_));
      sent += double(npatch) * sizeof(PatchEntry);
    }
    PTB_CUDA_OK(cudaMemcpyAsync(d_dest_ + 3 * size_t(b), dest + 3 * size_t(b), 3 * cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
    PTB_CUDA_OK(cudaMemcpyAsync(d_weights_ + b, weights + b, cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
    sent += 33.0 * double(cnt);
    PTB_CUDA_OK(cudaEventRecord(chunk_events_[k], copy_));
    PTB_CUDA_OK(cudaStreamWaitEvent(compute_, chunk_events_[k], 0));
    // the export below reuses d_origin_: the previous move's device->host copy out of it must be done
    PTB_CUDA_OK(cudaStreamWaitEvent(compute_, pos_events_[k], 0));
    if (npatch > 0 && relocate_patches(dp, int32_t(npatch), compute_)) return 1;
    if (launch_range(npatch < 0 ? d_origin_ : nullptr, d_dest_, d_flying_, d_weights_, b, e, compute_)) return 1;
    PTB_CUDA_OK(launch_export_positions(d_state_, d_origin_, b, e, compute_));
    ++launches_;
    PTB_CUDA_OK(cudaEventRecord(walk_events_[k], compute_));
    PTB_CUDA_OK(cudaStreamWaitEvent(d2h_, walk_events_[k], 0));
    static const bool debug_no_d2h = std::getenv("PUMITALLY_DEBUG_NO_D2H") != nullptr;  // timing experiments only: wrong results
    if (!debug_no_d2h)
    PTB_CUDA_OK(cudaMemcpyAsync(h_pos_ + 3 * size_t(b), d_origin_ + 3 * size_t(b), 3 * cnt * sizeof(double), cudaMemcpyDeviceToHost, d2h_));
    PTB_CUDA_OK(cudaEventRecord(pos_events_[k], d2h_));
  }
  PTB_CUDA_OK(cudaEventRecord(ev_copy1_, copy_));
  if (mark_move_done()) return 1;
  // dest and weights are read from the caller's own arrays: they must be on the device before the
  // caller gets them back (reference: blocking deep_copy)
  PTB_CUDA_OK(cudaStreamSynchronize(copy_));
  stage_host_s_ = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  stage_sent_bytes_ = sent;
  h2d_bytes_ += sent;
  d2h_bytes_ += 24.0 * double(n_);
  staged_chunk_ = chunk;
  staged_chunks_ = nchunks;
  pos_mirror_valid_ = true;
  initial_weight_pending_ = false;
  ++moves_;
  return 0;
}

// Device time the previous host move's uploads took (first copy could start -> last copy done), credited to
// the path that move used; feeds the staged-vs-direct choice for page-locked caller arrays.
void Engine::collect_upload_span() {
  if (span_tag_ < 0 || !ev_copy0_) return;
  if (span_choice_ >= 0) { span_tag_ = -1; return; }  // decided for this epoch
  float ms = 0.f;
  if (ev_done_ && cudaEventSynchronize(ev_done_) == cudaSuccess && cudaEventElapsedTime(&ms, ev_copy0_, ev_done_) == cudaSuccess) {
    span_ms_[span_tag_] += ms;
    ++span_n_[span_tag_];
    if (std::getenv("PUMITALLY_DEBUG_SPANS"))
      fprintf(stderr, "[pumitally] host move %llu: %s path, uploads + walk %.3f ms on the device\n",
              (unsigned long long)host_moves_ - 1, span_tag_ ? "direct" : "staged", ms);
  } else {
    cudaGetLastError();
  }
  span_tag_ = -1;
}

// marks the end of a host move's device work (after its last kernel): what collect_upload_span() measures up to
int Engine::mark_move_done() {
  if (!ev_done_) PTB_CUDA_OK(cudaEventCreate(&ev_done_));
  PTB_CUDA_OK(cudaEventRecord(ev_done_, compute_));
  return 0;
}

// Direct path: every array is copied from the caller's memory as it is.
int Engine::move_direct(const double *origin, const double *dest, int8_t *flying, const double *weights,
                        int nchunks, const MoveTally &dev, int32_t chunk) {
  mirror_valid_ = false;  // the staging slots do not see this move
  pos_mirror_valid_ = false;
  cudaEvent_t ev_prev_done = chunk_events_[nchunks], ev_fly = chunk_events_[nchunks + 1];
  PTB_CUDA_OK(cudaStreamSynchronize(copy_));  // staged copies of an earlier move
  staged_chunks_ = 0;
  PTB_CUDA_OK(cudaEventRecord(ev_prev_done, compute_));
  PTB_CUDA_OK(cudaStreamWaitEvent(copy_, ev_prev_done, 0));
  if (!ev_copy0_) {
    PTB_CUDA_OK(cudaEventCreate(&ev_copy0_));
    PTB_CUDA_OK(cudaEventCreate(&ev_copy1_));
  }
  PTB_CUDA_OK(cudaEventRecord(ev_copy0_, copy_));
  PTB_CUDA_OK(cudaMemcpyAsync(d_flying_, flying, size_t(n_), cudaMemcpyHostToDevice, copy_));
  PTB_CUDA_OK(cudaEventRecord(ev_fly, copy_));
  for (int k = 0; k < nchunks; ++k) {
    const int32_t b = int32_t(int64_t(k) * chunk), e = int32_t(std::min<int64_t>(n_, int64_t(b) + chunk));
    const size_t cnt = size_t(e - b);
    PTB_CUDA_OK(cudaMemcpyAsync(d_origin_ + 3 * size_t(b), origin + 3 * size_t(b), 3 * cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
    PTB_CUDA_OK(cudaMemcpyAsync(d_dest_ + 3 * size_t(b), dest + 3 * size_t(b), 3 * cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
    PTB_CUDA_OK(cudaMemcpyAsync(d_weights_ + b, weights + b, cnt * sizeof(double), cudaMemcpyHostToDevice, copy_));
    PTB_CUDA_OK(cudaEventRecord(chunk_events_[k], copy_));
    PTB_CUDA_OK(cudaStreamWaitEvent(compute_, chunk_events_[k], 0));
    if (launch_range(d_origin_, d_dest_, d_flying_, d_weights_, b, e, compute_, dev)) return 1;
  }
  PTB_CUDA_OK(cudaEventRecord(ev_copy1_, copy_));
  if (mark_move_done()) return 1;
  h2d_bytes_ += 57.0 * double(n_);
  stage_sent_bytes_ = 57.0 * double(n_);
  // reset the caller's flags once they are on the device (PumiTallyImpl.cpp:169-172)
  PTB_CUDA_OK(cudaEventSynchronize(ev_fly));
  if (n_) std::memset(flying, 0, size_t(n_));
  // caller may reuse its buffers on return (reference: blocking deep_copy)
  PTB_CUDA_OK(cudaStreamSynchronize(copy_));
  initial_weight_pending_ = false;
  ++moves_;
  return 0;
}

// The refusals every move kind shares; `device`: the device-pointer entry point's name in the message.
bool Engine::move_refused(const Move &m, bool device) const {
  static const char *const names[] = {"MoveToNextLocation", "MoveToNextLocationScored", "MoveToNextLocationTimed"};
  const MoveTally &t = m.tally;
  const char *why = nullptr;
  if (t.kind == MoveTally::kTimed) {
    if (ntime_ == 0) why = "the engine has no time bins (set_time_bins)";
    else if (!t.times || !t.speeds) why = "null times or speeds array";
    else if (!t.responses && nscores_ != 1) why = "null responses array with several scores";
  } else if (ntime_ > 0) {
    why = "the engine has time bins; use the timed move";
  } else if (t.kind == MoveTally::kScored && !t.responses) {
    why = "null responses array";
  } else if (t.kind == MoveTally::kPlain && nscores_ != 1) {
    why = "the engine has several scores; use the scored move";
  }
  if (!why && int64_t(m.size) != 3 * int64_t(n_)) why = "size != 3 * num_particles";
  if (!why && !initialized_) why = "called before CopyInitialPosition";
  if (why) fprintf(stderr, "[pumitally] ERROR: %s%s: %s\n", names[t.kind], device ? "(device)" : "", why);
  return why != nullptr;
}

int Engine::move_to_next_location_device(const Move &m, cudaStream_t stream) {
  if (move_refused(m, true)) return 1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  tallied_ = true;
  const bool scored = scored_move(m.tally);
  begin_move(scored);
  // (the staging arrays are not touched: "pinned dest slots == device dest array" keeps holding, and the
  // next host move's origins are compared against them and patched exactly as after a host move;
  // the position mirror of the pinned-caller path, however, is out of date after this move)
  pos_mirror_valid_ = false;
  MoveTally dev = m.tally;
  if (nbins_ == 1) dev.bins = nullptr;
  if (launch_range(m.origin, m.dest, m.flying, m.weights, 0, n_, stream, dev)) return 1;
  initial_weight_pending_ = false;
  ++moves_;
  if (scored) ++scored_moves_;
  return 0;
}

// Score filter (SURVEY section 8 f4; OpenMC: an energy / material / ... filter on the tally).  nbins flux
// arrays of E doubles, bin-major, plus one unreported array for the particles no bin matches.
int Engine::set_score_bins(int32_t nbins) {
  if (nbins < 1 || nbins > 4096) return 1;
  if (nccl_comm_) {
    fprintf(stderr, "[pumitally] ERROR: set_score_bins after comm_init (the exchange buffers are sized by then)\n");
    return 1;
  }
  return resize_flux(nbins, nscores_, ntime_, moments_, collision_, currents_, nmu_);
}

// Scores (walk_core.cuh, ScoreParams): the flux array becomes [bin][element][score_stride(nscores)].
int Engine::set_scores(int32_t nscores) {
  if (nscores < 1 || nscores > kMaxScores) return 1;
  if (nccl_comm_) {
    fprintf(stderr, "[pumitally] ERROR: set_scores after comm_init (the exchange buffers are sized by then)\n");
    return 1;
  }
  return resize_flux(nbins_, nscores, ntime_, moments_, collision_, currents_, nmu_);
}

// Time filter (walk_core.cuh, TimeParams): the flux array becomes [time][bin][element][stride], the edges live on
// the device.  Nothing changes unless the edges are valid and the new array can be allocated.
int Engine::set_time_bins(const double *edges, int32_t nedges) {
  if (nccl_comm_) {
    fprintf(stderr, "[pumitally] ERROR: set_time_bins after comm_init (the exchange buffers are sized by then)\n");
    return 1;
  }
  if (!edges && nedges == 0) {  // no time filter
    if (resize_flux(nbins_, nscores_, 0, moments_, collision_, currents_, nmu_)) return 1;
    cudaFree(d_edges_);
    d_edges_ = nullptr;
    return 0;
  }
  if (!edges || nedges < 2 || nedges - 1 > kMaxTimeBins) return 1;
  for (int32_t j = 0; j < nedges; ++j)
    if (!std::isfinite(edges[j]) || (j > 0 && !(edges[j] > edges[j - 1]))) return 1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  double *ne = nullptr;
  if (cudaMalloc(reinterpret_cast<void **>(&ne), size_t(nedges) * sizeof(double)) != cudaSuccess) {
    cudaGetLastError();
    return 1;
  }
  if (cudaMemcpy(ne, edges, size_t(nedges) * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
      resize_flux(nbins_, nscores_, nedges - 1, moments_, collision_, currents_, nmu_)) {
    cudaGetLastError();
    cudaFree(ne);
    return 1;
  }
  cudaFree(d_edges_);
  d_edges_ = ne;
  return 0;
}

// Linear moments (walk_core.cuh, moment_tally): the element's record grows from S to kMomentSlots * S doubles.
int Engine::set_moments(int32_t order) {
  if (order != 0 && order != 1) return 1;
  if (nccl_comm_) {
    fprintf(stderr, "[pumitally] ERROR: set_moments after comm_init (the exchange buffers are sized by then)\n");
    return 1;
  }
  return resize_flux(nbins_, nscores_, ntime_, order, collision_, currents_, nmu_);
}

// Collision estimator (walk_core.cuh, collision_event): a second tally of the same layout after the track-length one.
int Engine::set_collision_estimator(int32_t on) {
  if (on != 0 && on != 1) return 1;
  if (nccl_comm_) {
    fprintf(stderr, "[pumitally] ERROR: set_collision_estimator after comm_init (the exchange buffers are sized by then)\n");
    return 1;
  }
  return resize_flux(nbins_, nscores_, ntime_, moments_, on != 0, currents_, nmu_);
}

// Face currents (walk_core.cuh, CurrentParams): the current slots and the leakage slots after both tallies.
int Engine::set_face_currents(int32_t on) {
  if (on != 0 && on != 1) return 1;
  if (nccl_comm_) {
    fprintf(stderr, "[pumitally] ERROR: set_face_currents after comm_init (the exchange buffers are sized by then)\n");
    return 1;
  }
  if (resize_flux(nbins_, nscores_, ntime_, moments_, collision_, on != 0, nmu_)) return 1;
  if (!on) free_region_currents();  // (their statistics went with the batches resize_flux discarded)
  return 0;
}

// Cosine bins (walk_core.cuh, CurrentParams, MU): the current block becomes [time][bin][cosine][element][4], with
// [time][bin][cosine] leakage slots, and the edges live on the device.  Nothing changes unless the edges are valid and
// the new arrays can be allocated.  Region currents keep their pair plan; their lengths follow cur_arrays().
int Engine::set_current_cosine_bins(const double *edges, int32_t nedges) {
  const char *why = nccl_comm_ ? "after comm_init (the exchange buffers are sized by then)"
                    : (!edges && nedges == 0) ? nullptr
                    : (!edges || nedges < 2 || nedges - 1 > kMaxCosineBins)
                        ? "nedges must be 2..65 (1..64 cosine bins), or edges NULL with nedges 0"
                        : nullptr;
  for (int32_t j = 0; !why && edges && j < nedges; ++j)
    if (!std::isfinite(edges[j]) || edges[j] < 0.0 || edges[j] > 1.0 || (j > 0 && !(edges[j] > edges[j - 1])))
      why = "the edges must be finite, in [0, 1] and strictly increasing";
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: set_current_cosine_bins: %s\n", why);
    return 1;
  }
  const int32_t nmu = edges ? nedges - 1 : 0;
  double *ne = nullptr;
  if (nmu > 0) {
    PTB_CUDA_OK(cudaSetDevice(device_));
    if (cudaMalloc(reinterpret_cast<void **>(&ne), size_t(nedges) * sizeof(double)) != cudaSuccess ||
        cudaMemcpy(ne, edges, size_t(nedges) * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess) {
      cudaGetLastError();
      cudaFree(ne);
      return 1;
    }
  }
  if (resize_flux(nbins_, nscores_, ntime_, moments_, collision_, currents_, nmu)) {
    cudaFree(ne);
    return 1;
  }
  cudaFree(d_mu_edges_);
  d_mu_edges_ = ne;
  mu_edges_.assign(edges, edges + (nmu > 0 ? nedges : 0));
  return 0;
}

int Engine::resize_flux(int32_t nbins, int32_t nscores, int32_t ntime, int32_t moments, bool collision, bool currents,
                        int32_t nmu) {
  if (synchronize()) return 1;
  const size_t E = size_t(mesh_.ntets), stride = size_t(score_stride(nscores)) * (moments ? kMomentSlots : 1);
  // [time][bin][element][stride], the collision tally of the same layout, with face currents
  // [time][bin][cosine][element][4] and [time][bin][cosine] leakage slots, then the unreported array of the particles no
  // bin matches (and its currents, every cosine bin in one)
  const size_t arrays = size_t(ntime > 0 ? ntime : 1) * size_t(nbins);
  const size_t tally = arrays * (collision ? 2 : 1);
  const size_t reported = tally * E * stride + (currents ? arrays * size_t(nmu > 0 ? nmu : 1) * (4 * E + 1) : 0);
  const size_t len = reported + (nbins > 1 ? E * stride + (currents ? 4 * E : 0) : 0) + kFluxPad;
  double *nf = nullptr;
  const cudaError_t err = cudaMalloc(reinterpret_cast<void **>(&nf), len * sizeof(double));
  if (err != cudaSuccess) {
    cudaGetLastError();
    fprintf(stderr, "[pumitally] ERROR: no device memory for a flux array of %zu doubles (%s)\n", len,
            cudaGetErrorString(err));
    return 1;
  }
  double *nd = nullptr;  // the detector tally [time][bin][score][detector] of the new layout
  const int det_rc = ndet_ > 0 ? alloc_detectors(arrays * size_t(nscores) * size_t(ndet_), batch_stats_, &nd) : 0;
  if (det_rc || (batch_stats_ && alloc_stats(reported))) {  // statistics of the new layout, no batch folded yet
    cudaFree(nf);
    cudaFree(nd);
    return 1;
  }
  if (ndet_ > 0) {
    cudaFree(d_det_);
    d_det_ = nd;
  }
  if (nbins != sigma_bins_) {  // a table of another number of groups no longer applies
    cudaFree(d_sigma_);
    d_sigma_ = nullptr;
    sigma_bins_ = 0;
  }
  cudaFree(d_flux_);
  d_flux_ = nf;
  flux_alloc_ = len;
  nbins_ = nbins;
  nscores_ = nscores;
  stride_ = int32_t(stride);
  ntime_ = ntime;
  moments_ = moments;
  collision_ = collision;
  currents_ = currents;
  nmu_ = nmu;
  if (nbins > 1 && !d_mask_) PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_mask_), std::max<size_t>(size_t(n_), 16)));
  return reset_tally();  // a new set of arrays starts from zero
}

// A side array of a host-pointer move, a and, if not null, b (bytes each) back to back in u.d: one copy ahead of the
// particle data on the copy stream, through a pinned copy the worker pool makes when a caller's array is pageable (a
// pageable cudaMemcpyAsync of 40 MB blocks this thread for milliseconds before the staging of the particle data can
// even start).  u.ev is recorded after the copy.
int Engine::upload_aux(AuxUpload &u, const void *a, const void *b, size_t bytes) {
  PTB_CUDA_OK(cudaSetDevice(device_));
  const size_t total = bytes * (b ? 2 : 1);
  if (u.cap < total) {
    PTB_CUDA_OK(cudaDeviceSynchronize());
    cudaFree(u.d);
    if (u.h) cudaFreeHost(u.h);
    u.d = u.h = nullptr;
    u.cap = 0;
    PTB_CUDA_OK(cudaMalloc(&u.d, std::max<size_t>(total, 1)));
    u.cap = total;
  }
  if (!u.ev) PTB_CUDA_OK(cudaEventCreateWithFlags(&u.ev, cudaEventDisableTiming));
  // u.d is read by the previous move's kernels until they are done
  PTB_CUDA_OK(cudaEventRecord(u.ev, compute_));
  PTB_CUDA_OK(cudaStreamWaitEvent(copy_, u.ev, 0));
  const void *src[2] = {a, b};
  const int narr = b ? 2 : 1;
  bool staged = false;
  if (!host_is_pinned(a) || (b && !host_is_pinned(b))) {
    if (!u.h && cudaHostAlloc(&u.h, std::max<size_t>(u.cap, 1), cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      u.h = nullptr;
    }
    if (u.h) {  // the previous move's DMA out of it was waited for before that move returned
      for (int k = 0; k < narr; ++k) pool_copy(static_cast<char *>(u.h) + size_t(k) * bytes, src[k], bytes);
      PTB_CUDA_OK(cudaMemcpyAsync(u.d, u.h, total, cudaMemcpyHostToDevice, copy_));
      staged = true;
    }
  }
  if (!staged)
    for (int k = 0; k < narr; ++k)
      PTB_CUDA_OK(cudaMemcpyAsync(static_cast<char *>(u.d) + size_t(k) * bytes, src[k], bytes, cudaMemcpyHostToDevice, copy_));
  PTB_CUDA_OK(cudaEventRecord(u.ev, copy_));
  h2d_bytes_ += double(total);
  return 0;
}

void Engine::pool_copy(void *dst, const void *src, size_t bytes) {
  if (!stager_) {  // (the pool exists from the first staged move on)
    std::memcpy(dst, src, bytes);
    return;
  }
  HostPool &pool = stager_->pool();
  const size_t T = size_t(pool.size());
  pool.run([&](int t) {  // 64-byte pieces
    const size_t lo = (bytes * size_t(t) / T) & ~size_t(63), hi = size_t(t) == T - 1 ? bytes : (bytes * size_t(t + 1) / T) & ~size_t(63);
    std::memcpy(static_cast<char *>(dst) + lo, static_cast<const char *>(src) + lo, hi - lo);
  });
}

int Engine::synchronize() {
  PTB_CUDA_OK(cudaSetDevice(device_));
  PTB_CUDA_OK(cudaDeviceSynchronize());
  return 0;
}

int Engine::ensure_element_maps() {
  if (d_orig_of_internal_) return 0;
  const size_t E = std::max<size_t>(size_t(mesh_.ntets), 1);
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_orig_of_internal_), E * sizeof(int32_t)));
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_internal_of_orig_), E * sizeof(int32_t)));
  PTB_CUDA_OK(cudaMemcpy(d_orig_of_internal_, mesh_.orig_of_internal.data(), size_t(mesh_.ntets) * sizeof(int32_t), cudaMemcpyHostToDevice));
  PTB_CUDA_OK(cudaMemcpy(d_internal_of_orig_, mesh_.internal_of_orig.data(), size_t(mesh_.ntets) * sizeof(int32_t), cudaMemcpyHostToDevice));
  return 0;
}

// Places particles [first, first + count) at given positions in given elements (caller's numbering)
// without walking there: for drivers that hand particles between engines (spatial partition).  The
// elements are trusted to contain the positions.
int Engine::set_state_device(const double *d_xyz, const int32_t *d_elem, int32_t first, int32_t count, cudaStream_t stream) {
  if (first < 0 || count < 0 || int64_t(first) + count > n_) return 1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (ensure_element_maps()) return 1;
  PTB_CUDA_OK(launch_set_state(d_state_, d_xyz, d_elem, d_internal_of_orig_, first, first + count, stream));
  initialized_ = true;
  mirror_valid_ = false;
  pos_mirror_valid_ = false;
  return 0;
}

int Engine::get_state_device(double *d_xyz, int32_t *d_elem, int32_t first, int32_t count, cudaStream_t stream) {
  if (first < 0 || count < 0 || int64_t(first) + count > n_) return 1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (ensure_element_maps()) return 1;
  PTB_CUDA_OK(launch_get_state(d_state_, d_xyz, d_elem, d_orig_of_internal_, first, first + count, stream));
  return 0;
}

// (all time bins, score bins and scores: ntime * nbins * nscores * E values, [time][bin][score][element])
int Engine::get_flux_device(double *d_out, cudaStream_t stream) {
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (ensure_element_maps() || gather_shares()) return 1;
  const size_t E = size_t(mesh_.ntets);
  if (multi_results()) {
    for (int32_t b = 0; b < result_arrays(); ++b)
      PTB_CUDA_OK(launch_scores_to_caller_order(flux_view() + size_t(b) * bin_len(), d_orig_of_internal_,
                                                d_out + size_t(b) * size_t(nscores_) * E, mesh_.ntets, nscores_, stride_, stream));
    return 0;
  }
  for (int32_t b = 0; b < nbins_; ++b)
    PTB_CUDA_OK(launch_flux_to_caller_order(flux_view() + size_t(b) * E, d_orig_of_internal_, d_out + size_t(b) * E, mesh_.ntets, stream));
  return 0;
}

// Every time bin, bin and score of the tally, [time][bin][score][element] in the caller's numbering: raw, or
// normalised as get_normalized_flux does it.  (Time bin t of bin b is internal array t * nbins + b.)
int Engine::copy_results(std::vector<double> &out, bool normalized, size_t base) {
  const size_t E = size_t(mesh_.ntets), S = size_t(nscores_), B = size_t(result_arrays());
  double per_source = 1.0;
  if (normalized && !per_source_divisor(&per_source)) return 1;
  if (ensure_element_maps()) return 1;
  double *d_tmp = nullptr;
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_tmp), std::max<size_t>(S * E, 1) * sizeof(double)));
  out.resize(B * S * E);
  std::vector<double> tmp(S * E);
  int rc = 0;
  for (size_t b = 0; b < B && !rc; ++b) {
    const double *f = flux_view() + base + b * bin_len();
    cudaError_t e = normalized ? launch_normalize_scores(f, d_volume_, d_tmp, int64_t(E), nscores_, stride_, per_source, compute_)
                               : launch_scores_to_caller_order(f, d_orig_of_internal_, d_tmp, int64_t(E), nscores_, stride_, compute_);
    if (e == cudaSuccess) e = cudaStreamSynchronize(compute_);
    if (e == cudaSuccess) e = cudaMemcpy(normalized ? tmp.data() : out.data() + b * S * E, d_tmp, S * E * sizeof(double), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) {
      fprintf(stderr, "[pumitally] CUDA error %s reading the scores\n", cudaGetErrorString(e));
      rc = 1;
    } else if (normalized) {
      for (size_t k = 0; k < S; ++k)
        for (size_t i = 0; i < E; ++i) out[(b * S + k) * E + size_t(mesh_.orig_of_internal[i])] = tmp[k * E + i];
    }
  }
  cudaFree(d_tmp);
  return rc;
}

// n == E: the first (or only) score bin (score 0, time bin 0); n == ntime * nbins * nscores * E: everything,
// [time][bin][score][element]
int Engine::get_flux(double *out, int64_t n) {
  const int64_t E = mesh_.ntets;
  if (multi_results()) {
    if (n != E && n != int64_t(result_arrays()) * nscores_ * E) return 1;
    if (synchronize() || gather_shares()) return 1;
    std::vector<double> all;
    if (copy_results(all, false)) return 1;
    std::memcpy(out, all.data(), size_t(n) * sizeof(double));
    return 0;
  }
  if (n != E && n != int64_t(nbins_) * E) return 1;
  if (synchronize() || gather_shares()) return 1;
  std::vector<double> tmp(static_cast<size_t>(n));
  PTB_CUDA_OK(cudaMemcpy(tmp.data(), flux_view(), size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  for (int64_t b = 0; b * E < n; ++b)
    for (int64_t i = 0; i < E; ++i) out[b * E + mesh_.orig_of_internal[i]] = tmp[b * E + i];  // caller's numbering
  return 0;
}

// The linear moments of every result array, [time][bin][score][element][3] in the caller's numbering: m1 about each
// element's centroid, or the gradient g = M^-1 m1 divided by the source normalisation (linear_moments()).
int Engine::copy_moments(std::vector<double> &out, bool gradient, size_t base, const double *src) {
  const size_t E = size_t(mesh_.ntets), S = size_t(nscores_), B = size_t(result_arrays());
  const int slot = stride_ / kMomentSlots;
  double per_source = 1.0;
  if (gradient && !src && !per_source_divisor(&per_source)) return 1;
  std::vector<double> raw(B * bin_len());
  PTB_CUDA_OK(cudaMemcpy(raw.data(), (src ? src : flux_view()) + base, raw.size() * sizeof(double), cudaMemcpyDeviceToHost));
  out.resize(B * S * E * 3);
  const double *xyz = mesh_.coords.data();
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < int64_t(E); ++i) {
    double v[12];
    for (int q = 0; q < 4; ++q)
      for (int a = 0; a < 3; ++a) v[3 * q + a] = xyz[3 * size_t(mesh_.t2v[4 * i + q]) + a];
    const size_t o = size_t(mesh_.orig_of_internal[i]);
    for (size_t b = 0; b < B; ++b)
      for (size_t k = 0; k < S; ++k) {
        double m1[3], g[3];
        linear_moments(v, mesh_.center, raw.data() + b * bin_len() + size_t(i) * size_t(stride_), slot, int(k), m1, g);
        double *dst = out.data() + ((b * S + k) * E + o) * 3;
        for (int a = 0; a < 3; ++a) dst[a] = gradient ? g[a] / per_source : m1[a];
      }
  }
  return 0;
}

// n == 3E: time bin 0, bin 0, score 0; n == 3 * ntime * nbins * nscores * E: everything
int Engine::get_moments_entry(double *out, int64_t n, bool gradient, size_t base) {
  const int64_t E = mesh_.ntets;
  if (!moments_) {
    fprintf(stderr, "[pumitally] ERROR: the engine tallies no moments (set_moments)\n");
    return 1;
  }
  if (n != 3 * E && n != 3 * int64_t(result_arrays()) * nscores_ * E) return 1;
  if (synchronize() || gather_shares()) return 1;
  std::vector<double> all;
  if (copy_moments(all, gradient, base)) return 1;
  std::memcpy(out, all.data(), size_t(n) * sizeof(double));
  return 0;
}

int Engine::get_flux_moments(double *out, int64_t n) { return get_moments_entry(out, n, false); }
int Engine::get_flux_gradient(double *out, int64_t n) { return get_moments_entry(out, n, true); }

// The collision tally read as the track-length one is, through the general ([time][bin][score][element]) path.
int Engine::get_collision_results(int32_t kind, double *out, int64_t n) {
  if (!collision_) {
    fprintf(stderr, "[pumitally] ERROR: the collision estimator is off (set_collision_estimator)\n");
    return 1;
  }
  if (kind == 2 || kind == 3) return get_moments_entry(out, n, kind == 3, flux_len());
  if (kind != 0 && kind != 1) return 1;
  const int64_t E = mesh_.ntets;
  if (n != E && n != int64_t(result_arrays()) * nscores_ * E) return 1;
  if (synchronize() || gather_shares()) return 1;
  std::vector<double> all;
  if (copy_results(all, kind == 1, flux_len())) return 1;
  std::memcpy(out, all.data(), size_t(n) * sizeof(double));
  return 0;
}

// NormalizeFlux (PumiTallyImpl.cpp:382-409); n as for get_flux (the volumes are always E values)
int Engine::get_normalized_flux(double *out_flux, double *out_volume, int64_t n) {
  const int64_t E = mesh_.ntets;
  if (multi_results()) {
    if (n != E && n != int64_t(result_arrays()) * nscores_ * E) return 1;
    if (synchronize() || gather_shares()) return 1;
    if (out_flux) {
      std::vector<double> all;
      if (copy_results(all, true)) return 1;
      std::memcpy(out_flux, all.data(), size_t(n) * sizeof(double));
    }
    if (out_volume)
      for (int64_t i = 0; i < E; ++i) out_volume[mesh_.orig_of_internal[i]] = mesh_.volume[i];
    return 0;
  }
  if (n != E && n != int64_t(nbins_) * E) return 1;
  if (synchronize() || gather_shares()) return 1;
  if (out_flux) {
    double per_source = 1.0;
    if (!per_source_divisor(&per_source)) return 1;
    std::vector<double> tmp(static_cast<size_t>(E));
    for (int64_t b = 0; b * E < n; ++b) {
      PTB_CUDA_OK(launch_normalize(flux_view() + size_t(b * E), d_volume_, d_scratch_, E, per_source, compute_));
      PTB_CUDA_OK(cudaStreamSynchronize(compute_));
      PTB_CUDA_OK(cudaMemcpy(tmp.data(), d_scratch_, size_t(E) * sizeof(double), cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < E; ++i) out_flux[b * E + mesh_.orig_of_internal[i]] = tmp[i];
    }
  }
  if (out_volume)
    for (int64_t i = 0; i < E; ++i) out_volume[mesh_.orig_of_internal[i]] = mesh_.volume[i];
  return 0;
}

int Engine::get_element_ids(int32_t *out, int64_t n) {
  if (n != n_) return 1;
  if (synchronize()) return 1;
  std::vector<ParticleState> tmp(static_cast<size_t>(n_));
  PTB_CUDA_OK(cudaMemcpy(tmp.data(), d_state_, size_t(n_) * sizeof(ParticleState), cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < n_; ++i) out[i] = mesh_.orig_of_internal[tmp[i].elem];  // caller's numbering
  return 0;
}

int Engine::get_positions(double *out, int64_t n3) {
  if (n3 != 3 * int64_t(n_)) return 1;
  if (synchronize()) return 1;
  std::vector<ParticleState> tmp(static_cast<size_t>(n_));
  PTB_CUDA_OK(cudaMemcpy(tmp.data(), d_state_, size_t(n_) * sizeof(ParticleState), cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < n_; ++i) {
    out[3 * i] = tmp[i].x;
    out[3 * i + 1] = tmp[i].y;
    out[3 * i + 2] = tmp[i].z;
  }
  return 0;
}

int Engine::set_source_normalization(int mode, double value) {
  if (mode < 0 || mode > 3 || (mode == 2 && !(value > 0.0))) return 1;
  norm_mode_ = mode;
  norm_value_ = value;
  eval_valid_ = false;
  return 0;
}

double Engine::source_normalization() {
  switch (norm_mode_) {
    case 1: return double(std::max(n_, 1));
    case 2: return norm_value_;
    case 3: {
      double w = 0.0;
      cudaDeviceSynchronize();
      if (cudaMemcpy(&w, d_initial_weight_, sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) return 0.0;
      return w;
    }
    default: return 1.0;
  }
}

bool Engine::per_source_divisor(double *out) {
  *out = source_normalization();
  if (*out > 0.0) return true;
  fprintf(stderr, "[pumitally] ERROR: source normalisation divisor is %g (no source weight seen yet?)\n", *out);
  return false;
}

int Engine::reset_tally() {
  if (synchronize()) return 1;
  collect_timers(true);
  PTB_CUDA_OK(cudaMemset(d_initial_weight_, 0, sizeof(double)));
  initial_weight_pending_ = true;
  PTB_CUDA_OK(cudaMemset(d_flux_, 0, flux_alloc_ * sizeof(double)));
  scored_moves_ = 0;
  PTB_CUDA_OK(cudaMemset(d_stats_, 0, sizeof(DeviceStats)));
  PTB_CUDA_OK(cudaMemset(d_coll_counts_, 0, 3 * sizeof(unsigned long long)));
  PTB_CUDA_OK(cudaMemset(d_det_counts_, 0, kDetCountersVoid * sizeof(unsigned long long)));
  if (ndet_ > 0) PTB_CUDA_OK(cudaMemset(d_det_, 0, 2 * det_len() * sizeof(double)));
  det_global_valid_ = false;
  flux_global_valid_ = flux_owned_only_ = eval_valid_ = tallied_ = false;
  kernel_ms_ = 0.0;
  h2d_bytes_ = 0.0;
  moves_ = 0;
  return 0;
}

int Engine::get_stats(EngineStats *out) {
  if (synchronize()) return 1;
  collect_timers(true);
  DeviceStats s;
  PTB_CUDA_OK(cudaMemcpy(&s, d_stats_, sizeof(s), cudaMemcpyDeviceToHost));
  out->segments = s.segments;
  out->tracks = s.tracks;
  out->relocations = s.relocations;
  out->lost = s.lost;
  out->moves = moves_;
  out->kernel_ms = kernel_ms_;
  out->h2d_bytes = h2d_bytes_;
  out->plane_fallbacks = s.fallbacks;
  if (s.lost)  // reference wording, PumiTallyImpl.cpp:455-458
    printf("ERROR: Not all particles are found. May need more loops in search\n");
  return 0;
}

// While the tet table still half-fits the L2, streaming the particles in storage order through the TMA
// stages is fastest.  Once the table is more than twice the L2, most record fetches are random 32-byte
// DRAM accesses and processing the particles in spatial order (binning pass + gather staging) pays for
// itself: on an H100 (50 MB of L2) that is already config c2 (128 MB of records; 6.3 ms per move against
// 18.2 ms streaming, 400 W card) and config c5 (1.26 GB).
int Engine::choose_variant() const {
  int l2 = 0;
  cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, device_);
  const double table = double(mesh_.ntets) * sizeof(TetRecord);
  return (l2 > 0 && table > 2.0 * double(l2)) ? kVariantPersistGatherL1 : kVariantPersistRefill8;
}

int64_t Engine::get_option(const std::string &name) const {
  if (name == "variant")  // the kernel the next move will use outside the auto-tuner's exploration moves
    return (auto_variant_ && autotune_ && variant_ == kVariantPersistRefill8) ? tuned_variant_ : variant_;
  if (name == "launches") return int64_t(launches_);
  if (name == "autotune") return autotune_ ? 1 : 0;
  if (name == "block") return block_;
  if (name == "chunk") return chunk_;
  if (name == "seed_grid") return seed_grid_mode_;
  if (name == "seed_grid_active") return use_seed_grid_ ? 1 : 0;
  if (name == "hull_convex") return mesh_.hull_convex ? 1 : 0;
  if (name == "bin_midpoint") return bin_midpoint_ ? 1 : 0;
  if (name == "max_iters") return max_iters_;
  if (name == "l2_fetch") {
    size_t g = 0;
    return cudaDeviceGetLimit(&g, cudaLimitMaxL2FetchGranularity) == cudaSuccess ? int64_t(g) : -1;
  }
  if (name == "allreduce_us") return int64_t(allreduce_ms_ * 1e3);  // device time of the last batch-end exchange
  if (name == "score_bins") return nbins_;
  if (name == "scores") return nscores_;
  if (name == "time_bins") return ntime_;
  if (name == "moments") return moments_;
  if (name == "locate_candidates") return int64_t(cand_entries_);  // entries of the point-location candidate lists
  if (name == "collision_estimator") return collision_ ? 1 : 0;
  if (name == "face_currents") return currents_ ? 1 : 0;
  if (name == "current_cosine_bins") return nmu_;
  if (name == "batch_statistics") return batch_stats_ ? 1 : 0;
  if (name == "batches") return batches_;  // batches folded into the statistics
  if (name == "regions") return nregions_;
  if (name == "region_currents") return rc_on() ? 1 : 0;
  if (name == "region_current_pairs") return region_current_pair_count();
  // collision events since the last reset: tallied, located outside the mesh, rejected (non-finite inputs)
  if (name == "collisions" || name == "collisions_outside" || name == "collisions_rejected") {
    unsigned long long c[3] = {0, 0, 0};
    if (cudaSetDevice(device_) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpy(c, d_coll_counts_, sizeof(c), cudaMemcpyDeviceToHost) != cudaSuccess) {
      cudaGetLastError();
      return -1;
    }
    return int64_t(c[name == "collisions" ? 0 : name == "collisions_outside" ? 1 : 2]);
  }
  if (name == "point_detectors") return ndet_;
  if (name == "detector_void") return det_void_ ? 1 : 0;
  if (name == "detector_hull_candidates") return int64_t(hull_entries_);  // entries of the void's hull-tet lists
  // detector rays and events since the last reset (kDetCount* in walk_kernels.hpp)
  static const char *const kDetNames[kDetCountersVoid] = {
      "detector_rays",       "detector_rays_shadowed",  "detector_rays_lost",       "detector_inside_r0",
      "detector_crossings",  "detector_events_outside", "detector_events_rejected", "detector_hull_entries"};
  for (int c = 0; c < kDetCountersVoid; ++c)
    if (name == kDetNames[c]) {
      unsigned long long v[kDetCountersVoid] = {};
      if (cudaSetDevice(device_) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess ||
          cudaMemcpy(v, d_det_counts_, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) {
        cudaGetLastError();
        return -1;
      }
      return int64_t(v[c]);
    }
  if (name == "walk_blocks_per_sm") return walk_blocks_per_sm();  // occupancy of the last persistent walk kernel launched
  if (name == "die_split") return die_split_ ? 1 : 0;
  if (name == "l2_partition0_sms") return die0_sms_;  // SMs in the L2 partition of SM 0 (0: no map found)
  if (name == "exchange_choice") return exchange_choice_;  // what exchange_tally() does: 0 all-reduce, 1 reduce-scatter
  if (name == "exchange_allreduce_us") return int64_t(exchange_ms_[0] * 1e3);  // comm_init's measurement of the two
  if (name == "exchange_reduce_scatter_us") return int64_t(exchange_ms_[1] * 1e3);
  if (name == "d2h_bytes") return int64_t(d2h_bytes_);  // particle positions sent back by the pinned-caller path, cumulative
  if (name == "host_path") return host_path_;
  if (name == "host_path_last") return span_tag_ == 1 ? 0 : 1;  // path of the last host move: 1 staged, 0 direct
  if (name == "pinned_path") return pinned_path_ ? 1 : 0;
  if (name == "position_mirror") return pos_mirror_valid_ ? 1 : 0;  // the last host move took the pinned-caller path
  if (name == "host_threads") return stager_ ? stager_->threads() : host_threads_;
  if (name == "stage_host_us") return int64_t(stage_host_s_ * 1e6);   // last staged move: host time from entry to return
  if (name == "stage_sent_bytes") return int64_t(stage_sent_bytes_);  // last staged move: bytes put on the wire
  if (name == "staged") return stage_ready_ ? 1 : 0;
  if (name == "stage_copy_us") {  // last staged move: device time from "copy stream free" to the last upload's end
    float ms = 0.f;
    if (!ev_copy0_ || cudaEventSynchronize(ev_copy1_) != cudaSuccess || cudaEventElapsedTime(&ms, ev_copy0_, ev_copy1_) != cudaSuccess) {
      cudaGetLastError();
      return -1;
    }
    return int64_t(ms * 1e3);
  }
  if (name == "host_node") return pool_node_;  // NUMA node the staging workers run on (-1: not pinned to one)
  return -1;
}

int Engine::set_option(const std::string &name, int64_t v) {
  if (name == "variant") {
    if (v == -1) {  // automatic
      variant_ = choose_variant();
      auto_variant_ = true;
      return 0;
    }
    if (v < 0 || v >= kNumVariants || !walk_variant_available(int(v))) return 1;
    if (v >= kVariantEdge && v <= kVariantEdgeOcc6) {
      if (synchronize()) return 1;
      try {
        if (!upload_compact()) return 1;
      } catch (const std::exception &ex) {
        fprintf(stderr, "%s\n", ex.what());
        return 1;
      }
    }
    variant_ = int(v);
    auto_variant_ = false;
  } else if (name == "autotune") {
    autotune_ = v != 0;
  } else if (name == "block") {
    if (v != 64 && v != 128 && v != 256) return 1;
    block_ = int(v);
  } else if (name == "chunk") {
    if (v < 1024) return 1;
    chunk_ = int32_t(std::min<int64_t>(v, INT_MAX)) & ~1023;  // keeps every range 16-byte aligned
    chunk_user_set_ = true;
  } else if (name == "die_split") {
    // Experiment, off by default:
    // the SMs of each L2 partition take the sorted particles from their own end of the sequence.
    die_split_ = v != 0;
    if (die_split_) {
      // which SMs share an L2 partition: probed once per device and process (a few ms)
      struct Cached { bool done = false; uint32_t mask[8]; int die0 = 0, nsms = 0; };
      static Cached cache[64];
      static std::mutex cache_mutex;
      std::lock_guard<std::mutex> lock(cache_mutex);
      Cached &c = cache[device_ & 63];
      if (!c.done) {
        PTB_CUDA_OK(cudaSetDevice(device_));
        PTB_CUDA_OK(cudaDeviceSynchronize());
        if (probe_l2_partitions(c.mask, &c.die0, &c.nsms, compute_) != 0) c.die0 = 0;
        c.done = true;
      }
      for (int i = 0; i < 8; ++i) die_mask_[i] = c.mask[i];
      die0_sms_ = c.die0;
      nsms_ = c.nsms;
    }
  } else if (name == "exchange_choice") {
    exchange_choice_ = v ? 1 : 0;  // the caller must set the same value on every rank
  } else if (name == "seed_grid") {
    if (v < 0 || v > 2) return 1;
    seed_grid_mode_ = int(v);
    use_seed_grid_ = v == 2 || (v == 1 && mesh_.hull_convex);
  } else if (name == "register_host") {
    register_host_ = v != 0;
  } else if (name == "max_iters") {  // crossing limit per walk (the tracer's loop limit); 0 = number of tets + 16
    if (v < 0 || v > INT_MAX) return 1;
    max_iters_ = int32_t(v);
  } else if (name == "l2_fetch") {  // bytes an L2 miss fetches from DRAM: 32, 64 or 128 (device-wide limit)
    if (v != 32 && v != 64 && v != 128) return 1;
    if (cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, size_t(v)) != cudaSuccess) { cudaGetLastError(); return 1; }
  } else if (name == "host_path") {  // 2 = automatic (default), 1 = staged through the pinned slots, 0 = direct copies
    if (v < 0 || v > 2) return 1;
    host_path_ = int(v);
    if (host_path_ == 0) mirror_valid_ = false;
  } else if (name == "pinned_path") {  // 0 = page-locked caller arrays also go through the staging slots
    pinned_path_ = v != 0;
  } else if (name == "host_threads") {  // workers of the staging pool; before the first host-pointer call
    if (v < 1 || v > 256 || stager_) return 1;
    host_threads_ = int(v);
  } else if (name == "bin_midpoint") {  // binning key: cell of the track's midpoint instead of its start
    bin_midpoint_ = v != 0;
  } else if (name == "morton") {
    morton_ = v != 0;
  } else if (name == "claim_run") {
    if (v != 1 && v != 2 && v != 4) return 1;
    claim_run_ = int(v);
  } else {
    return 1;
  }
  return 0;
}

int64_t Engine::debug_order(int32_t *out, int64_t n) {
  if (!last_work_count_ || synchronize()) return -1;
  unsigned int cnt = 0;
  if (cudaMemcpy(&cnt, last_work_count_, sizeof(cnt), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  const int64_t m = std::min<int64_t>(n, cnt);
  if (m > 0 && cudaMemcpy(out, d_order_, size_t(m) * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return cnt;
}

// FinalizeTallies (PumiTallyImpl.cpp:411-416).  With the collision estimator every array of the track-length tally is
// followed by its collision twin, the same name prefixed "collision_".  With batch statistics and at least one batch
// folded, the "_mean" / "_rel_err" arrays (batch_arrays) of both tallies follow all of these, and with weight windows
// their bounds (ww_arrays) follow, then the face currents and, with a mesh source, its strengths (source_arrays).
int Engine::write_tally_results() {
  VtkArrays coll;
  if (collision_ && (synchronize() || gather_shares() || scored_arrays(flux_len(), "collision_", coll, nullptr))) return 1;
  if (batch_stats_ && batches_ > 0 &&
      (synchronize() || batch_arrays(0, "", coll) || (collision_ && batch_arrays(1, "collision_", coll))))
    return 1;
  if (ww_groups_ > 0 && ww_arrays(coll)) return 1;
  if (currents_ && current_arrays(coll)) return 1;
  if (src_groups_ > 0 && source_arrays(coll)) return 1;
  if (multi_results()) return write_scored_results(coll);
  const size_t E = size_t(mesh_.ntets);
  std::vector<double> nf(E * size_t(nbins_)), vol(E);
  if (get_normalized_flux(nf.data(), vol.data(), int64_t(nf.size()))) return 1;  // caller's element order
  // filtered tally: "flux" is the sum over the bins (what the unfiltered tally would hold), and every
  // bin is written as "flux_bin<k>" next to it
  std::vector<std::pair<std::string, const double *>> extra;
  std::vector<double> per_bin;
  if (nbins_ > 1) {
    per_bin.assign(nf.begin(), nf.end());
    for (int32_t b = 0; b < nbins_; ++b) extra.emplace_back("flux_bin" + std::to_string(b), per_bin.data() + size_t(b) * E);
    for (int32_t b = 1; b < nbins_; ++b)
      for (size_t i = 0; i < E; ++i) nf[i] += nf[size_t(b) * E + i];
    nf.resize(E);
  }
  std::vector<int> ncomp(extra.size(), 1);  // (the face currents have four components, everything else one)
  extra.insert(extra.end(), coll.named.begin(), coll.named.end());
  ncomp.insert(ncomp.end(), coll.ncomp.begin(), coll.ncomp.end());
  std::string err;
  if (!write_vtk_dataset(output_name_, mesh_, nf, vol, rank_, nranks_, &err, extra, ncomp)) {
    fprintf(stderr, "[pumitally] ERROR: %s\n", err.c_str());
    return 1;
  }
  return 0;
}

// Scored or timed tally: "flux" and "flux_bin<b>" are score 0, exactly as a one-score engine writes them; every
// score k >= 1 adds "score<k>" (the sum over the bins) and, with several bins, "score<k>_bin<b>".  With time bins
// these are sums over the time bins, and every time bin j adds the same arrays with "_t<j>" after the score name:
// "flux_t<j>", "flux_t<j>_bin<b>", "score<k>_t<j>", "score<k>_t<j>_bin<b>".  With moments every one of these arrays
// is followed by "<name>_grad", its normalised gradient (3 components; a sum's gradient is the sum of the gradients).
int Engine::write_scored_results(VtkArrays &coll) {
  const size_t E = size_t(mesh_.ntets);
  std::vector<double> vol(E), flux;
  if (get_normalized_flux(nullptr, vol.data(), int64_t(E))) return 1;  // (synchronises and gathers the shares)
  VtkArrays a;
  if (scored_arrays(0, "", a, &flux)) return 1;
  a.named.insert(a.named.end(), coll.named.begin(), coll.named.end());
  a.ncomp.insert(a.ncomp.end(), coll.ncomp.begin(), coll.ncomp.end());
  std::string err;
  if (!write_vtk_dataset(output_name_, mesh_, flux, vol, rank_, nranks_, &err, a.named, a.ncomp)) {
    fprintf(stderr, "[pumitally] ERROR: %s\n", err.c_str());
    return 1;
  }
  return 0;
}

// The normalised results of the tally at `base` as write_scored_results names them (its data must be current: after
// synchronize() and gather_shares()).
int Engine::scored_arrays(size_t base, const std::string &prefix, VtkArrays &a, std::vector<double> *main) {
  const size_t E = size_t(mesh_.ntets), S = size_t(nscores_), B = size_t(nbins_), T = nslices();
  std::vector<double> all, grad;
  if (copy_results(all, true, base)) return 1;
  if (moments_ && copy_moments(grad, true, base)) return 1;
  // the same sums for the gradients, 3 values per element: gsets[q] [bin][score][element][3], gsums[q * S + k]
  std::vector<std::vector<double>> gsets, gsums;
  if (moments_) {
    gsets.emplace_back(grad.begin(), grad.begin() + B * S * E * 3);
    for (size_t t = 1; t < T; ++t)
      for (size_t i = 0; i < B * S * E * 3; ++i) gsets[0][i] += grad[t * B * S * E * 3 + i];
    if (ntime_ > 0)
      for (size_t t = 0; t < T; ++t)
        gsets.emplace_back(grad.begin() + t * B * S * E * 3, grad.begin() + (t + 1) * B * S * E * 3);
    for (size_t q = 0; q < gsets.size(); ++q)
      for (size_t k = 0; k < S; ++k) {
        std::vector<double> sum(gsets[q].begin() + k * E * 3, gsets[q].begin() + (k + 1) * E * 3);
        for (size_t b = 1; b < B; ++b)
          for (size_t i = 0; i < E * 3; ++i) sum[i] += gsets[q][(b * S + k) * E * 3 + i];
        gsums.push_back(std::move(sum));
      }
  }
  // sets[0]: the sum over the time bins; sets[1 + j]: time bin j (only with a time filter).  [bin][score][element]
  std::vector<std::vector<double>> sets;
  sets.emplace_back(all.begin(), all.begin() + B * S * E);
  for (size_t t = 1; t < T; ++t)
    for (size_t i = 0; i < B * S * E; ++i) sets[0][i] += all[t * B * S * E + i];
  if (ntime_ > 0)
    for (size_t t = 0; t < T; ++t) sets.emplace_back(all.begin() + t * B * S * E, all.begin() + (t + 1) * B * S * E);
  // per set and score: the sum over the bins
  std::vector<std::vector<double>> sums(sets.size() * S);
  for (size_t q = 0; q < sets.size(); ++q)
    for (size_t k = 0; k < S; ++k) {
      std::vector<double> &sum = sums[q * S + k];
      sum.assign(sets[q].begin() + k * E, sets[q].begin() + (k + 1) * E);
      for (size_t b = 1; b < B; ++b)
        for (size_t i = 0; i < E; ++i) sum[i] += sets[q][(b * S + k) * E + i];
    }
  auto add = [&](const std::string &name, const double *v, const double *g) {
    if (v) {
      a.named.emplace_back(prefix + name, v);
      a.ncomp.push_back(1);
    }
    if (moments_) {
      a.named.emplace_back(prefix + name + "_grad", g);
      a.ncomp.push_back(3);
    }
  };
  for (size_t q = 0; q < sets.size(); ++q) {
    const std::string t = q == 0 ? "" : "_t" + std::to_string(q - 1);
    for (size_t k = 0; k < S; ++k) {
      const std::string name = k == 0 ? "flux" + t : "score" + std::to_string(k) + t;
      // (set 0, score 0 is the main array)
      add(name, (q > 0 || k > 0 || !main) ? sums[q * S + k].data() : nullptr, moments_ ? gsums[q * S + k].data() : nullptr);
      if (B > 1)
        for (size_t b = 0; b < B; ++b)
          add(name + "_bin" + std::to_string(b), sets[q].data() + (b * S + k) * E,
              moments_ ? gsets[q].data() + (b * S + k) * E * 3 : nullptr);
    }
  }
  if (main) *main = sums[0];
  // the pointers above point into these vectors' storage, which moving them keeps
  for (auto *v : {&gsets, &gsums, &sets, &sums})
    for (auto &x : *v) a.data.push_back(std::move(x));
  return 0;
}

// ------------------------------------------------------------------ point queries

namespace {
double mesh_extent(const HostMesh &m) {
  return std::max({m.bbox_hi[0] - m.bbox_lo[0], m.bbox_hi[1] - m.bbox_lo[1], m.bbox_hi[2] - m.bbox_lo[2]});
}

constexpr int64_t kPointsPerLaunch = int64_t(1) << 30;

// Every slice of the arena starts 256-byte aligned, as a cudaMalloc of its own would.
size_t arena_slice(size_t bytes) { return (bytes + 255) & ~size_t(255); }

// One host array of a staged call (Engine::staged), `per` T per item; nullptr is absent, and then absent on the device
// too.  A const T is an input, uploaded before each chunk's enqueue; any other T is an output, copied back after it.
template <class T>
struct Staged {
  T *h;
  size_t per;
  std::remove_const_t<T> *d = nullptr;  // its slice of the arena
  size_t bytes(size_t items) const { return h ? arena_slice(items * per * sizeof(T)) : 0; }
  void carve(char *&next, size_t items) {
    d = h ? reinterpret_cast<std::remove_const_t<T> *>(next) : nullptr;
    next += bytes(items);
  }
  cudaError_t upload(size_t first, size_t count, cudaStream_t s) const {
    if constexpr (std::is_const_v<T>)
      if (h) return cudaMemcpyAsync(d, h + first * per, count * per * sizeof(T), cudaMemcpyHostToDevice, s);
    return cudaSuccess;
  }
  cudaError_t copy_back(size_t first, size_t count, cudaStream_t s) const {
    if constexpr (!std::is_const_v<T>)
      if (h) return cudaMemcpyAsync(h + first * per, d, count * per * sizeof(T), cudaMemcpyDeviceToHost, s);
    return cudaSuccess;
  }
};

template <class T>
Staged<T> stage(T *h, size_t per = 1) {
  return {h, per};
}
}  // namespace

LocateParams Engine::locate_params() const {
  LocateParams p{};
  p.tets = d_tets_;
  p.grid = grid_;  // the seeds are used whatever the relocation walks do (option seed_grid)
  p.max_iters = max_iters_ > 0 ? max_iters_ : int32_t(std::min<int64_t>(mesh_.ntets + 16, INT_MAX));
  p.cx = mesh_.center[0]; p.cy = mesh_.center[1]; p.cz = mesh_.center[2];
  p.sx = mesh_.centroid0[0]; p.sy = mesh_.centroid0[1]; p.sz = mesh_.centroid0[2];
  p.start_elem = mesh_.start_elem;
  p.convex = mesh_.hull_convex ? 1 : 0;
  p.cand_off = d_cand_off_;
  p.cand = d_cand_;
  p.slack = kLocateSlack * mesh_extent(mesh_);
  return p;
}

// A convex hull needs no candidate lists: a walk that meets it proves the point outside.
int Engine::ensure_candidates() {
  if (mesh_.hull_convex || candidates_ready_) return 0;
  std::vector<int64_t> off;
  std::vector<int32_t> tets;
  cell_candidates(mesh_, grid_, kLocateBand * mesh_extent(mesh_), &off, &tets);
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_cand_off_), off.size() * sizeof(int64_t)));
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_cand_), std::max<size_t>(tets.size(), 1) * sizeof(int32_t)));
  PTB_CUDA_OK(cudaMemcpy(d_cand_off_, off.data(), off.size() * sizeof(int64_t), cudaMemcpyHostToDevice));
  PTB_CUDA_OK(cudaMemcpy(d_cand_, tets.data(), tets.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
  cand_entries_ = tets.size();
  candidates_ready_ = true;
  return 0;
}

// The hull-tet lists of the detector void over the seed grid, padded as the point-location lists are.
int Engine::ensure_hull_grid() {
  if (hull_ready_) return 0;
  std::vector<int64_t> off;
  std::vector<int32_t> tets;
  HullGrid h = hull_grid(mesh_, grid_, kLocateBand * mesh_extent(mesh_), &off, &tets);
  int64_t *doff = nullptr;
  int32_t *dtets = nullptr;
  if (cudaMalloc(reinterpret_cast<void **>(&doff), off.size() * sizeof(int64_t)) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void **>(&dtets), std::max<size_t>(tets.size(), 1) * sizeof(int32_t)) != cudaSuccess ||
      cudaMemcpy(doff, off.data(), off.size() * sizeof(int64_t), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(dtets, tets.data(), tets.size() * sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess) {
    const cudaError_t err = cudaGetLastError();
    cudaFree(doff);
    cudaFree(dtets);
    fprintf(stderr, "[pumitally] ERROR: no device memory for the hull grid of the detector void (%s)\n",
            cudaGetErrorString(err));
    return 1;
  }
  h.off = doff;
  h.tets = dtets;
  hull_ = h;
  d_hull_off_ = doff;
  d_hull_tets_ = dtets;
  hull_entries_ = tets.size();
  hull_ready_ = true;
  return 0;
}

int Engine::ensure_arena(size_t bytes) {
  if (bytes <= arena_bytes_) return 0;
  cudaFree(d_arena_);
  d_arena_ = nullptr;
  arena_bytes_ = 0;
  PTB_CUDA_OK(cudaMalloc(&d_arena_, bytes));
  arena_bytes_ = bytes;
  return 0;
}

template <class Setup, class Enqueue, class... A>
int Engine::staged(int64_t n, Setup &&setup, Enqueue &&enqueue, A... a) {
  const int64_t chunk = std::min<int64_t>(chunk_, n);
  const size_t items = n > 0 ? size_t(chunk) : 0;
  if (int rc = setup((a.bytes(items) + ... + size_t(0)))) return std::max(rc, 0);
  char *next = static_cast<char *>(d_arena_);
  (a.carve(next, items), ...);
  for (int64_t b = 0; b < n; b += chunk) {
    const int64_t cnt = std::min(chunk, n - b);
    cudaError_t e = cudaSuccess;
    const auto ok = [&e](cudaError_t r) { return (e = r) == cudaSuccess; };  // the first failure ends the chunk
    (void)((ok(a.upload(size_t(b), size_t(cnt), compute_)) && ...) && ok(enqueue(b, cnt, a.d...)) &&
           (ok(a.copy_back(size_t(b), size_t(cnt), compute_)) && ...));
    PTB_CUDA_OK(e);
  }
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  return 0;
}

int Engine::locate_setup(const double *xyz, int64_t npts, const int32_t *elem, size_t arena) {
  if (npts < 0 || (npts > 0 && (!xyz || !elem))) return 1;
  if (npts == 0) return -1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  return ensure_element_maps() || ensure_candidates() || ensure_arena(arena);
}

cudaError_t Engine::enqueue_locate(const double *xyz, int64_t npts, int32_t *elem, cudaStream_t stream) {
  const LocateParams p = locate_params();
  for (int64_t b = 0; b < npts; b += kPointsPerLaunch)
    if (cudaError_t e = launch_locate(p, xyz + 3 * b, std::min(kPointsPerLaunch, npts - b), nullptr, elem + b,
                                      d_orig_of_internal_, stream))
      return e;
  return cudaSuccess;
}

int Engine::locate_points(const double *xyz, int64_t npts, int32_t *out_elem) {
  return staged(
      npts, [&](size_t arena) { return locate_setup(xyz, npts, out_elem, arena); },
      [&](int64_t, int64_t cnt, const double *x, int32_t *e) { return enqueue_locate(x, cnt, e, compute_); },
      stage(xyz, 3), stage(out_elem));
}

// The mesh tables a query reads never change after construction, so it needs no ordering against moves.
int Engine::locate_points_device(const double *d_xyz, int64_t npts, int32_t *d_elem, cudaStream_t stream) {
  if (int rc = locate_setup(d_xyz, npts, d_elem, 0)) return std::max(rc, 0);
  PTB_CUDA_OK(enqueue_locate(d_xyz, npts, d_elem, stream));
  return 0;
}

// The normalised results exactly as get_normalized_flux computes them (normalize_scores), and with moments the
// gradient get_flux_gradient returns (copy_moments: linear_moments() in fp64 on the host), in internal element order.
int Engine::build_eval_table() {
  const size_t E = size_t(mesh_.ntets), S = size_t(nscores_), B = size_t(result_arrays());
  double per_source = 1.0;
  if (!per_source_divisor(&per_source)) return 1;
  cudaFree(d_eval_vals_); cudaFree(d_eval_grads_); cudaFree(d_eval_cen_);
  d_eval_vals_ = d_eval_grads_ = d_eval_cen_ = nullptr;
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_eval_vals_), std::max<size_t>(B * S * E, 1) * sizeof(double)));
  for (size_t b = 0; b < B; ++b)
    PTB_CUDA_OK(launch_normalize_scores(flux_view() + b * bin_len(), d_volume_, d_eval_vals_ + b * S * E, int64_t(E),
                                        nscores_, stride_, per_source, compute_));
  if (moments_) {
    std::vector<double> g;  // [time][bin][score][caller's element][3]
    if (copy_moments(g, true)) return 1;
    std::vector<double> gi(g.size()), cen(3 * E);
    const double *xyz = mesh_.coords.data();
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < int64_t(E); ++i) {
      const size_t o = size_t(mesh_.orig_of_internal[i]);
      for (size_t r = 0; r < B * S; ++r)
        for (int a = 0; a < 3; ++a) gi[(r * E + size_t(i)) * 3 + a] = g[(r * E + o) * 3 + a];
      for (int a = 0; a < 3; ++a) {  // the vertex average, as linear_moments() forms it
        const int32_t *v = &mesh_.t2v[4 * size_t(i)];
        cen[3 * size_t(i) + a] = 0.25 * (xyz[3 * size_t(v[0]) + a] + xyz[3 * size_t(v[1]) + a] + xyz[3 * size_t(v[2]) + a] +
                                         xyz[3 * size_t(v[3]) + a]);
      }
    }
    PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_eval_grads_), std::max<size_t>(gi.size(), 1) * sizeof(double)));
    PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_eval_cen_), std::max<size_t>(cen.size(), 1) * sizeof(double)));
    PTB_CUDA_OK(cudaMemcpy(d_eval_grads_, gi.data(), gi.size() * sizeof(double), cudaMemcpyHostToDevice));
    PTB_CUDA_OK(cudaMemcpy(d_eval_cen_, cen.data(), cen.size() * sizeof(double), cudaMemcpyHostToDevice));
  }
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  eval_valid_ = true;
  return 0;
}

int Engine::evaluate_points(const double *xyz, int64_t npts, double *out, int64_t n, int32_t *out_elem) {
  const int64_t R = int64_t(result_arrays()) * nscores_;
  if (npts < 0 || (npts > 0 && (!xyz || !out)) || (n != npts && n != R * npts)) {
    fprintf(stderr, "[pumitally] ERROR: evaluate_points: n must be npts or ntime * nbins * nscores * npts (%lld)\n",
            (long long)(R * npts));
    return 1;
  }
  if (synchronize() || gather_shares()) return 1;
  if (!eval_valid_ && build_eval_table()) return 1;
  if (npts == 0) return 0;
  const int64_t rows = n == npts ? 1 : R;
  // the results of a chunk are at most 256 MB of device memory
  const int64_t chunk = std::min<int64_t>(std::min<int64_t>(chunk_, std::max<int64_t>(1024, (int64_t(1) << 25) / rows)), npts);
  // arena slices: points, internal and caller's element ids, results [rows][cnt]
  const size_t c = size_t(chunk), xyz_bytes = arena_slice(3 * c * sizeof(double));
  const size_t id_bytes = arena_slice(c * sizeof(int32_t));
  if (ensure_element_maps() || ensure_candidates() ||
      ensure_arena(xyz_bytes + 2 * id_bytes + size_t(rows) * c * sizeof(double)))
    return 1;
  char *arena = static_cast<char *>(d_arena_);
  double *qxyz = reinterpret_cast<double *>(arena);
  int32_t *qint = reinterpret_cast<int32_t *>(arena + xyz_bytes);
  int32_t *qelem = reinterpret_cast<int32_t *>(arena + xyz_bytes + id_bytes);
  double *qout = reinterpret_cast<double *>(arena + xyz_bytes + 2 * id_bytes);
  const LocateParams p = locate_params();
  for (int64_t b = 0; b < npts; b += chunk) {
    const int64_t cnt = std::min(chunk, npts - b);
    PTB_CUDA_OK(cudaMemcpyAsync(qxyz, xyz + 3 * b, size_t(cnt) * 3 * sizeof(double), cudaMemcpyHostToDevice, compute_));
    PTB_CUDA_OK(launch_locate(p, qxyz, cnt, qint, out_elem ? qelem : nullptr, d_orig_of_internal_, compute_));
    PTB_CUDA_OK(launch_evaluate(qxyz, qint, cnt, d_eval_vals_, moments_ ? d_eval_grads_ : nullptr, d_eval_cen_,
                                mesh_.ntets, int32_t(rows), qout, cnt, compute_));
    PTB_CUDA_OK(cudaMemcpy2DAsync(out + b, size_t(npts) * sizeof(double), qout, size_t(cnt) * sizeof(double),
                                  size_t(cnt) * sizeof(double), size_t(rows), cudaMemcpyDeviceToHost, compute_));
    if (out_elem)
      PTB_CUDA_OK(cudaMemcpyAsync(out_elem + b, qelem, size_t(cnt) * sizeof(int32_t), cudaMemcpyDeviceToHost, compute_));
  }
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  return 0;
}

// ------------------------------------------------------------------ collision estimator

CollisionParams Engine::collision_params() const {
  CollisionParams c{};
  c.flux = d_flux_ + flux_len();
  c.edges = d_edges_;
  c.nt = ntime_;
  c.nbins = nbins_;
  c.nscores = nscores_;
  c.stride = stride_;
  c.moments = moments_;
  c.bin_stride = int64_t(bin_len());
  c.slice = int64_t(nbins_) * int64_t(bin_len());
  c.cx = mesh_.center[0]; c.cy = mesh_.center[1]; c.cz = mesh_.center[2];
  return c;
}

// The refusals every collision call shares, checked before anything is uploaded.
bool Engine::collision_refused(const double *responses, const double *times) const {
  const char *why = !collision_                       ? "the collision estimator is off (set_collision_estimator)"
                    : (!responses && nscores_ > 1)    ? "responses are required with several scores"
                    : (!times && ntime_ > 0)          ? "times are required while time bins are set"
                                                      : nullptr;
  if (why) fprintf(stderr, "[pumitally] ERROR: collision events refused: %s\n", why);
  return why != nullptr;
}

int Engine::collide_located_setup(const double *xyz, int64_t n, const double *w, const double *r, const double *t,
                                  size_t arena) {
  if (collision_refused(r, t) || n < 0 || (n > 0 && (!xyz || !w))) return 1;
  if (n == 0) return -1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (ensure_candidates() || ensure_arena(arena)) return 1;
  flux_global_valid_ = flux_owned_only_ = eval_valid_ = false;  // the local tally moves on, as with a move
  tallied_ = true;
  return 0;
}

cudaError_t Engine::enqueue_collide_located(const double *xyz, int64_t n, const double *w, const double *r,
                                            const int32_t *bins, const double *t, cudaStream_t stream) {
  const LocateParams l = locate_params();
  const CollisionParams p = collision_params();
  const size_t S = size_t(nscores_);
  for (int64_t b = 0; b < n; b += kPointsPerLaunch)
    if (cudaError_t e = launch_collide_located(l, p, xyz + 3 * b, std::min(kPointsPerLaunch, n - b), w + b,
                                               r ? r + S * size_t(b) : nullptr, bins ? bins + b : nullptr,
                                               ntime_ > 0 ? t + b : nullptr, d_coll_counts_, stream))
      return e;
  return cudaSuccess;
}

int Engine::tally_collisions(const double *xyz, int64_t nevents, const double *weights, const double *responses,
                             const int32_t *bins, const double *times) {
  return staged(
      nevents, [&](size_t arena) { return collide_located_setup(xyz, nevents, weights, responses, times, arena); },
      [&](int64_t, int64_t cnt, const double *x, const double *w, const double *r, const double *t, const int32_t *bn) {
        return enqueue_collide_located(x, cnt, w, r, bn, t, compute_);
      },
      // times are read only while time bins are set, so only then do they travel
      stage(xyz, 3), stage(weights), stage(responses, size_t(nscores_)), stage(ntime_ > 0 ? times : nullptr),
      stage(bins));
}

// The mesh tables location reads never change after construction, so located events need no ordering against moves.
int Engine::tally_collisions_device(const double *d_xyz, int64_t nevents, const double *d_weights,
                                    const double *d_responses, const int32_t *d_bins, const double *d_times,
                                    cudaStream_t stream) {
  if (int rc = collide_located_setup(d_xyz, nevents, d_weights, d_responses, d_times, 0)) return std::max(rc, 0);
  PTB_CUDA_OK(enqueue_collide_located(d_xyz, nevents, d_weights, d_responses, d_bins, d_times, stream));
  return 0;
}

int Engine::collide_particles_setup(const int8_t *collided, const double *w, const double *r, const double *t,
                                    int32_t n, size_t arena, cudaStream_t stream) {
  if (collision_refused(r, t)) return 1;
  if (n != n_ || (n > 0 && (!collided || !w))) {
    fprintf(stderr, "[pumitally] ERROR: collision events at the particles: n must be num_particles (%d)\n", n_);
    return 1;
  }
  if (n == 0) return -1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (ensure_arena(arena) || follow_last_stream(stream)) return 1;  // reads the particle state the last move wrote
  flux_global_valid_ = flux_owned_only_ = eval_valid_ = false;
  tallied_ = true;
  return 0;
}

cudaError_t Engine::enqueue_collide_particles(int32_t first, int32_t n, const int8_t *collided, const double *w,
                                              const double *r, const int32_t *bins, const double *t,
                                              cudaStream_t stream) {
  return launch_collide_particles(d_state_ + first, collided, n, collision_params(), w, r, bins,
                                  ntime_ > 0 ? t : nullptr, d_coll_counts_, stream);
}

int Engine::tally_collisions_at_particles(const int8_t *collided, const double *weights, const double *responses,
                                          const int32_t *bins, const double *times, int32_t n) {
  return staged(
      n, [&](size_t arena) { return collide_particles_setup(collided, weights, responses, times, n, arena, compute_); },
      [&](int64_t b, int64_t cnt, const int8_t *c, const double *w, const double *r, const double *t,
          const int32_t *bn) {
        return enqueue_collide_particles(int32_t(b), int32_t(cnt), c, w, r, bn, t, compute_);
      },
      stage(collided), stage(weights), stage(responses, size_t(nscores_)), stage(ntime_ > 0 ? times : nullptr),
      stage(bins));
}

int Engine::tally_collisions_at_particles_device(const int8_t *d_collided, const double *d_weights,
                                                 const double *d_responses, const int32_t *d_bins,
                                                 const double *d_times, int32_t n, cudaStream_t stream) {
  if (int rc = collide_particles_setup(d_collided, d_weights, d_responses, d_times, n, 0, stream))
    return std::max(rc, 0);
  PTB_CUDA_OK(enqueue_collide_particles(0, n, d_collided, d_weights, d_responses, d_bins, d_times, stream));
  return 0;
}

// ------------------------------------------------------------------ point detectors

// d_det_: [open][exchanged sum], then with batch statistics [mean][M2], each L doubles.
int Engine::alloc_detectors(size_t L, bool stats, double **out) {
  *out = nullptr;
  const size_t bytes = std::max<size_t>((stats ? 4 : 2) * L, 1) * sizeof(double);
  if (cudaMalloc(reinterpret_cast<void **>(out), bytes) != cudaSuccess || cudaMemset(*out, 0, bytes) != cudaSuccess) {
    const cudaError_t err = cudaGetLastError();
    cudaFree(*out);
    *out = nullptr;
    fprintf(stderr, "[pumitally] ERROR: no device memory for the detector tally of %zu results (%s)\n", L,
            cudaGetErrorString(err));
    return 1;
  }
  return 0;
}

int Engine::set_point_detectors(const double *xyz, int32_t ndet, const double *r0) {
  const bool remove = !xyz && !r0 && ndet == 0;
  const char *why = nccl_comm_ ? "after comm_init (the exchange buffers are sized by then)"
                    : remove   ? nullptr
                    : (!xyz || !r0 || ndet < 1 || ndet > kMaxDetectors)
                        ? "ndet must be 1..256 with positions and radii, or (NULL, 0, NULL)"
                        : nullptr;
  for (int32_t d = 0; !why && !remove && d < ndet; ++d)
    if (!std::isfinite(r0[d]) || r0[d] < 0.0) why = "every exclusion radius must be finite and >= 0";
  std::vector<int32_t> elem(size_t(std::max(ndet, 0)), -1);
  if (!why && !remove) {
    if (synchronize() || ensure_candidates() || ensure_arena(arena_slice(3 * size_t(ndet) * sizeof(double)) +
                                                             arena_slice(size_t(ndet) * sizeof(int32_t))))
      return 1;
    double *dx = static_cast<double *>(d_arena_);
    int32_t *de = reinterpret_cast<int32_t *>(static_cast<char *>(d_arena_) + arena_slice(3 * size_t(ndet) * sizeof(double)));
    PTB_CUDA_OK(cudaMemcpy(dx, xyz, 3 * size_t(ndet) * sizeof(double), cudaMemcpyHostToDevice));
    PTB_CUDA_OK(launch_locate(locate_params(), dx, ndet, de, nullptr, nullptr, compute_));
    PTB_CUDA_OK(cudaMemcpyAsync(elem.data(), de, size_t(ndet) * sizeof(int32_t), cudaMemcpyDeviceToHost, compute_));
    PTB_CUDA_OK(cudaStreamSynchronize(compute_));
    for (int32_t d = 0; d < ndet; ++d)
      if (!std::isfinite(xyz[3 * d]) || !std::isfinite(xyz[3 * d + 1]) || !std::isfinite(xyz[3 * d + 2]))
        why = "every detector must have finite coordinates";
      else if (elem[size_t(d)] < 0 && !det_void_)
        why = "every detector must lie inside the mesh (or the detector void be on: set_detector_void)";
  }
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: set_point_detectors: %s\n", why);
    return 1;
  }
  if (synchronize()) return 1;
  double *nd = nullptr, *npos = nullptr, *nr0 = nullptr;
  if (!remove) {
    if (alloc_detectors(nslices() * size_t(nbins_) * size_t(nscores_) * size_t(ndet), batch_stats_, &nd)) return 1;
    if (cudaMalloc(reinterpret_cast<void **>(&npos), 3 * size_t(ndet) * sizeof(double)) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void **>(&nr0), size_t(ndet) * sizeof(double)) != cudaSuccess ||
        cudaMemcpy(npos, xyz, 3 * size_t(ndet) * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(nr0, r0, size_t(ndet) * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess) {
      cudaGetLastError();
      cudaFree(nd);
      cudaFree(npos);
      cudaFree(nr0);
      fprintf(stderr, "[pumitally] ERROR: set_point_detectors: no device memory for the detectors\n");
      return 1;
    }
  }
  if (batch_stats_ && alloc_stats(reported_len())) {  // discards the folded batches, as every set_* call does
    cudaFree(nd);
    cudaFree(npos);
    cudaFree(nr0);
    return 1;
  }
  cudaFree(d_det_);
  cudaFree(d_det_pos_);
  cudaFree(d_det_r0_);
  d_det_ = nd;
  d_det_pos_ = npos;
  d_det_r0_ = nr0;
  ndet_ = remove ? 0 : ndet;
  det_xyz_.assign(xyz, xyz + 3 * size_t(ndet_));
  det_r0_.assign(r0, r0 + size_t(ndet_));
  det_elem_ = remove ? std::vector<int32_t>() : elem;
  return reset_tally();
}

int Engine::set_detector_void(int32_t on) {
  const bool outside = std::count(det_elem_.begin(), det_elem_.end(), -1) > 0;
  const char *why = nccl_comm_                  ? "after comm_init (the exchange buffers are sized by then)"
                    : (on != 0 && on != 1)      ? "on must be 0 or 1"
                    : (on == 0 && det_void_ && outside)
                        ? "a point detector lies outside the mesh (move or remove it first: set_point_detectors)"
                        : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: set_detector_void: %s\n", why);
    return 1;
  }
  if ((on != 0) == det_void_) return 0;
  if (synchronize()) return 1;
  if (batch_stats_ && alloc_stats(reported_len())) return 1;  // discards the folded batches, as every set_* call does
  det_void_ = on != 0;
  return reset_tally();
}

int Engine::set_detector_cross_sections(const double *sigma_t, int64_t n) {
  const int64_t E = mesh_.ntets;
  const char *why = !sigma_t || n != int64_t(nbins_) * E ? "n must be nbins * num_elements" : nullptr;
  for (int64_t i = 0; !why && i < n; ++i)
    if (!std::isfinite(sigma_t[i]) || sigma_t[i] < 0.0) why = "every cross section must be finite and >= 0";
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: set_detector_cross_sections: %s\n", why);
    return 1;
  }
  std::vector<double> internal(static_cast<size_t>(n));  // [bin][internal element]
  for (int64_t b = 0; b < nbins_; ++b)
    for (int64_t i = 0; i < E; ++i) internal[size_t(b * E + i)] = sigma_t[b * E + mesh_.orig_of_internal[size_t(i)]];
  if (synchronize()) return 1;
  double *ns = nullptr;
  if (cudaMalloc(reinterpret_cast<void **>(&ns), size_t(n) * sizeof(double)) != cudaSuccess ||
      cudaMemcpy(ns, internal.data(), size_t(n) * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaGetLastError();
    cudaFree(ns);
    fprintf(stderr, "[pumitally] ERROR: set_detector_cross_sections: no device memory for the table\n");
    return 1;
  }
  cudaFree(d_sigma_);
  d_sigma_ = ns;
  sigma_bins_ = nbins_;
  sigma_crc_ = ckpt::crc32(internal.data(), internal.size() * sizeof(double));
  return 0;
}

DetectorParams Engine::detector_params() const {
  DetectorParams p{};
  p.tally = d_det_;
  p.sigma = d_sigma_;
  p.pos = d_det_pos_;
  p.r0 = d_det_r0_;
  p.edges = d_edges_;
  p.nt = ntime_;
  p.nbins = nbins_;
  p.nscores = nscores_;
  p.ndet = ndet_;
  p.zero_r0 = std::count(det_r0_.begin(), det_r0_.end(), 0.0) > 0 ? 1 : 0;
  p.E = mesh_.ntets;
  return p;
}

bool Engine::detector_refused(const double *responses, const double *times, const double *speeds) const {
  const char *why = ndet_ == 0                       ? "no point detectors are set (set_point_detectors)"
                    : !d_sigma_                      ? "no cross-section table is set (set_detector_cross_sections)"
                    : (!responses && nscores_ > 1)   ? "responses are required with several scores"
                    : ((!times || !speeds) && ntime_ > 0) ? "times and speeds are required while time bins are set"
                                                     : nullptr;
  if (why) fprintf(stderr, "[pumitally] ERROR: detector events refused: %s\n", why);
  return why != nullptr;
}

int Engine::detect_located_setup(const double *xyz, int64_t n, const double *w, const double *r, const double *t,
                                 const double *v, size_t arena) {
  if (detector_refused(r, t, v) || n < 0 || (n > 0 && (!xyz || !w))) return 1;
  if (n == 0) return -1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (ensure_candidates() || (det_void_ && ensure_hull_grid()) || ensure_arena(arena)) return 1;
  det_global_valid_ = false;
  tallied_ = true;  // a checkpoint now holds the open batch, the detector tally with it
  return 0;
}

cudaError_t Engine::enqueue_detect_located(const double *xyz, int64_t n, const double *w, const double *pdf,
                                           const double *r, const int32_t *bins, const double *t, const double *v,
                                           cudaStream_t stream) {
  const LocateParams l = locate_params();
  const DetectorParams p = detector_params();
  const size_t S = size_t(nscores_), D = size_t(ndet_);
  const int64_t per = std::max<int64_t>(1, kPointsPerLaunch / ndet_);  // rays per launch stay below 2^30
  for (int64_t b = 0; b < n; b += per)
    if (cudaError_t e = launch_detect_located(l, p, xyz + 3 * b, std::min(per, n - b), w + b,
                                              pdf ? pdf + D * size_t(b) : nullptr, r ? r + S * size_t(b) : nullptr,
                                              bins ? bins + b : nullptr, ntime_ > 0 ? t + b : nullptr,
                                              ntime_ > 0 ? v + b : nullptr, d_det_counts_, stream, hull_grid_params()))
      return e;
  return cudaSuccess;
}

int Engine::tally_detectors(const double *xyz, int64_t nevents, const double *weights, const double *pdf,
                            const double *responses, const int32_t *bins, const double *times, const double *speeds) {
  return staged(
      nevents,
      [&](size_t arena) { return detect_located_setup(xyz, nevents, weights, responses, times, speeds, arena); },
      [&](int64_t, int64_t cnt, const double *x, const double *w, const double *p, const double *r, const double *t,
          const double *v, const int32_t *bn) { return enqueue_detect_located(x, cnt, w, p, r, bn, t, v, compute_); },
      // times and speeds are read only while time bins are set, so only then do they travel
      stage(xyz, 3), stage(weights), stage(pdf, size_t(ndet_)), stage(responses, size_t(nscores_)),
      stage(ntime_ > 0 ? times : nullptr), stage(ntime_ > 0 ? speeds : nullptr), stage(bins));
}

int Engine::tally_detectors_device(const double *d_xyz, int64_t nevents, const double *d_weights, const double *d_pdf,
                                   const double *d_responses, const int32_t *d_bins, const double *d_times,
                                   const double *d_speeds, cudaStream_t stream) {
  if (int rc = detect_located_setup(d_xyz, nevents, d_weights, d_responses, d_times, d_speeds, 0))
    return std::max(rc, 0);
  PTB_CUDA_OK(enqueue_detect_located(d_xyz, nevents, d_weights, d_pdf, d_responses, d_bins, d_times, d_speeds, stream));
  return 0;
}

int Engine::detect_particles_setup(const int8_t *flagged, const double *w, const double *r, const double *t,
                                   const double *v, int32_t n, size_t arena, cudaStream_t stream) {
  if (detector_refused(r, t, v)) return 1;
  if (n != n_ || (n > 0 && (!flagged || !w))) {
    fprintf(stderr, "[pumitally] ERROR: detector events at the particles: n must be num_particles (%d)\n", n_);
    return 1;
  }
  if (n == 0) return -1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  // reads the particle state the last move wrote
  if ((det_void_ && ensure_hull_grid()) || ensure_arena(arena) || follow_last_stream(stream)) return 1;
  det_global_valid_ = false;
  tallied_ = true;
  return 0;
}

int Engine::tally_detectors_at_particles(const int8_t *flagged, const double *weights, const double *pdf,
                                         const double *responses, const int32_t *bins, const double *times,
                                         const double *speeds, int32_t n) {
  WalkParams wp{};
  wp.tets = d_tets_;
  wp.max_iters = locate_params().max_iters;
  wp.cx = mesh_.center[0]; wp.cy = mesh_.center[1]; wp.cz = mesh_.center[2];
  return staged(
      n, [&](size_t arena) { return detect_particles_setup(flagged, weights, responses, times, speeds, n, arena, compute_); },
      [&](int64_t b, int64_t cnt, const int8_t *c, const double *w, const double *p, const double *r, const double *t,
          const double *v, const int32_t *bn) {
        return launch_detect_particles(wp, detector_params(), d_state_ + b, c, int32_t(cnt), w, p, r, bn,
                                       ntime_ > 0 ? t : nullptr, ntime_ > 0 ? v : nullptr, d_det_counts_, compute_,
                                       hull_grid_params());
      },
      stage(flagged), stage(weights), stage(pdf, size_t(ndet_)), stage(responses, size_t(nscores_)),
      stage(ntime_ > 0 ? times : nullptr), stage(ntime_ > 0 ? speeds : nullptr), stage(bins));
}

int Engine::tally_detectors_at_particles_device(const int8_t *d_flagged, const double *d_weights, const double *d_pdf,
                                                const double *d_responses, const int32_t *d_bins, const double *d_times,
                                                const double *d_speeds, int32_t n, cudaStream_t stream) {
  if (int rc = detect_particles_setup(d_flagged, d_weights, d_responses, d_times, d_speeds, n, 0, stream))
    return std::max(rc, 0);
  WalkParams wp{};
  wp.tets = d_tets_;
  wp.max_iters = locate_params().max_iters;
  wp.cx = mesh_.center[0]; wp.cy = mesh_.center[1]; wp.cz = mesh_.center[2];
  PTB_CUDA_OK(launch_detect_particles(wp, detector_params(), d_state_, d_flagged, n, d_weights, d_pdf, d_responses,
                                      d_bins, ntime_ > 0 ? d_times : nullptr, ntime_ > 0 ? d_speeds : nullptr,
                                      d_det_counts_, stream, hull_grid_params()));
  return 0;
}

int Engine::exchange_detectors() {
  if (ndet_ == 0 || !sharded()) return 0;
  const size_t L = det_len();
  if (nccl_allreduce_sum_f64(nccl_comm_, d_det_, d_det_ + L, L, compute_)) return 1;
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  det_global_valid_ = true;
  return 0;
}

int Engine::get_detector_results(int32_t kind, double *out, int64_t n) {
  const size_t L = det_len();
  const char *why = ndet_ == 0                ? "no point detectors are set (set_point_detectors)"
                    : (kind < 0 || kind > 3)  ? "kind must be 0 (value), 1 (batch mean), 2 (standard error) or 3 "
                                                "(relative error)"
                    : (n != int64_t(L) || !out) ? "n must be ntime * nbins * nscores * ndet"
                                              : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: get_detector_results: %s\n", why);
    return 1;
  }
  if (kind > 0 && batch_refused(0, kind - 1)) return 1;
  if (synchronize()) return 1;
  if (kind == 0) {
    double div = 1.0;
    if (!per_source_divisor(&div)) return 1;
    PTB_CUDA_OK(cudaMemcpy(out, d_det_ + (det_global_valid_ ? L : 0), L * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < L; ++i) out[i] /= div;
    return 0;
  }
  std::vector<double> m(2 * L);
  PTB_CUDA_OK(cudaMemcpy(m.data(), d_det_ + 2 * L, 2 * L * sizeof(double), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < L; ++i) out[i] = batch_readout(m[i], m[L + i], double(batches_), 1.0, kind - 1);
  return 0;
}

// ------------------------------------------------------------------ batch statistics

int Engine::alloc_stats(size_t len) {
  double *nm = nullptr, *nq = nullptr;
  const size_t bytes = std::max<size_t>(len, 1) * sizeof(double);
  if (cudaMalloc(reinterpret_cast<void **>(&nm), bytes) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void **>(&nq), bytes) != cudaSuccess || cudaMemset(nm, 0, bytes) != cudaSuccess ||
      cudaMemset(nq, 0, bytes) != cudaSuccess) {
    const cudaError_t err = cudaGetLastError();
    cudaFree(nm);
    cudaFree(nq);
    fprintf(stderr, "[pumitally] ERROR: no device memory for the batch statistics of %zu results (%s)\n", len,
            cudaGetErrorString(err));
    return 1;
  }
  free_stats();
  d_mean_ = nm;
  d_m2_ = nq;
  return 0;
}

void Engine::free_stats() {
  cudaFree(d_mean_);
  cudaFree(d_m2_);
  cudaFree(d_region_stats_);
  d_mean_ = d_m2_ = d_region_stats_ = nullptr;
  batches_ = 0;
}

int Engine::set_batch_statistics(int32_t on) {
  if (on != 0 && on != 1) return 1;
  if (nccl_comm_) {
    fprintf(stderr, "[pumitally] ERROR: set_batch_statistics after comm_init (the exchange buffers are sized by then)\n");
    return 1;
  }
  if (synchronize()) return 1;
  double *nd = nullptr;
  if (ndet_ > 0 && alloc_detectors(det_len(), on != 0, &nd)) return 1;
  if (on) {
    if (alloc_stats(reported_len())) {  // (a second call with 1 discards the folded batches)
      cudaFree(nd);
      return 1;
    }
  } else {
    free_stats();
  }
  if (ndet_ > 0) {
    cudaFree(d_det_);
    d_det_ = nd;
  }
  batch_stats_ = on != 0;
  return reset_tally();
}

bool Engine::batch_refused(int32_t tally, int32_t kind) const {
  const char *why = !batch_stats_                            ? "batch statistics are off (set_batch_statistics)"
                    : (tally != 0 && tally != 1)             ? "tally must be 0 (track length) or 1 (collision)"
                    : (tally == 1 && !collision_)            ? "the collision estimator is off (set_collision_estimator)"
                    : (kind < 0 || kind > 3)                 ? "kind must be 0 (mean), 1 (standard error), 2 (relative "
                                                               "error) or 3 (gradient of the mean)"
                    : batches_ < 1                           ? "no batch has been folded yet (end_batch)"
                    : (batches_ < 2 && (kind == 1 || kind == 2)) ? "errors need at least two batches"
                    : (kind == 3 && !moments_)               ? "the engine tallies no moments (set_moments)"
                                                             : nullptr;
  if (why) fprintf(stderr, "[pumitally] ERROR: batch results refused: %s\n", why);
  return why != nullptr;
}

// Closes the open batch: its divisor d_b (as get_normalized_flux's, summed over the ranks for modes 1 and 3) goes to
// d_batch_div_[0] on the device, every reported double x of the batch (this rank's share of the summed tally with
// several ranks) is folded as x / d_b, and the tally is reset.
int Engine::end_batch() {
  if (!batch_stats_) {
    fprintf(stderr, "[pumitally] ERROR: end_batch: batch statistics are off (set_batch_statistics)\n");
    return 1;
  }
  if (synchronize() || (nregions_ > 0 && (ensure_region_work() || ensure_region_stats()))) return 1;
  const double local = norm_mode_ == 1 ? double(std::max(n_, 1)) : norm_mode_ == 2 ? norm_value_ : 1.0;
  if (norm_mode_ == 3)
    PTB_CUDA_OK(cudaMemcpyAsync(d_batch_div_ + 1, d_initial_weight_, sizeof(double), cudaMemcpyDeviceToDevice, compute_));
  else
    PTB_CUDA_OK(cudaMemcpyAsync(d_batch_div_ + 1, &local, sizeof(double), cudaMemcpyHostToDevice, compute_));
  if (sharded() && (norm_mode_ == 1 || norm_mode_ == 3)) {  // the whole batch's source
    if (nccl_allreduce_sum_f64(nccl_comm_, d_batch_div_ + 1, d_batch_div_, 1, compute_)) return 1;
  } else {
    PTB_CUDA_OK(cudaMemcpyAsync(d_batch_div_, d_batch_div_ + 1, sizeof(double), cudaMemcpyDeviceToDevice, compute_));
  }
  double div = 0.0;
  PTB_CUDA_OK(cudaMemcpyAsync(&div, d_batch_div_, sizeof(double), cudaMemcpyDeviceToHost, compute_));
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  if (!(div > 0.0)) {  // the same value on every rank: all of them refuse
    fprintf(stderr, "[pumitally] ERROR: end_batch: the batch's source-normalisation divisor is %g\n", div);
    return 1;
  }
  const size_t L = reported_len();
  const double nb = double(batches_ + 1);
  // the batch's leakage: its hull slots summed into the leakage slots, which the exchange and the fold then carry
  if (currents_ && leakage_sums(d_flux_ + current_base(), d_flux_ + leak_base())) return 1;
  if (nregions_ > 0) {  // region sums of this rank's batch, summed over the ranks: the same statistics on every rank
    const size_t RL = region_len();
    double *sums = d_region_stats_;
    if (region_sums(d_flux_, int64_t(collision_ ? 2 : 1) * result_arrays(), sums)) return 1;
    if (rc_on() && region_current_sums(d_flux_ + current_base(), sums + rc_base())) return 1;
    if (sharded() && nccl_allreduce_sum_f64(nccl_comm_, sums, sums, RL, compute_)) return 1;
    PTB_CUDA_OK(launch_batch_fold(sums, sums + RL, sums + 2 * RL, int64_t(RL), d_batch_div_, nb, compute_));
  }
  if (ndet_ > 0) {  // the detector tally summed over the ranks, folded the same on every rank
    const size_t DL = det_len();
    if (batches_ == 0) PTB_CUDA_OK(cudaMemsetAsync(d_det_ + 2 * DL, 0, 2 * DL * sizeof(double), compute_));
    if (sharded() && nccl_allreduce_sum_f64(nccl_comm_, d_det_, d_det_ + DL, DL, compute_)) return 1;
    PTB_CUDA_OK(launch_batch_fold(d_det_ + (sharded() ? DL : 0), d_det_ + 2 * DL, d_det_ + 3 * DL, int64_t(DL),
                                  d_batch_div_, nb, compute_));
  }
  if (sharded()) {
    const size_t lo = size_t(rank_) * share_;  // the last share ends in padding (or a binned move's unreported array)
    if (nccl_reduce_scatter_sum_f64(nccl_comm_, d_flux_, d_flux_global_ + lo, share_, compute_)) return 1;
    PTB_CUDA_OK(launch_batch_fold(d_flux_global_ + lo, d_mean_, d_m2_, lo < L ? int64_t(std::min(share_, L - lo)) : 0,
                                  d_batch_div_, nb, compute_));
  } else {
    PTB_CUDA_OK(launch_batch_fold(d_flux_, d_mean_, d_m2_, int64_t(L), d_batch_div_, nb, compute_));
  }
  ++batches_;
  return reset_tally();
}

int Engine::stats_view(const double **mean, const double **m2, double **tmp) {
  *tmp = nullptr;
  if (!sharded()) {
    *mean = d_mean_;
    *m2 = d_m2_;
    return 0;
  }
  const size_t full = share_ * size_t(nranks_);
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(tmp), 2 * full * sizeof(double)));
  *mean = *tmp;
  *m2 = *tmp + full;
  if (nccl_all_gather_f64(nccl_comm_, d_mean_, *tmp, share_, compute_) ||
      nccl_all_gather_f64(nccl_comm_, d_m2_, *tmp + full, share_, compute_))
    return 1;
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  return 0;
}

int Engine::copy_batch_results(std::vector<double> &out, int32_t tally, int32_t kind) {
  const size_t E = size_t(mesh_.ntets), S = size_t(nscores_), R = size_t(result_arrays());
  if (ensure_element_maps()) return 1;
  const double *mean = nullptr, *m2 = nullptr;
  double *tmp = nullptr, *d_out = nullptr;
  int rc = stats_view(&mean, &m2, &tmp);
  if (!rc) {
    const size_t base = size_t(tally) * flux_len();
    out.resize(R * S * E);
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&d_out), std::max<size_t>(out.size(), 1) * sizeof(double));
    if (e == cudaSuccess)
      e = launch_batch_readout(mean + base, m2 + base, d_volume_, d_orig_of_internal_, d_out, int64_t(E), int32_t(R),
                               nscores_, stride_, double(batches_), kind, compute_);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(out.data(), d_out, out.size() * sizeof(double), cudaMemcpyDeviceToHost, compute_);
    if (e == cudaSuccess) e = cudaStreamSynchronize(compute_);
    if (e != cudaSuccess) {
      fprintf(stderr, "[pumitally] CUDA error %s reading the batch statistics\n", cudaGetErrorString(e));
      rc = 1;
    }
  }
  cudaFree(d_out);
  cudaFree(tmp);
  return rc;
}

int Engine::get_batch_results(int32_t tally, int32_t kind, double *out, int64_t n) {
  if (batch_refused(tally, kind)) return 1;
  const int64_t E = mesh_.ntets, m = kind == 3 ? 3 : 1;
  if (n != m * E && n != m * int64_t(result_arrays()) * nscores_ * E) {
    fprintf(stderr, "[pumitally] ERROR: get_batch_results: n must be %lld or %lld\n", (long long)(m * E),
            (long long)(m * int64_t(result_arrays()) * nscores_ * E));
    return 1;
  }
  if (synchronize()) return 1;
  std::vector<double> all;
  if (kind == 3) {  // the gradient of the mean records, which are already per source
    const double *mean = nullptr, *m2 = nullptr;
    double *tmp = nullptr;
    const int rc = stats_view(&mean, &m2, &tmp) || copy_moments(all, true, size_t(tally) * flux_len(), mean);
    cudaFree(tmp);
    if (rc) return 1;
  } else if (copy_batch_results(all, tally, kind)) {
    return 1;
  }
  std::memcpy(out, all.data(), size_t(n) * sizeof(double));
  return 0;
}

int Engine::get_batch_max_rel_err(int32_t tally, int32_t score, double *out_max, int64_t *out_nonzero) {
  if (batch_refused(tally, 2)) return 1;
  if (score < 0 || score >= nscores_ || !out_max || !out_nonzero) {
    fprintf(stderr, "[pumitally] ERROR: get_batch_max_rel_err: score must be in [0, %d)\n", nscores_);
    return 1;
  }
  if (synchronize()) return 1;
  const size_t L = reported_len(), goff = sharded() ? size_t(rank_) * share_ : 0;
  const int64_t n = goff < L ? int64_t(std::min(stats_len(), L - goff)) : 0;
  PTB_CUDA_OK(launch_batch_max_rel_err(d_mean_, d_m2_, n, int64_t(goff), int64_t(size_t(tally) * flux_len()),
                                       int64_t(flux_len()), stride_, score, double(batches_), d_stats_red_, compute_));
  unsigned long long red[2] = {0, 0};
  PTB_CUDA_OK(cudaMemcpyAsync(red, d_stats_red_, sizeof(red), cudaMemcpyDeviceToHost, compute_));
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  double mx = 0.0, cnt = double(red[1]);
  std::memcpy(&mx, &red[0], sizeof(double));
  if (sharded()) {  // max and sum over the ranks, from every rank's pair
    std::vector<double> all(2 * size_t(nranks_) + 2);
    all[0] = mx;
    all[1] = cnt;
    double *d = nullptr;
    PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d), all.size() * sizeof(double)));
    cudaError_t e = cudaMemcpyAsync(d, all.data(), 2 * sizeof(double), cudaMemcpyHostToDevice, compute_);
    const int rc = e != cudaSuccess || nccl_all_gather_f64(nccl_comm_, d, d + 2, 2, compute_);
    if (!rc) e = cudaMemcpyAsync(all.data(), d, all.size() * sizeof(double), cudaMemcpyDeviceToHost, compute_);
    if (!rc && e == cudaSuccess) e = cudaStreamSynchronize(compute_);
    cudaFree(d);
    if (rc || e != cudaSuccess) return 1;
    mx = cnt = 0.0;
    for (int r = 0; r < nranks_; ++r) {
      mx = std::max(mx, all[2 + 2 * size_t(r)]);
      cnt += all[3 + 2 * size_t(r)];
    }
  }
  *out_max = mx;
  *out_nonzero = int64_t(cnt);
  return 0;
}

// "<name>_mean" for every scalar array write_scored_results (or the plain writer) names, in its order: the sum of the
// means where the array is a sum over bins or time bins.  With two batches or more, "<name>_rel_err" follows for every
// such array that is exactly one (time bin, bin, score) result; a sum's error would need the covariances of its terms.
int Engine::batch_arrays(int32_t tally, const std::string &prefix, VtkArrays &a) {
  const size_t E = size_t(mesh_.ntets), S = size_t(nscores_), B = size_t(nbins_), T = nslices();
  std::vector<double> mean, rel;
  const bool errs = batches_ >= 2;
  if (copy_batch_results(mean, tally, 0) || (errs && copy_batch_results(rel, tally, 2))) return 1;
  auto add = [&](const std::string &name, std::vector<double> v) {
    a.data.push_back(std::move(v));  // (moving a vector keeps its storage: earlier pointers stay valid)
    a.named.emplace_back(prefix + name, a.data.back().data());
    a.ncomp.push_back(1);
  };
  auto at = [&](const std::vector<double> &v, size_t t, size_t b, size_t k) { return v.data() + ((t * B + b) * S + k) * E; };
  auto sum = [&](size_t t0, size_t t1, size_t b0, size_t b1, size_t k) {  // of the means
    std::vector<double> s(E, 0.0);
    for (size_t t = t0; t < t1; ++t)
      for (size_t b = b0; b < b1; ++b) {
        const double *p = at(mean, t, b, k);
        for (size_t i = 0; i < E; ++i) s[i] += p[i];
      }
    return s;
  };
  // set 0: the sum over the time bins (time bin 0 itself without a time filter); set 1 + j: time bin j
  const size_t nsets = ntime_ > 0 ? T + 1 : 1;
  for (size_t q = 0; q < nsets; ++q) {
    const std::string ts = q == 0 ? "" : "_t" + std::to_string(q - 1);
    const size_t t0 = q == 0 ? 0 : q - 1, t1 = q == 0 ? T : q;
    const bool single_time = ntime_ == 0 || q > 0;
    for (size_t k = 0; k < S; ++k) {
      const std::string name = (k == 0 ? "flux" : "score" + std::to_string(k)) + ts;
      add(name + "_mean", sum(t0, t1, 0, B, k));
      if (errs && single_time && B == 1) add(name + "_rel_err", std::vector<double>(at(rel, t0, 0, k), at(rel, t0, 0, k) + E));
      if (B > 1)
        for (size_t b = 0; b < B; ++b) {
          const std::string bn = name + "_bin" + std::to_string(b);
          add(bn + "_mean", sum(t0, t1, b, b + 1, k));
          if (errs && single_time) add(bn + "_rel_err", std::vector<double>(at(rel, t0, b, k), at(rel, t0, b, k) + E));
        }
    }
  }
  return 0;
}

// ------------------------------------------------------------------ face currents

int Engine::ensure_face_maps() {
  if (d_face_opp_) return 0;
  const int64_t E = mesh_.ntets;
  std::vector<uint32_t> opp(size_t(4 * E)), hull;
  for (int64_t e = 0; e < E; ++e)
    for (int f = 0; f < 4; ++f) {
      const int32_t nb = mesh_.t2t[size_t(4 * e + f)];
      int back = f;  // the neighbour's local index of the shared face, found as the packer finds it (tet_mesh.cpp)
      if (nb >= 0)
        for (int q = 0; q < 4; ++q)
          if (mesh_.t2t[4 * size_t(nb) + q] == int32_t(e)) back = q;
      opp[size_t(4 * e + f)] = nb >= 0 ? 4 * uint32_t(nb) + uint32_t(back) : kNoFace;
      if (nb < 0) hull.push_back(uint32_t(4 * e + f));
    }
  uint32_t *dopp = nullptr, *dhull = nullptr;
  if (cudaMalloc(reinterpret_cast<void **>(&dopp), opp.size() * sizeof(uint32_t)) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void **>(&dhull), std::max<size_t>(hull.size(), 1) * sizeof(uint32_t)) != cudaSuccess ||
      cudaMemcpy(dopp, opp.data(), opp.size() * sizeof(uint32_t), cudaMemcpyHostToDevice) != cudaSuccess ||
      (!hull.empty() &&
       cudaMemcpy(dhull, hull.data(), hull.size() * sizeof(uint32_t), cudaMemcpyHostToDevice) != cudaSuccess)) {
    const cudaError_t err = cudaGetLastError();
    cudaFree(dopp);
    cudaFree(dhull);
    fprintf(stderr, "[pumitally] ERROR: no device memory for the face maps (%s)\n", cudaGetErrorString(err));
    return 1;
  }
  d_face_opp_ = dopp;
  d_hull_slots_ = dhull;
  nhull_ = int64_t(hull.size());
  return 0;
}

int Engine::leakage_sums(const double *cur, double *out) {
  if (ensure_face_maps()) return 1;
  PTB_CUDA_OK(launch_leakage(cur, mesh_.ntets, cur_arrays(), d_hull_slots_, nhull_, out, compute_));
  return 0;
}

int Engine::get_face_current_results(int32_t direction, int32_t kind, double *out, int64_t n) {
  const int64_t E = mesh_.ntets, R = cur_arrays();
  const char *why = !currents_                               ? "face currents are off (set_face_currents)"
                    : (direction != 0 && direction != 1)     ? "direction must be 0 (outgoing) or 1 (incoming)"
                    : (kind < 0 || kind > 3)                 ? "kind must be 0 (value), 1 (batch mean), 2 (standard "
                                                               "error) or 3 (relative error)"
                    : (n != R * E * 4 || !out)               ? "n must be ntime * nbins * cosine bins * E * 4"
                                                             : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: get_face_current_results: %s\n", why);
    return 1;
  }
  if (kind > 0 && batch_refused(0, kind - 1)) return 1;
  if (synchronize() || ensure_element_maps() || ensure_face_maps()) return 1;
  double div = 1.0;
  const double *mean = nullptr, *m2 = nullptr;
  double *tmp = nullptr, *d_out = nullptr;
  if (kind == 0) {
    if (gather_shares() || !per_source_divisor(&div)) return 1;
    mean = flux_view();
  } else if (stats_view(&mean, &m2, &tmp)) {
    cudaFree(tmp);
    return 1;
  }
  const size_t base = current_base();
  cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&d_out), size_t(n) * sizeof(double));
  if (e == cudaSuccess)
    e = launch_current_readout(mean + base, m2 ? m2 + base : nullptr, d_face_opp_, d_orig_of_internal_, d_out, E,
                               int32_t(R), direction, kind - 1, double(batches_), div, compute_);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, size_t(n) * sizeof(double), cudaMemcpyDeviceToHost, compute_);
  if (e == cudaSuccess) e = cudaStreamSynchronize(compute_);
  cudaFree(d_out);
  cudaFree(tmp);
  if (e != cudaSuccess) {
    fprintf(stderr, "[pumitally] CUDA error %s reading the face currents\n", cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

// The open tally's leakage is summed from its hull slots (its leakage slots fill only at end_batch); the batch kinds
// read the folded leakage slots.
int Engine::get_leakage(int32_t kind, double *out, int64_t n) {
  const int64_t R = cur_arrays();
  const char *why = !currents_                 ? "face currents are off (set_face_currents)"
                    : (kind < 0 || kind > 3)   ? "kind must be 0 (value), 1 (batch mean), 2 (standard error) or 3 "
                                                 "(relative error)"
                    : (n != R || !out)         ? "n must be ntime * nbins * cosine bins"
                                               : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: get_leakage: %s\n", why);
    return 1;
  }
  if (kind > 0 && batch_refused(0, kind - 1)) return 1;
  if (synchronize()) return 1;
  std::vector<double> mean(static_cast<size_t>(R)), m2(static_cast<size_t>(R));
  if (kind == 0) {
    double div = 1.0, *d_sum = nullptr;
    if (gather_shares() || !per_source_divisor(&div)) return 1;
    PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_sum), size_t(R) * sizeof(double)));
    int rc = leakage_sums(flux_view() + current_base(), d_sum);
    if (!rc && (cudaMemcpyAsync(mean.data(), d_sum, size_t(R) * sizeof(double), cudaMemcpyDeviceToHost, compute_) !=
                    cudaSuccess ||
                cudaStreamSynchronize(compute_) != cudaSuccess))
      rc = 1;
    cudaFree(d_sum);
    if (rc) {
      fprintf(stderr, "[pumitally] CUDA error %s reading the leakage\n", cudaGetErrorString(cudaGetLastError()));
      return 1;
    }
    for (int64_t r = 0; r < R; ++r) out[r] = mean[size_t(r)] / div;
    return 0;
  }
  const double *dm = nullptr, *dq = nullptr;
  double *tmp = nullptr;
  int rc = stats_view(&dm, &dq, &tmp);
  if (!rc && (cudaMemcpy(mean.data(), dm + leak_base(), size_t(R) * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess ||
              cudaMemcpy(m2.data(), dq + leak_base(), size_t(R) * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess))
    rc = 1;
  cudaFree(tmp);
  if (rc) return 1;
  for (int64_t r = 0; r < R; ++r)
    out[r] = batch_readout(mean[size_t(r)], kind == 1 ? 0.0 : m2[size_t(r)], double(batches_), 1.0, kind - 1);
  return 0;
}

// With C > 1 cosine bins, also current_out_mu<k> and current_in_mu<k>: cosine bin k summed over time and score bins.
int Engine::current_arrays(VtkArrays &a) {
  const size_t E = size_t(mesh_.ntets), R = size_t(cur_arrays()), C = ncos();
  for (int32_t dir = 0; dir < 2; ++dir) {
    std::vector<double> all(R * E * 4);
    if (get_face_current_results(dir, 0, all.data(), int64_t(all.size()))) return 1;
    // per cosine bin k: the sum over the arrays r with r % C == k, into all[k * 4E ..]; then their sum into sum
    for (size_t r = C; r < R; ++r)
      for (size_t i = 0; i < E * 4; ++i) all[(r % C) * E * 4 + i] += all[r * E * 4 + i];
    all.resize(C * E * 4);
    // component k is the face opposite vertex k of the cell as written, which swaps vertices 2 and 3 of a negatively
    // oriented tet
    for (size_t k = 0; k < C; ++k)
      for (size_t i = 0; i < E; ++i)
        if (vtk_cell_flipped(mesh_, mesh_.t2v.data() + 4 * i)) {
          double *c = all.data() + k * E * 4 + 4 * size_t(mesh_.orig_of_internal[i]);
          std::swap(c[2], c[3]);
        }
    std::vector<double> sum(all.begin(), all.begin() + std::ptrdiff_t(E * 4));
    for (size_t k = 1; k < C; ++k)
      for (size_t i = 0; i < E * 4; ++i) sum[i] += all[k * E * 4 + i];
    const char *name = dir == 0 ? "current_out" : "current_in";
    a.data.push_back(std::move(sum));
    a.named.emplace_back(name, a.data.back().data());
    a.ncomp.push_back(4);
    for (size_t k = 0; C > 1 && k < C; ++k) {
      a.data.emplace_back(all.begin() + std::ptrdiff_t(k * E * 4), all.begin() + std::ptrdiff_t((k + 1) * E * 4));
      a.named.emplace_back(std::string(name) + "_mu" + std::to_string(k), a.data.back().data());
      a.ncomp.push_back(4);
    }
  }
  return 0;
}

// ------------------------------------------------------------------ region tallies

void Engine::free_regions() {
  cudaFree(d_region_elems_);
  cudaFree(d_region_starts_);
  cudaFree(d_region_ident_);
  cudaFree(d_region_volume_);
  cudaFree(d_region_work_);
  cudaFree(d_region_stats_);
  d_region_elems_ = d_region_starts_ = d_region_ident_ = nullptr;
  d_region_volume_ = d_region_work_ = d_region_stats_ = nullptr;
  region_scratch_ = 0;
  region_levels_.clear();
  region_volume_.clear();
  region_of_internal_.clear();
  nregions_ = 0;
}

int Engine::set_regions(const int32_t *region_of_element, int64_t n, int32_t nregions) {
  if (nccl_comm_) {
    fprintf(stderr, "[pumitally] ERROR: set_regions after comm_init (the batch statistics are sized by then)\n");
    return 1;
  }
  const int64_t E = mesh_.ntets;
  const bool remove = !region_of_element && nregions == 0;
  if (!remove) {
    const char *why = !region_of_element                  ? "the region map is null (remove the regions with nregions 0)"
                      : n != E                            ? "n must be the number of elements"
                      : (nregions < 1 || nregions > E)    ? "nregions must be in [1, number of elements]"
                                                          : nullptr;
    for (int64_t e = 0; !why && e < n; ++e)
      if (region_of_element[e] < -1 || region_of_element[e] >= nregions) why = "a region id is outside [-1, nregions)";
    if (why) {
      fprintf(stderr, "[pumitally] ERROR: set_regions: %s\n", why);
      return 1;
    }
  }
  if (synchronize()) return 1;
  // the new plan's device arrays first: nothing changes unless all of them (and fresh statistics) can be had
  RegionPlan plan;
  std::vector<double> vol;
  int32_t *elems = nullptr, *starts = nullptr, *ident = nullptr;
  double *dvol = nullptr;
  RegionCurrentPlan rc;  // with region currents on, the new map's pair plan
  int32_t *rc_dev[4] = {nullptr, nullptr, nullptr, nullptr};
  double *rc_ones = nullptr;
  auto release_rc = [&] {
    for (int32_t *d : rc_dev) cudaFree(d);
    cudaFree(rc_ones);
  };
  std::vector<int32_t> region_of_internal;
  if (!remove) {
    region_of_internal.resize(static_cast<size_t>(E));
    for (int64_t i = 0; i < E; ++i) region_of_internal[size_t(i)] = region_of_element[mesh_.orig_of_internal[size_t(i)]];
    plan = build_region_plan(region_of_internal.data(), E, nregions);
    vol = region_sums_host(plan, mesh_.volume.data());
    std::vector<int32_t> id(static_cast<size_t>(nregions));
    for (int32_t g = 0; g < nregions; ++g) id[size_t(g)] = g;
    auto up = [](auto **d, const auto &h) {
      const size_t bytes = std::max<size_t>(h.size(), 1) * sizeof(h[0]);
      return cudaMalloc(reinterpret_cast<void **>(d), bytes) == cudaSuccess &&
             cudaMemcpy(*d, h.data(), h.size() * sizeof(h[0]), cudaMemcpyHostToDevice) == cudaSuccess;
    };
    if (!up(&elems, plan.elems) || !up(&starts, plan.starts) || !up(&ident, id) || !up(&dvol, vol)) {
      const cudaError_t err = cudaGetLastError();
      cudaFree(elems); cudaFree(starts); cudaFree(ident); cudaFree(dvol);
      fprintf(stderr, "[pumitally] ERROR: no device memory for the regions (%s)\n", cudaGetErrorString(err));
      return 1;
    }
    if (rc_on() && build_region_currents(region_of_internal.data(), &rc, rc_dev, &rc_ones)) {
      cudaFree(elems); cudaFree(starts); cudaFree(ident); cudaFree(dvol);
      return 1;
    }
  }
  if (batch_stats_ && alloc_stats(reported_len())) {  // discards the folded batches (element and region)
    cudaFree(elems); cudaFree(starts); cudaFree(ident); cudaFree(dvol);
    release_rc();
    return 1;
  }
  free_regions();
  free_region_currents();  // removed, or replaced by the new map's plan below
  region_hash_ = remove ? 0 : ckpt::hash64(region_of_element, size_t(E) * sizeof(int32_t), uint64_t(nregions));
  if (!remove) {
    nregions_ = nregions;
    region_of_internal_ = std::move(region_of_internal);
    region_levels_ = plan.levels;
    region_volume_ = std::move(vol);
    d_region_elems_ = elems;
    d_region_starts_ = starts;
    d_region_ident_ = ident;
    d_region_volume_ = dvol;
    if (!rc.from.empty()) install_region_currents(std::move(rc), rc_dev, rc_ones);
  }
  return reset_tally();
}

int Engine::ensure_region_work() {
  const int64_t A = 2 * int64_t(result_arrays());  // (both tallies)
  RegionPlan p;
  p.levels = region_levels_;
  // the region sums of both tallies, or the region currents' partials and nets, whichever needs more
  const int64_t R = cur_arrays(), P = region_current_pair_count();
  const int64_t scratch = std::max(region_scratch_len(p, A, nscores_), region_scratch_len(rc_plan_.sums, R, 1));
  const size_t need = size_t(scratch) + std::max(size_t(A) * size_t(nregions_) * size_t(nscores_), 2 * size_t(R * P));
  if (d_region_work_ && scratch == region_scratch_ && need <= region_work_len_) return 0;
  cudaFree(d_region_work_);
  d_region_work_ = nullptr;
  region_work_len_ = 0;
  if (cudaMalloc(reinterpret_cast<void **>(&d_region_work_), std::max<size_t>(need, 1) * sizeof(double)) != cudaSuccess) {
    const cudaError_t err = cudaGetLastError();
    d_region_work_ = nullptr;
    fprintf(stderr, "[pumitally] ERROR: no device memory for the region sums (%s)\n", cudaGetErrorString(err));
    return 1;
  }
  region_scratch_ = scratch;
  region_work_len_ = need;
  return 0;
}

int Engine::ensure_region_stats() {
  if (d_region_stats_) return 0;
  const size_t bytes = std::max<size_t>(3 * region_len(), 1) * sizeof(double);
  if (cudaMalloc(reinterpret_cast<void **>(&d_region_stats_), bytes) != cudaSuccess ||
      cudaMemset(d_region_stats_, 0, bytes) != cudaSuccess) {
    const cudaError_t err = cudaGetLastError();
    cudaFree(d_region_stats_);
    d_region_stats_ = nullptr;
    fprintf(stderr, "[pumitally] ERROR: no device memory for the region statistics (%s)\n", cudaGetErrorString(err));
    return 1;
  }
  return 0;
}

int Engine::region_sums(const double *flux, int64_t narrays, double *out) {
  PTB_CUDA_OK(launch_region_sums(flux, int64_t(bin_len()), stride_, nscores_, narrays, d_region_elems_,
                                 d_region_starts_, region_levels_.data(), int(region_levels_.size()), d_region_work_,
                                 region_scratch_, out, compute_));
  return 0;
}

bool Engine::region_refused(int32_t tally, int32_t kind, int32_t max_kind, int64_t n) const {
  const int64_t one = nregions_, all = int64_t(result_arrays()) * nscores_ * nregions_;
  const char *why = nregions_ == 0                          ? "no regions are set (set_regions)"
                    : (tally != 0 && tally != 1)            ? "tally must be 0 (track length) or 1 (collision)"
                    : (tally == 1 && !collision_)           ? "the collision estimator is off (set_collision_estimator)"
                    : (kind < 0 || kind > max_kind)         ? "kind out of range"
                    : (n != one && n != all)                ? "n must be nregions or ntime * nbins * nscores * nregions"
                                                            : nullptr;
  if (why) fprintf(stderr, "[pumitally] ERROR: region results refused: %s\n", why);
  return why != nullptr;
}

int Engine::get_region_volumes(double *out, int64_t n) {
  if (nregions_ == 0 || n != nregions_) {
    fprintf(stderr, "[pumitally] ERROR: get_region_volumes: %s\n", nregions_ ? "n must be nregions" : "no regions are set");
    return 1;
  }
  std::memcpy(out, region_volume_.data(), size_t(n) * sizeof(double));
  return 0;
}

// The region sums of the open tally, read where copy_results reads it (flux_view(), after gather_shares()).  Kind 1
// divides as normalize_scores does, sum / V_G / d: a one-element region gives get_normalized_flux's bits.
int Engine::get_region_results(int32_t tally, int32_t kind, double *out, int64_t n) {
  if (region_refused(tally, kind, 1, n)) return 1;
  if (synchronize() || gather_shares() || ensure_region_work()) return 1;
  double per_source = 1.0;
  if (kind == 1 && !per_source_divisor(&per_source)) return 1;
  const size_t R = size_t(result_arrays()), S = size_t(nscores_), G = size_t(nregions_);
  double *d_out = d_region_work_ + region_scratch_;
  if (region_sums(flux_view() + size_t(tally) * flux_len(), int64_t(R), d_out)) return 1;
  const int64_t rows = n / int64_t(G);  // (r, k) pairs asked for: 1, or all of them
  std::vector<double> sums(size_t(n) == G ? G * S : R * G * S);
  PTB_CUDA_OK(cudaMemcpyAsync(sums.data(), d_out, sums.size() * sizeof(double), cudaMemcpyDeviceToHost, compute_));
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  const double *vol = region_volume_.data();
#pragma omp parallel for schedule(static)
  for (int64_t q = 0; q < rows; ++q) {  // [r][g][k] -> [r][k][g]
    const size_t r = size_t(q) / S, k = size_t(q) % S;
    const double *src = sums.data() + r * G * S + k;
    double *dst = out + size_t(q) * G;
    if (kind == 1)
      for (size_t g = 0; g < G; ++g) dst[g] = src[g * S] / vol[g] / per_source;
    else
      for (size_t g = 0; g < G; ++g) dst[g] = src[g * S];
  }
  return 0;
}

int Engine::get_region_batch_results(int32_t tally, int32_t kind, double *out, int64_t n) {
  if (region_refused(tally, kind, 2, n) || batch_refused(tally, kind)) return 1;
  if (synchronize()) return 1;
  const size_t R = size_t(result_arrays()), S = size_t(nscores_), G = size_t(nregions_), RL = region_len();
  const size_t base = size_t(tally) * R * G * S;
  double *d_out = nullptr;
  cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&d_out), R * S * G * sizeof(double));
  if (e == cudaSuccess)
    e = launch_batch_readout(d_region_stats_ + RL + base, d_region_stats_ + 2 * RL + base, d_region_volume_,
                             d_region_ident_, d_out, int64_t(G), int32_t(R), nscores_, nscores_, double(batches_), kind,
                             compute_);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, size_t(n) * sizeof(double), cudaMemcpyDeviceToHost, compute_);
  if (e == cudaSuccess) e = cudaStreamSynchronize(compute_);
  cudaFree(d_out);
  if (e != cudaSuccess) {
    fprintf(stderr, "[pumitally] CUDA error %s reading the region statistics\n", cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

// ------------------------------------------------------------------ region currents

void Engine::free_region_currents() {
  cudaFree(d_rc_slots_);
  cudaFree(d_rc_starts_);
  cudaFree(d_rc_rev_);
  cudaFree(d_rc_ident_);
  cudaFree(d_rc_ones_);
  d_rc_slots_ = d_rc_starts_ = d_rc_rev_ = d_rc_ident_ = nullptr;
  d_rc_ones_ = nullptr;
  rc_plan_ = RegionCurrentPlan();
}

int Engine::build_region_currents(const int32_t *region_of_internal, RegionCurrentPlan *plan, int32_t *dev[4],
                                  double **ones) {
  const int64_t E = mesh_.ntets;
  std::vector<double> area(size_t(4 * E));
  for (int64_t e = 0; e < E; ++e)
    for (int f = 0; f < 4; ++f) area[size_t(4 * e + f)] = face_area(mesh_.coords.data(), mesh_.t2v.data(), e, f);
  *plan = build_region_current_plan(region_of_internal, mesh_.t2t.data(), E, area.data());
  const size_t P = plan->from.size();
  std::vector<int32_t> id(P);
  for (size_t q = 0; q < P; ++q) id[q] = int32_t(q);
  const std::vector<double> one(P, 1.0);
  auto up = [](auto **d, const auto &h) {
    const size_t bytes = std::max<size_t>(h.size(), 1) * sizeof(h[0]);
    return cudaMalloc(reinterpret_cast<void **>(d), bytes) == cudaSuccess &&
           cudaMemcpy(*d, h.data(), h.size() * sizeof(h[0]), cudaMemcpyHostToDevice) == cudaSuccess;
  };
  if (!up(&dev[0], plan->sums.elems) || !up(&dev[1], plan->sums.starts) || !up(&dev[2], plan->rev) ||
      !up(&dev[3], id) || !up(ones, one)) {
    const cudaError_t err = cudaGetLastError();
    for (int i = 0; i < 4; ++i) cudaFree(dev[i]);
    cudaFree(*ones);
    fprintf(stderr, "[pumitally] ERROR: no device memory for the region currents (%s)\n", cudaGetErrorString(err));
    return 1;
  }
  return 0;
}

void Engine::install_region_currents(RegionCurrentPlan &&plan, int32_t *dev[4], double *ones) {
  rc_plan_ = std::move(plan);
  d_rc_slots_ = dev[0];
  d_rc_starts_ = dev[1];
  d_rc_rev_ = dev[2];
  d_rc_ident_ = dev[3];
  d_rc_ones_ = ones;
}

int Engine::set_region_currents(int32_t on) {
  const int64_t E = mesh_.ntets;
  const char *why = (on != 0 && on != 1)               ? "on must be 0 or 1"
                    : nccl_comm_                        ? "after comm_init (the batch statistics are sized by then)"
                    : (on && nregions_ == 0)            ? "no regions are set (set_regions)"
                    : (on && !currents_)                ? "face currents are off (set_face_currents)"
                    : (on && 4 * E > INT32_MAX)         ? "4 * number of elements exceeds INT32_MAX"
                                                        : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: set_region_currents: %s\n", why);
    return 1;
  }
  if (synchronize()) return 1;
  RegionCurrentPlan plan;
  int32_t *dev[4] = {nullptr, nullptr, nullptr, nullptr};
  double *ones = nullptr;
  if (on) {
    if (build_region_currents(region_of_internal_.data(), &plan, dev, &ones)) return 1;
  }
  if (batch_stats_ && alloc_stats(reported_len())) {  // discards the folded batches (element and region)
    for (int32_t *d : dev) cudaFree(d);
    cudaFree(ones);
    return 1;
  }
  free_region_currents();
  if (on) install_region_currents(std::move(plan), dev, ones);
  return reset_tally();
}

int Engine::get_region_current_pairs(int32_t *from, int32_t *to, int64_t n) {
  const int64_t P = region_current_pair_count();
  if (!rc_on() || n != P || !from || !to) {
    fprintf(stderr, "[pumitally] ERROR: get_region_current_pairs: %s\n",
            rc_on() ? "n must be the pair count" : "region currents are off (set_region_currents)");
    return 1;
  }
  std::memcpy(from, rc_plan_.from.data(), size_t(P) * sizeof(int32_t));
  std::memcpy(to, rc_plan_.to.data(), size_t(P) * sizeof(int32_t));
  return 0;
}

int Engine::get_region_current_areas(double *out, int64_t n) {
  if (!rc_on() || n != region_current_pair_count() || !out) {
    fprintf(stderr, "[pumitally] ERROR: get_region_current_areas: %s\n",
            rc_on() ? "n must be the pair count" : "region currents are off (set_region_currents)");
    return 1;
  }
  std::memcpy(out, rc_plan_.area.data(), size_t(n) * sizeof(double));
  return 0;
}

int Engine::region_current_sums(const double *cur, double *out) {
  const int64_t R = cur_arrays(), P = region_current_pair_count();
  PTB_CUDA_OK(launch_region_sums(cur, 4 * mesh_.ntets, 1, 1, R, d_rc_slots_, d_rc_starts_, rc_plan_.sums.levels.data(),
                                 int(rc_plan_.sums.levels.size()), d_region_work_, region_scratch_, out, compute_));
  PTB_CUDA_OK(launch_region_net(out, d_rc_rev_, P, R, out + R * P, compute_));
  return 0;
}

int Engine::get_region_current_results(int32_t which, int32_t kind, double *out, int64_t n) {
  const int64_t R = cur_arrays(), P = region_current_pair_count();
  const char *why = !rc_on()                            ? "region currents are off (set_region_currents)"
                    : (which != 0 && which != 1)        ? "which must be 0 (partial) or 1 (net)"
                    : (kind < 0 || kind > 3)            ? "kind must be 0 (value), 1 (batch mean), 2 (standard "
                                                          "error) or 3 (relative error)"
                    : (n != R * P || !out)              ? "n must be ntime * nbins * cosine bins * the pair count"
                                                        : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: get_region_current_results: %s\n", why);
    return 1;
  }
  if (kind > 0 && batch_refused(0, kind - 1)) return 1;
  if (synchronize()) return 1;
  if (kind == 0) {  // the open tally's currents, read where get_region_results reads the tally
    double div = 1.0;
    if (gather_shares() || !per_source_divisor(&div) || ensure_region_work()) return 1;
    double *d_out = d_region_work_ + region_scratch_;
    if (region_current_sums(flux_view() + current_base(), d_out)) return 1;
    PTB_CUDA_OK(cudaMemcpyAsync(out, d_out + size_t(which) * size_t(R * P), size_t(n) * sizeof(double),
                                cudaMemcpyDeviceToHost, compute_));
    PTB_CUDA_OK(cudaStreamSynchronize(compute_));
    for (int64_t i = 0; i < n; ++i) out[i] /= div;
    return 0;
  }
  if (ensure_region_stats()) return 1;
  const size_t RL = region_len(), base = rc_base() + size_t(which) * size_t(R * P);
  double *d_out = nullptr;
  cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&d_out), std::max<size_t>(size_t(n), 1) * sizeof(double));
  if (e == cudaSuccess)
    e = launch_batch_readout(d_region_stats_ + RL + base, d_region_stats_ + 2 * RL + base, d_rc_ones_, d_rc_ident_,
                             d_out, P, int32_t(R), 1, 1, double(batches_), kind - 1, compute_);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, size_t(n) * sizeof(double), cudaMemcpyDeviceToHost, compute_);
  if (e == cudaSuccess) e = cudaStreamSynchronize(compute_);
  cudaFree(d_out);
  if (e != cudaSuccess) {
    fprintf(stderr, "[pumitally] CUDA error %s reading the region-current statistics\n", cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

// ------------------------------------------------------------------ checkpoints

namespace {

constexpr size_t kCheckpointChunk = size_t(64) << 20;  // bytes per pinned chunk buffer; two per call

// The two pinned chunk buffers of one save, load or merge, each with the event of its last device copy.
struct ChunkBuffers {
  void *h[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  size_t bytes = 0;
  bool ok = true;
  explicit ChunkBuffers(size_t b) : bytes(b) {
    for (int i = 0; i < 2; ++i)
      ok = ok && cudaHostAlloc(&h[i], b, cudaHostAllocDefault) == cudaSuccess &&
           cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) cudaGetLastError();
  }
  ~ChunkBuffers() {
    for (int i = 0; i < 2; ++i) {
      if (h[i]) cudaFreeHost(h[i]);
      if (ev[i]) cudaEventDestroy(ev[i]);
    }
  }
};

// chunk size for sections of at most `largest` bytes: no 128 MB of pinned memory for a small tally
size_t chunk_bytes_for(uint64_t largest) {
  return size_t(std::max<uint64_t>(4096, std::min<uint64_t>(kCheckpointChunk, largest)));
}

}  // namespace

ckpt::Fingerprint Engine::fingerprint() {
  const size_t E = size_t(mesh_.ntets);
  if (!mesh_hashed_) {  // computed once: the mesh never changes
    std::vector<int32_t> t2v(4 * E);  // in the caller's numbering
    for (size_t i = 0; i < E; ++i)
      std::memcpy(&t2v[4 * size_t(mesh_.orig_of_internal[i])], &mesh_.t2v[4 * i], 4 * sizeof(int32_t));
    mesh_hash_ = ckpt::hash64(t2v.data(), t2v.size() * sizeof(int32_t),
                              ckpt::hash64(mesh_.coords.data(), mesh_.coords.size() * sizeof(double)));
    order_hash_ = ckpt::hash64(mesh_.orig_of_internal.data(), E * sizeof(int32_t));
    mesh_hashed_ = true;
  }
  ckpt::Fingerprint f;
  f.nelems = mesh_.ntets;
  f.nverts = mesh_.nverts;
  f.mesh_hash = mesh_hash_;
  f.order_hash = order_hash_;
  f.nbins = nbins_;
  f.nscores = nscores_;
  f.stride = stride_;
  f.moments = moments_;
  f.collision = collision_ ? 1 : 0;
  f.batch_stats = batch_stats_ ? 1 : 0;
  f.nregions = nregions_;
  f.region_hash = region_hash_;
  f.norm_mode = norm_mode_;
  f.norm_value = norm_mode_ == 2 ? norm_value_ : 0.0;
  f.rank = sharded() ? rank_ : 0;
  f.nranks = sharded() ? nranks_ : 1;
  f.share = sharded() ? share_ : 0;
  if (ntime_ > 0) {
    f.edges.resize(size_t(ntime_) + 1);
    if (cudaMemcpy(f.edges.data(), d_edges_, f.edges.size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess)
      f.edges.assign(f.edges.size(), std::nan(""));  // (compares unequal to every file's edges)
  }
  if (currents_) f.mu_edges = mu_edges_;  // the cosine bins shape the arrays only with face currents on
  f.det_xyz = det_xyz_;
  f.det_r0 = det_r0_;
  f.sigma_crc = ndet_ > 0 && d_sigma_ ? sigma_crc_ : 0;
  f.det_void = det_void_ && ndet_ > 0 ? 1 : 0;  // without detectors the mode shapes nothing a file holds
  return f;
}

int Engine::save_checkpoint(const std::string &path) {
  if (synchronize()) return 1;
  auto refuse = [&](const std::string &why) {
    fprintf(stderr, "[pumitally] ERROR: save_checkpoint: %s: %s\n", path.c_str(), why.c_str());
    return 1;
  };
  const ckpt::Fingerprint f = fingerprint();
  ckpt::Header h;
  const size_t RL = batch_stats_ && nregions_ ? region_len() : 0;
  h.batches = batch_stats_ ? batches_ : 0;
  h.open = tallied_ ? 1 : 0;
  h.open_len = tallied_ ? reported_len() : 0;
  h.stats_len = batch_stats_ ? stats_len() : 0;
  h.region_len = RL;
  const size_t DL = det_len();
  h.det_len = DL;
  h.det_words = uint32_t(f.det_void ? ckpt::kDetCountWordsVoid : ckpt::kDetCountWords);
  std::vector<uint8_t> scalars, det_counts;
  if (tallied_) {
    ckpt::OpenScalars s;
    DeviceStats ds;
    unsigned long long cc[3];
    PTB_CUDA_OK(cudaMemcpy(&s.initial_weight, d_initial_weight_, sizeof(double), cudaMemcpyDeviceToHost));
    PTB_CUDA_OK(cudaMemcpy(&ds, d_stats_, sizeof(ds), cudaMemcpyDeviceToHost));
    PTB_CUDA_OK(cudaMemcpy(cc, d_coll_counts_, sizeof(cc), cudaMemcpyDeviceToHost));
    s.initial_weight_pending = initial_weight_pending_ ? 1 : 0;
    for (int i = 0; i < 3; ++i) s.coll_counts[i] = cc[i];
    s.segments = ds.segments;
    s.tracks = ds.tracks;
    s.relocations = ds.relocations;
    s.lost = ds.lost;
    s.fallbacks = ds.fallbacks;
    s.moves = moves_;
    s.scored_moves = scored_moves_;
    scalars = ckpt::pack_open_scalars(s);
    if (DL) {
      unsigned long long dc[kDetCountersVoid];  // the hull entries (the last) only with the detector void on
      PTB_CUDA_OK(cudaMemcpy(dc, d_det_counts_, sizeof(dc), cudaMemcpyDeviceToHost));
      det_counts.resize(8 * size_t(h.det_words));
      std::memcpy(det_counts.data(), dc, det_counts.size());  // (little-endian hosts only, as the rest of the engine)
    }
  }
  // the arrays of the sections, in file order (nullptr: zeros -- region statistics before the first end_batch)
  struct Src { uint32_t id; const double *d; const uint8_t *host; uint64_t bytes; };
  std::vector<Src> src;
  if (h.open) {
    src.push_back({ckpt::kOpenTally, d_flux_, nullptr, 8 * h.open_len});
    src.push_back({ckpt::kOpenScalars, nullptr, scalars.data(), scalars.size()});
  }
  if (h.stats_len) {
    src.push_back({ckpt::kMean, d_mean_, nullptr, 8 * h.stats_len});
    src.push_back({ckpt::kM2, d_m2_, nullptr, 8 * h.stats_len});
  }
  if (RL) {
    src.push_back({ckpt::kRegionMean, d_region_stats_ ? d_region_stats_ + RL : nullptr, nullptr, 8 * RL});
    src.push_back({ckpt::kRegionM2, d_region_stats_ ? d_region_stats_ + 2 * RL : nullptr, nullptr, 8 * RL});
  }
  if (DL && h.open) {
    src.push_back({ckpt::kDetOpen, d_det_, nullptr, 8 * DL});
    src.push_back({ckpt::kDetCounts, nullptr, det_counts.data(), det_counts.size()});
  }
  if (DL && h.stats_len) {  // (zeros before the first end_batch: the fold starts from zeros then too)
    src.push_back({ckpt::kDetMean, batches_ > 0 ? d_det_ + 2 * DL : nullptr, nullptr, 8 * DL});
    src.push_back({ckpt::kDetM2, batches_ > 0 ? d_det_ + 3 * DL : nullptr, nullptr, 8 * DL});
  }
  uint64_t largest = 0;
  for (const Src &s : src) largest = std::max(largest, s.bytes);
  ChunkBuffers buf(chunk_bytes_for(largest));
  if (!buf.ok) return refuse("no pinned host memory for the chunk buffers");
  const std::string tmp = path + ".tmp";
  FILE *fp = std::fopen(tmp.c_str(), "wb");
  if (!fp) return refuse(std::string("cannot create ") + tmp + " (" + std::strerror(errno) + ")");
  ckpt::Writer w([&](const void *p, size_t n) { return std::fwrite(p, 1, n, fp) == n; },
                 [&](uint64_t off, const void *p, size_t n) {
                   return fseeko(fp, off_t(off), SEEK_SET) == 0 && std::fwrite(p, 1, n, fp) == n &&
                          fseeko(fp, 0, SEEK_END) == 0;
                 });
  bool ok = w.begin(h, f);
  for (const Src &s : src) {
    if (!ok) break;
    const size_t C = buf.bytes;
    // Chunk k + 1 is copied into the other buffer (whose chunk k - 1 has been written) while chunk k is checksummed
    // and written.
    auto issue = [&](size_t k) {
      const uint64_t off = uint64_t(k) * C;
      if (off >= s.bytes) return true;
      const size_t n = size_t(std::min<uint64_t>(C, s.bytes - off));
      if (!s.d) {
        std::memset(buf.h[k & 1], 0, n);
        return true;
      }
      return cudaMemcpyAsync(buf.h[k & 1], reinterpret_cast<const char *>(s.d) + off, n, cudaMemcpyDeviceToHost,
                             copy_) == cudaSuccess &&
             cudaEventRecord(buf.ev[k & 1], copy_) == cudaSuccess;
    };
    if (s.host) {
      ok = w.section(s.id, s.bytes, C, [&](size_t, uint64_t off, size_t) -> const void * { return s.host + off; });
    } else {
      ok = w.section(s.id, s.bytes, C, [&](size_t k, uint64_t, size_t) -> const void * {
        if ((k == 0 && !issue(0)) || !issue(k + 1)) return nullptr;
        if (s.d && cudaEventSynchronize(buf.ev[k & 1]) != cudaSuccess) return nullptr;
        return buf.h[k & 1];
      });
    }
  }
  cudaStreamSynchronize(copy_);  // (nothing may still be copying into the buffers when they are freed)
  std::string why = ok ? "" : (w.error().empty() ? "write failed" : w.error());
  if (ok && (std::fflush(fp) != 0 || fsync(fileno(fp)) != 0)) {
    ok = false;
    why = std::string("flush failed (") + std::strerror(errno) + ")";
  }
  if (std::fclose(fp) != 0 && ok) {
    ok = false;
    why = std::string("close failed (") + std::strerror(errno) + ")";
  }
  if (ok && std::rename(tmp.c_str(), path.c_str()) != 0) {
    ok = false;
    why = std::string("cannot rename ") + tmp + " (" + std::strerror(errno) + ")";
  }
  if (!ok) {
    std::remove(tmp.c_str());
    cudaGetLastError();
    return refuse(why);
  }
  return 0;
}

int Engine::load_checkpoint(const std::string &path) { return read_checkpoint(path, false); }
int Engine::merge_checkpoint(const std::string &path) { return read_checkpoint(path, true); }

// Load: every section arrives in new device buffers, which replace the engine's only once all of them arrived intact.
// Merge: the file's statistics arrive in device scratch and are merged into the engine's by one launch per array.
int Engine::read_checkpoint(const std::string &path, bool merge) {
  const char *what = merge ? "merge_checkpoint" : "load_checkpoint";
  auto refuse = [&](const std::string &why) {
    fprintf(stderr, "[pumitally] ERROR: %s: %s: %s\n", what, path.c_str(), why.c_str());
    return 1;
  };
  if (merge && !batch_stats_) return refuse("batch statistics are off (set_batch_statistics)");
  if (synchronize()) return 1;
  FILE *fp = std::fopen(path.c_str(), "rb");
  if (!fp) return refuse(std::strerror(errno));
  std::unique_ptr<FILE, int (*)(FILE *)> closer(fp, std::fclose);
  struct stat st;
  if (fstat(fileno(fp), &st) != 0 || !S_ISREG(st.st_mode)) return refuse("not a regular file");
  ckpt::Reader r([&](void *p, size_t n) { return std::fread(p, 1, n, fp) == n; }, uint64_t(st.st_size));
  ckpt::Header h;
  ckpt::Fingerprint ff;
  if (!r.begin(&h, &ff)) return refuse(r.error());
  if (const char *field = ckpt::fingerprint_mismatch(fingerprint(), ff, merge))
    return refuse(std::string("the checkpoint differs from this engine in: ") + field);
  const size_t RL = batch_stats_ && nregions_ ? region_len() : 0;
  // the lengths this engine would have with face currents on or off (the fingerprint does not hold the setting)
  auto lengths_match = [&](bool currents, size_t region_len) {
    const size_t rep = reported_len_for(currents);
    const size_t SL = !batch_stats_ ? 0 : sharded() ? (rep + size_t(nranks_) - 1) / size_t(nranks_) : rep;
    return h.stats_len == SL && h.region_len == region_len && (!h.open || h.open_len == rep) &&
           (batch_stats_ || h.batches == 0) && h.det_len == det_len();
  };
  // Region currents add 2 ntime nbins P region results (P >= 1: every mesh has a hull), and need face currents.  Saved
  // with them on, a file has face currents on and a region length above rc_base() by a multiple of 2 ntime nbins.
  const size_t RCA = 2 * size_t(cur_arrays());
  const bool rc_differ = RL && (rc_on() ? lengths_match(true, rc_base())
                                        : h.region_len > RL && (h.region_len - RL) % RCA == 0 &&
                                              lengths_match(true, h.region_len));
  if (!lengths_match(currents_, RL))
    return refuse(lengths_match(!currents_, RL)
                      ? std::string("the face currents differ: the checkpoint was saved with them ") +
                            (currents_ ? "off" : "on") + " (set_face_currents)"
                  : rc_differ ? std::string("the region currents differ: the checkpoint was saved with them ") +
                                    (rc_on() ? "off" : "on") + " (set_region_currents)"
                              : std::string("the declared lengths do not match this engine's configuration"));
  const size_t SL = batch_stats_ ? stats_len() : 0;
  if (merge && h.open)
    return refuse("the checkpoint holds an open batch, which a merge would drop (save at a batch end)");
  // new buffers: the open tally (whole allocation, zero past the reported part), the statistics, the region statistics
  // (load: the engine's [sums][mean][M2] layout; merge: [mean][M2] scratch)
  double *nflux = nullptr, *nmean = nullptr, *nm2 = nullptr, *nreg = nullptr, *ndet = nullptr;
  const size_t DL = det_len();
  auto release = [&] {
    cudaFree(ndet);
    cudaFree(nflux);
    cudaFree(nmean);
    cudaFree(nm2);
    cudaFree(nreg);
    cudaGetLastError();
  };
  auto alloc = [&](double **p, size_t n) {
    return cudaMalloc(reinterpret_cast<void **>(p), std::max<size_t>(n, 1) * sizeof(double)) == cudaSuccess &&
           cudaMemset(*p, 0, std::max<size_t>(n, 1) * sizeof(double)) == cudaSuccess;
  };
  const size_t reg_off = merge ? 0 : RL;  // where the region means go in nreg
  if ((!merge && h.open && !alloc(&nflux, flux_alloc_)) || (SL && (!alloc(&nmean, SL) || !alloc(&nm2, SL))) ||
      (RL && !alloc(&nreg, (merge ? 2 : 3) * RL)) || (DL && alloc_detectors(DL, batch_stats_, &ndet))) {
    release();
    return refuse("no device memory for a second copy of the checkpoint's arrays");
  }
  std::vector<uint8_t> scalars(8 * ckpt::kOpenScalarWords), det_counts(8 * size_t(h.det_words));
  struct Dst { uint32_t id; double *d; uint64_t bytes; };
  std::vector<Dst> dst;
  if (h.open) {
    dst.push_back({ckpt::kOpenTally, nflux, 8 * h.open_len});
    dst.push_back({ckpt::kOpenScalars, nullptr, scalars.size()});
  }
  if (SL) {
    dst.push_back({ckpt::kMean, nmean, 8 * SL});
    dst.push_back({ckpt::kM2, nm2, 8 * SL});
  }
  if (RL) {
    dst.push_back({ckpt::kRegionMean, nreg + reg_off, 8 * RL});
    dst.push_back({ckpt::kRegionM2, nreg + reg_off + RL, 8 * RL});
  }
  if (DL && h.open) {  // [open] of the new detector buffer; the counters arrive on the host
    dst.push_back({ckpt::kDetOpen, ndet, 8 * DL});
    dst.push_back({ckpt::kDetCounts, nullptr, det_counts.size()});
  }
  if (DL && SL) {  // [mean][M2] of the new detector buffer
    dst.push_back({ckpt::kDetMean, ndet + 2 * DL, 8 * DL});
    dst.push_back({ckpt::kDetM2, ndet + 3 * DL, 8 * DL});
  }
  uint64_t largest = 0;
  for (const Dst &d : dst) largest = std::max(largest, d.bytes);
  bool ok = true;
  std::string why;
  {
    ChunkBuffers buf(chunk_bytes_for(largest));
    if (!buf.ok) {
      ok = false;
      why = "no pinned host memory for the chunk buffers";
    }
    for (const Dst &d : dst) {
      if (!ok) break;
      if (!d.d) {
        uint8_t *host = d.id == ckpt::kDetCounts ? det_counts.data() : scalars.data();
        ok = r.section(d.id, d.bytes, buf.bytes, [&](size_t) -> void * { return host; },
                       [](size_t, uint64_t, const void *, size_t) { return true; });
      } else {
        // chunk k is read into the buffer whose last copy (chunk k - 2, or a chunk of the section before) has finished;
        // its own copy then overlaps the reading and checksumming of chunk k + 1
        ok = r.section(
            d.id, d.bytes, buf.bytes,
            [&](size_t k) -> void * {
              return cudaEventSynchronize(buf.ev[k & 1]) == cudaSuccess ? buf.h[k & 1] : nullptr;
            },
            [&](size_t k, uint64_t off, const void *p, size_t n) {
              return cudaMemcpyAsync(reinterpret_cast<char *>(d.d) + off, p, n, cudaMemcpyHostToDevice, copy_) ==
                         cudaSuccess &&
                     cudaEventRecord(buf.ev[k & 1], copy_) == cudaSuccess;
            });
      }
      if (!ok) why = r.error();
    }
    if (cudaStreamSynchronize(copy_) != cudaSuccess && ok) {
      ok = false;
      why = "a copy to the device failed";
    }
  }
  ckpt::OpenScalars sc;
  if (ok && !r.at_end()) {
    ok = false;
    why = "data after the last section";
  }
  if (ok && h.open && !ckpt::unpack_open_scalars(scalars.data(), scalars.size(), &sc)) {
    ok = false;
    why = "corrupt open-batch counters";
  }
  if (ok && merge && RL && ensure_region_stats()) {
    ok = false;
    why = "no device memory for the region statistics";
  }
  if (!ok) {
    release();
    return refuse(why);
  }
  if (merge) {  // in place, (na, nb) -> na + nb batches; a file of no batches changes nothing
    if (h.batches > 0) {
      const double na = double(batches_), nb = double(h.batches);
      cudaError_t e = launch_batch_merge(nmean, nm2, d_mean_, d_m2_, int64_t(SL), na, nb, compute_);
      if (e == cudaSuccess && RL)
        e = launch_batch_merge(nreg, nreg + RL, d_region_stats_ + RL, d_region_stats_ + 2 * RL, int64_t(RL), na, nb,
                               compute_);
      if (e == cudaSuccess && DL) {
        if (batches_ == 0) e = cudaMemsetAsync(d_det_ + 2 * DL, 0, 2 * DL * sizeof(double), compute_);
        if (e == cudaSuccess)
          e = launch_batch_merge(ndet + 2 * DL, ndet + 3 * DL, d_det_ + 2 * DL, d_det_ + 3 * DL, int64_t(DL), na, nb,
                                 compute_);
      }
      if (e == cudaSuccess) e = cudaStreamSynchronize(compute_);
      release();
      PTB_CUDA_OK(e);
      batches_ += h.batches;
    } else {
      release();
    }
    return 0;
  }
  // load: swap the new state in
  if (h.open) {
    cudaFree(d_flux_);
    d_flux_ = nflux;
    nflux = nullptr;
  } else {
    PTB_CUDA_OK(cudaMemset(d_flux_, 0, flux_alloc_ * sizeof(double)));  // (sc: a reset tally's counters)
  }
  if (SL) {
    cudaFree(d_mean_);
    cudaFree(d_m2_);
    d_mean_ = nmean;
    d_m2_ = nm2;
    nmean = nm2 = nullptr;
  }
  if (RL) {
    cudaFree(d_region_stats_);
    d_region_stats_ = nreg;
    nreg = nullptr;
  }
  if (DL) {
    cudaFree(d_det_);
    d_det_ = ndet;
    ndet = nullptr;
    det_global_valid_ = false;
    unsigned long long dc[kDetCountersVoid] = {};
    if (h.open) std::memcpy(dc, det_counts.data(), det_counts.size());
    PTB_CUDA_OK(cudaMemcpy(d_det_counts_, dc, sizeof(dc), cudaMemcpyHostToDevice));
  }
  batches_ = h.batches;
  DeviceStats ds{sc.segments, sc.tracks, sc.relocations, sc.lost, sc.fallbacks};
  const unsigned long long cc[3] = {sc.coll_counts[0], sc.coll_counts[1], sc.coll_counts[2]};
  PTB_CUDA_OK(cudaMemcpy(d_initial_weight_, &sc.initial_weight, sizeof(double), cudaMemcpyHostToDevice));
  PTB_CUDA_OK(cudaMemcpy(d_stats_, &ds, sizeof(ds), cudaMemcpyHostToDevice));
  PTB_CUDA_OK(cudaMemcpy(d_coll_counts_, cc, sizeof(cc), cudaMemcpyHostToDevice));
  initial_weight_pending_ = sc.initial_weight_pending != 0;
  moves_ = sc.moves;
  scored_moves_ = sc.scored_moves;
  tallied_ = h.open != 0;
  flux_global_valid_ = flux_owned_only_ = eval_valid_ = false;
  return 0;
}

// ------------------------------------------------------------------ weight windows

void Engine::free_weight_windows() {
  cudaFree(d_ww_);
  d_ww_ = nullptr;
  ww_groups_ = 0;
}

int Engine::alloc_weight_windows(int32_t ngroups, double2 **out) {
  const size_t bytes = size_t(ngroups) * size_t(std::max<int64_t>(mesh_.ntets, 1)) * sizeof(double2);
  if (cudaMalloc(reinterpret_cast<void **>(out), bytes) != cudaSuccess) {
    const cudaError_t err = cudaGetLastError();
    *out = nullptr;
    fprintf(stderr, "[pumitally] ERROR: no device memory for the weight windows (%zu bytes: %s)\n", bytes,
            cudaGetErrorString(err));
    return 1;
  }
  return 0;
}

int Engine::set_weight_windows(const double *lower, const double *upper, int64_t n, int32_t ngroups) {
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (!lower && ngroups == 0) {
    if (synchronize()) return 1;  // a device lookup may still read the table
    free_weight_windows();
    return 0;
  }
  const int64_t E = mesh_.ntets;
  const char *why = ngroups < 1                       ? "ngroups must be >= 1 (0 with lower == NULL removes the windows)"
                    : (!lower || !upper)              ? "null bound array"
                    : n != int64_t(ngroups) * E       ? "n must be ngroups * num_elements"
                                                      : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: set_weight_windows refused: %s\n", why);
    return 1;
  }
  std::vector<double2> h = std::vector<double2>(size_t(n));
  for (int64_t g = 0; g < ngroups; ++g)
    for (int64_t o = 0; o < E; ++o) {
      const size_t i = size_t(g * E + o);
      const int k = ww_entry(lower[i], upper[i]);
      if (k < 0) {
        fprintf(stderr,
                "[pumitally] ERROR: set_weight_windows refused: group %lld, element %lld: lower %g, upper %g (a window "
                "needs finite bounds with upper > lower; lower <= 0 means no window)\n",
                (long long)g, (long long)o, lower[i], upper[i]);
        return 1;
      }
      h[size_t(g * E + mesh_.internal_of_orig[size_t(o)])] =
          k ? make_double2(lower[i], upper[i]) : make_double2(kNoWindow, kNoWindow);
    }
  double2 *d = nullptr;
  if (synchronize() || alloc_weight_windows(ngroups, &d)) return 1;
  const cudaError_t e = cudaMemcpy(d, h.data(), h.size() * sizeof(double2), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(d);
    fprintf(stderr, "[pumitally] CUDA error %s uploading the weight windows\n", cudaGetErrorString(e));
    return 1;
  }
  free_weight_windows();
  d_ww_ = d;
  ww_groups_ = ngroups;
  return 0;
}

int Engine::get_weight_windows(double *lower, double *upper, int64_t n) {
  const int64_t E = mesh_.ntets, want = int64_t(ww_groups_) * E;
  if (n != want || (n > 0 && (!lower || !upper))) {
    fprintf(stderr, "[pumitally] ERROR: get_weight_windows: n must be ngroups * num_elements (%lld)\n", (long long)want);
    return 1;
  }
  if (n == 0) return 0;
  PTB_CUDA_OK(cudaSetDevice(device_));
  std::vector<double2> h = std::vector<double2>(size_t(n));
  PTB_CUDA_OK(cudaMemcpy(h.data(), d_ww_, h.size() * sizeof(double2), cudaMemcpyDeviceToHost));
  for (int64_t g = 0; g < ww_groups_; ++g)
    for (int64_t i = 0; i < E; ++i) {
      const size_t o = size_t(g * E + mesh_.orig_of_internal[size_t(i)]);
      lower[o] = h[size_t(g * E + i)].x;
      upper[o] = h[size_t(g * E + i)].y;
    }
  return 0;
}

// The statistics of (tally, time_bin, bin b, score) for every element are at base + b * bin_len() + e * stride_ of the
// whole reported tally, which stats_view gives every rank.
int Engine::generate_weight_windows(int32_t tally, int32_t score, int32_t time_bin, double ratio, double max_rel_err) {
  const char *why = !batch_stats_                          ? "batch statistics are off (set_batch_statistics)"
                    : batches_ < 2                         ? "at least two batches must be folded (end_batch)"
                    : (tally != 0 && tally != 1)           ? "tally must be 0 (track length) or 1 (collision)"
                    : (tally == 1 && !collision_)          ? "the collision estimator is off (set_collision_estimator)"
                    : (score < 0 || score >= nscores_)     ? "score must be in [0, nscores)"
                    : (time_bin < 0 || time_bin >= int32_t(nslices())) ? "time_bin must be in [0, max(ntime, 1))"
                    : !(ratio > 1.0 && ratio <= DBL_MAX)   ? "ratio must be finite and > 1"
                    : !(max_rel_err > 0.0)                 ? "max_rel_err must be > 0"
                                                           : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: generate_weight_windows refused: %s\n", why);
    return 1;
  }
  if (synchronize()) return 1;
  const double *mean = nullptr, *m2 = nullptr;
  double *tmp = nullptr;
  double2 *d = nullptr;
  unsigned long long *red = nullptr;
  int rc = stats_view(&mean, &m2, &tmp);
  if (!rc) rc = alloc_weight_windows(nbins_, &d);
  if (!rc && cudaMalloc(reinterpret_cast<void **>(&red), size_t(nbins_) * sizeof(unsigned long long)) != cudaSuccess) {
    fprintf(stderr, "[pumitally] ERROR: generate_weight_windows: %s\n", cudaGetErrorString(cudaGetLastError()));
    rc = 1;
  }
  if (!rc) {
    const size_t base = size_t(tally) * flux_len() + size_t(time_bin) * size_t(nbins_) * bin_len() + size_t(score);
    const double c = 2.0 / (ratio + 1.0);
    cudaError_t e = launch_ww_generate(mean + base, m2 + base, d_volume_, mesh_.ntets, nbins_, int64_t(bin_len()),
                                       stride_, double(batches_), max_rel_err, c, ratio, red, d, compute_);
    if (e == cudaSuccess) e = cudaStreamSynchronize(compute_);
    if (e != cudaSuccess) {
      fprintf(stderr, "[pumitally] CUDA error %s generating the weight windows\n", cudaGetErrorString(e));
      rc = 1;
    }
  }
  cudaFree(red);
  cudaFree(tmp);
  if (rc) {
    cudaFree(d);
    return 1;
  }
  free_weight_windows();
  d_ww_ = d;
  ww_groups_ = nbins_;
  return 0;
}

int Engine::ww_particles_setup(int32_t n, const double *lower, const double *upper, size_t arena,
                               cudaStream_t stream) {
  const char *why = n != n_ ? "n must be num_particles" : !initialized_ ? "called before CopyInitialPosition" : nullptr;
  if (why) fprintf(stderr, "[pumitally] ERROR: weight windows at the particles refused: %s\n", why);
  if (why || (n > 0 && (!lower || !upper))) return 1;
  if (n == 0) return -1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  return ensure_arena(arena) || follow_last_stream(stream);  // reads the particle state the last move wrote
}

cudaError_t Engine::enqueue_ww_particles(int32_t first, int32_t n, const int32_t *groups, double *lower,
                                         double *upper, cudaStream_t stream) {
  return launch_ww_particles(d_state_ + first, n, groups, d_ww_, ww_groups_, mesh_.ntets, lower, upper, stream);
}

int Engine::weight_windows_at_particles(const int32_t *groups, double *lower, double *upper, int32_t n) {
  return staged(
      n, [&](size_t arena) { return ww_particles_setup(n, lower, upper, arena, compute_); },
      [&](int64_t b, int64_t cnt, const int32_t *g, double *lo, double *up) {
        return enqueue_ww_particles(int32_t(b), int32_t(cnt), g, lo, up, compute_);
      },
      stage(groups), stage(lower), stage(upper));
}

int Engine::weight_windows_at_particles_device(const int32_t *d_groups, double *d_lower, double *d_upper, int32_t n,
                                               cudaStream_t stream) {
  if (int rc = ww_particles_setup(n, d_lower, d_upper, 0, stream)) return std::max(rc, 0);
  PTB_CUDA_OK(enqueue_ww_particles(0, n, d_groups, d_lower, d_upper, stream));
  return 0;
}

int Engine::ww_points_setup(const double *xyz, int64_t npts, const double *lower, const double *upper, size_t arena) {
  if (npts < 0) fprintf(stderr, "[pumitally] ERROR: weight windows at points refused: npts must be >= 0\n");
  if (npts < 0 || (npts > 0 && (!xyz || !lower || !upper))) return 1;
  if (npts == 0) return -1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  return ensure_candidates() || ensure_arena(arena);
}

cudaError_t Engine::enqueue_ww_points(const double *xyz, int64_t npts, const int32_t *groups, double *lower,
                                      double *upper, cudaStream_t stream) {
  const LocateParams p = locate_params();
  for (int64_t b = 0; b < npts; b += kPointsPerLaunch)
    if (cudaError_t e = launch_ww_points(p, xyz + 3 * b, std::min(kPointsPerLaunch, npts - b),
                                         groups ? groups + b : nullptr, d_ww_, ww_groups_, mesh_.ntets, lower + b,
                                         upper + b, stream))
      return e;
  return cudaSuccess;
}

int Engine::weight_windows_at_points(const double *xyz, int64_t npts, const int32_t *groups, double *lower,
                                     double *upper) {
  return staged(
      npts, [&](size_t arena) { return ww_points_setup(xyz, npts, lower, upper, arena); },
      [&](int64_t, int64_t cnt, const double *x, const int32_t *g, double *lo, double *up) {
        return enqueue_ww_points(x, cnt, g, lo, up, compute_);
      },
      stage(xyz, 3), stage(groups), stage(lower), stage(upper));
}

// The mesh tables location reads never change after construction, so a point lookup needs no ordering against moves.
int Engine::weight_windows_at_points_device(const double *d_xyz, int64_t npts, const int32_t *d_groups, double *d_lower,
                                            double *d_upper, cudaStream_t stream) {
  if (int rc = ww_points_setup(d_xyz, npts, d_lower, d_upper, 0)) return std::max(rc, 0);
  PTB_CUDA_OK(enqueue_ww_points(d_xyz, npts, d_groups, d_lower, d_upper, stream));
  return 0;
}

int Engine::ww_arrays(VtkArrays &a) {
  const size_t E = size_t(mesh_.ntets), G = size_t(ww_groups_);
  std::vector<double> lo(G * E), hi(G * E);
  if (get_weight_windows(lo.data(), hi.data(), int64_t(G * E))) return 1;
  for (size_t g = 0; g < G; ++g) {
    const std::string suffix = G == 1 ? "" : "_g" + std::to_string(g);
    for (auto &[name, v] : {std::make_pair("ww_lower", &lo), std::make_pair("ww_upper", &hi)}) {
      a.data.emplace_back(v->begin() + g * E, v->begin() + (g + 1) * E);  // (a moved vector keeps its storage)
      a.named.emplace_back(name + suffix, a.data.back().data());
      a.ncomp.push_back(1);
    }
  }
  return 0;
}

// ------------------------------------------------------------------ mesh source

void Engine::free_source() {
  cudaFree(d_src_cdf_);
  cudaFree(d_src_bias_);
  d_src_cdf_ = d_src_bias_ = nullptr;
  src_groups_ = 0;
  src_total_ = src_strength_ = 0.0;
  src_last_ = -1;
  std::vector<double>().swap(src_given_);
}

SourceTable Engine::source_table() const {
  SourceTable S;
  S.cdf = d_src_cdf_;
  S.bias = d_src_bias_;
  S.verts = d_src_verts_;
  S.E = mesh_.ntets;
  S.K = int64_t(src_groups_) * mesh_.ntets;
  S.klast = src_last_;
  S.total = src_total_;
  S.ratio = src_total_ / src_strength_;
  return S;
}

int Engine::set_source(const double *strength, const double *bias, int64_t n, int32_t ngroups, int32_t per_volume) {
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (!strength && ngroups == 0) {
    if (synchronize()) return 1;  // a device sampling call may still read the table
    free_source();
    return 0;
  }
  const int64_t E = mesh_.ntets;
  const char *why = ngroups < 1                 ? "ngroups must be >= 1 (0 with strength == NULL removes the source)"
                    : !strength                 ? "null strength array"
                    : E < 1                     ? "the mesh has no elements"
                    : n != int64_t(ngroups) * E ? "n must be ngroups * num_elements"
                                                : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: set_source refused: %s\n", why);
    return 1;
  }
  std::vector<double> vol(static_cast<size_t>(E)), cdf(static_cast<size_t>(n));
  for (int64_t i = 0; i < E; ++i) vol[size_t(mesh_.orig_of_internal[size_t(i)])] = mesh_.volume[size_t(i)];
  double T = 0.0, Q = 0.0;
  int64_t klast = -1, bad = -1;
  why = source_build(strength, bias, vol.data(), E, ngroups, per_volume != 0, cdf.data(), &T, &Q, &klast, &bad);
  if (why) {
    if (bad >= 0)
      fprintf(stderr, "[pumitally] ERROR: set_source refused: %s (group %lld, element %lld: strength %g, bias %g)\n",
              why, (long long)(bad / E), (long long)(bad % E), strength[bad], bias ? bias[bad] : 1.0);
    else
      fprintf(stderr, "[pumitally] ERROR: set_source refused: %s (T = %g, Q = %g)\n", why, T, Q);
    return 1;
  }
  if (synchronize()) return 1;
  if (!d_src_verts_) {  // each element's four vertices, caller's numbering and local order: 96 B per element
    std::vector<double> v(size_t(12) * size_t(E));
    for (int64_t i = 0; i < E; ++i) {
      double *o = &v[size_t(12) * size_t(mesh_.orig_of_internal[size_t(i)])];
      for (int q = 0; q < 4; ++q)
        for (int a = 0; a < 3; ++a) o[3 * q + a] = mesh_.coords[3 * size_t(mesh_.t2v[4 * size_t(i) + q]) + a];
    }
    double *d = nullptr;
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&d), v.size() * sizeof(double));
    if (e == cudaSuccess) e = cudaMemcpy(d, v.data(), v.size() * sizeof(double), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      cudaFree(d);
      fprintf(stderr, "[pumitally] ERROR: set_source: no device memory for the element vertices (%zu bytes: %s)\n",
              v.size() * sizeof(double), cudaGetErrorString(e));
      return 1;
    }
    d_src_verts_ = d;
  }
  double *d_cdf = nullptr, *d_bias = nullptr;
  const size_t bytes = size_t(n) * sizeof(double);
  cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&d_cdf), bytes);
  if (e == cudaSuccess) e = cudaMemcpy(d_cdf, cdf.data(), bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && bias) e = cudaMalloc(reinterpret_cast<void **>(&d_bias), bytes);
  if (e == cudaSuccess && bias) e = cudaMemcpy(d_bias, bias, bytes, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(d_cdf);
    cudaFree(d_bias);
    fprintf(stderr, "[pumitally] ERROR: set_source: no device memory for the source (%zu bytes: %s)\n",
            (bias ? 2 : 1) * bytes, cudaGetErrorString(e));
    return 1;
  }
  free_source();
  d_src_cdf_ = d_cdf;
  d_src_bias_ = d_bias;
  src_groups_ = ngroups;
  src_total_ = T;
  src_strength_ = Q;
  src_last_ = klast;
  src_given_.assign(strength, strength + n);
  return 0;
}

int Engine::get_source_strength(double *total) {
  if (src_groups_ == 0 || !total) {
    fprintf(stderr, "[pumitally] ERROR: get_source_strength refused: %s\n",
            src_groups_ == 0 ? "no source is set (set_source)" : "null output");
    return 1;
  }
  *total = src_strength_;
  return 0;
}

int Engine::source_setup(int64_t first, int64_t n, bool outputs, int32_t place, size_t arena, cudaStream_t stream) {
  const char *why = src_groups_ == 0                 ? "no source is set (set_source)"
                    : first < 0                      ? "first must be >= 0"
                    : n < 0                          ? "n must be >= 0"
                    : n > INT64_MAX - first          ? "first + n overflows"
                    : (place && n != int64_t(n_))    ? "with place, n must be num_particles"
                                                     : nullptr;
  if (why) {
    fprintf(stderr, "[pumitally] ERROR: sample_source refused: %s\n", why);
    return 1;
  }
  if (n == 0 || !(place || outputs)) return -1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (ensure_arena(arena)) return 1;
  if (place) {  // the initial placement, as set_state_device makes it
    if (ensure_element_maps() || follow_last_stream(stream)) return 1;  // writes the particle state
    initialized_ = true;
    mirror_valid_ = false;
    pos_mirror_valid_ = false;
  }
  return 0;
}

cudaError_t Engine::enqueue_source(uint64_t seed, int64_t first, int64_t b, int64_t n, double *xyz, int32_t *elem,
                                   int32_t *group, double *weight, bool place, cudaStream_t stream) {
  return launch_source_sample(source_table(), seed, uint64_t(first + b), n, xyz, elem, group, weight,
                              place ? d_state_ + b : nullptr, d_internal_of_orig_, stream);
}

int Engine::sample_source(uint64_t seed, int64_t first, int64_t n, double *xyz, int32_t *elem, int32_t *group,
                          double *weight, int32_t place) {
  return staged(
      n, [&](size_t arena) { return source_setup(first, n, xyz || elem || group || weight, place, arena, compute_); },
      [&](int64_t b, int64_t cnt, double *x, int32_t *e, int32_t *g, double *w) {
        return enqueue_source(seed, first, b, cnt, x, e, g, w, place, compute_);
      },
      stage(xyz, 3), stage(elem), stage(group), stage(weight));
}

int Engine::sample_source_device(uint64_t seed, int64_t first, int64_t n, double *d_xyz, int32_t *d_elem,
                                 int32_t *d_group, double *d_weight, int32_t place, cudaStream_t stream) {
  if (int rc = source_setup(first, n, d_xyz || d_elem || d_group || d_weight, place, 0, stream)) return std::max(rc, 0);
  PTB_CUDA_OK(enqueue_source(seed, first, 0, n, d_xyz, d_elem, d_group, d_weight, place, stream));
  return 0;
}

int Engine::source_arrays(VtkArrays &a) {
  const size_t E = size_t(mesh_.ntets), G = size_t(src_groups_);
  for (size_t g = 0; g < G; ++g) {
    a.data.emplace_back(src_given_.begin() + g * E, src_given_.begin() + (g + 1) * E);
    a.named.emplace_back(G == 1 ? std::string("source") : "source_g" + std::to_string(g), a.data.back().data());
    a.ncomp.push_back(1);
  }
  return 0;
}

// ------------------------------------------------------------------ multi-GPU

int Engine::comm_init(int rank, int nranks, const uint8_t id[128]) {
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (nccl_comm_) return 1;
  if (nccl_comm_init_rank(&nccl_comm_, nranks, id, rank)) return 1;
  rank_ = rank;
  nranks_ = nranks;
  // NCCL sets up its NVLink connections lazily inside the first collective: pay that here,
  // on the scratch array, not in the first batch-end exchange
  if (nranks < 1 || size_t(nranks) > kFluxPad) return 1;
  share_ = (reported_len() + size_t(nranks) - 1) / size_t(nranks);
  PTB_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&d_flux_global_), std::max<size_t>(share_ * size_t(nranks), 1) * sizeof(double)));
  // batch statistics from here on live sharded: this rank's share only, and no batch of the single-rank layout is kept
  if (batch_stats_ && alloc_stats(stats_len())) return 1;
  PTB_CUDA_OK(cudaEventCreate(&ev_ar0_));
  PTB_CUDA_OK(cudaEventCreate(&ev_ar1_));
  PTB_CUDA_OK(cudaMemsetAsync(d_scratch_, 0, size_t(mesh_.ntets) * sizeof(double), compute_));
  if (nccl_allreduce_sum_f64(nccl_comm_, d_scratch_, d_flux_global_, size_t(mesh_.ntets), compute_)) return 1;
  // ... and so does every other collective the first time it is used (the first ncclReduceScatter can take
  // most of a second): warm up the reduce-scatter / all-gather pair of reduce_tally_to_owners too.
  // d_flux_ is all zeros here or holds this rank's tally, which the exchange does not modify.
  if (nccl_reduce_scatter_sum_f64(nccl_comm_, d_flux_, d_flux_global_ + size_t(rank_) * share_, share_, compute_)) return 1;
  if (nccl_all_gather_f64(nccl_comm_, d_flux_global_ + size_t(rank_) * share_, d_flux_global_, share_, compute_)) return 1;
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  // Which of the two batch-end exchanges is quicker depends on the array size and on what NCCL picks for it
  // (either can be the quicker by a large factor):
  // time both on this mesh and let exchange_tally() use the quicker one.  The times are summed over the ranks
  // so that every rank takes the same decision.
  double t[2] = {1e30, 1e30};
  for (int rep = 0; rep < 3; ++rep)
    for (int which = 0; which < 2; ++which) {
      PTB_CUDA_OK(cudaEventRecord(ev_ar0_, compute_));
      if (which == 0 ? nccl_allreduce_sum_f64(nccl_comm_, d_flux_, d_flux_global_, reported_len(), compute_)
                     : nccl_reduce_scatter_sum_f64(nccl_comm_, d_flux_, d_flux_global_ + size_t(rank_) * share_, share_, compute_))
        return 1;
      PTB_CUDA_OK(cudaEventRecord(ev_ar1_, compute_));
      PTB_CUDA_OK(cudaStreamSynchronize(compute_));
      float ms = 0.f;
      PTB_CUDA_OK(cudaEventElapsedTime(&ms, ev_ar0_, ev_ar1_));
      t[which] = std::min(t[which], double(ms));
    }
  double *d_t = d_scratch_;  // E >= 2 doubles of scratch: meshes have more than two elements
  if (mesh_.ntets < 4) { exchange_choice_ = 0; return 0; }
  PTB_CUDA_OK(cudaMemcpyAsync(d_t, t, sizeof(t), cudaMemcpyHostToDevice, compute_));
  if (nccl_allreduce_sum_f64(nccl_comm_, d_t, d_t + 2, 2, compute_)) return 1;
  PTB_CUDA_OK(cudaMemcpyAsync(t, d_t + 2, sizeof(t), cudaMemcpyDeviceToHost, compute_));
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  exchange_ms_[0] = t[0] / nranks;
  exchange_ms_[1] = t[1] / nranks;
  exchange_choice_ = t[1] < t[0] ? 1 : 0;
  return 0;
}

// The batch-end exchange this mesh and this machine do quickest (chosen in comm_init)
int Engine::exchange_tally() { return exchange_choice_ == 1 ? reduce_tally_to_owners() : allreduce_tally(); }

// Batch-end exchange: sum the per-rank tallies.  Every rank holds a full-buffer
// picpart (all elements are ghosts of every other rank), so the ghost-layer
// array is the whole flux array.  Out of place: d_flux_ stays this rank's own running tally, the
// sum over ranks lands in d_flux_global_ -- the call may be repeated after every batch.
int Engine::allreduce_tally() {
  if (!nccl_comm_) return nranks_ == 1 ? 0 : 1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  PTB_CUDA_OK(cudaDeviceSynchronize());
  PTB_CUDA_OK(cudaEventRecord(ev_ar0_, compute_));
  if (nccl_allreduce_sum_f64(nccl_comm_, d_flux_, d_flux_global_, reported_len(), compute_)) return 1;
  PTB_CUDA_OK(cudaEventRecord(ev_ar1_, compute_));
  if (exchange_detectors()) return 1;
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, ev_ar0_, ev_ar1_) == cudaSuccess) allreduce_ms_ = ms;
  flux_global_valid_ = true;
  flux_owned_only_ = false;
  eval_valid_ = false;
  return 0;
}

int Engine::reduce_tally_to_owners() {
  if (!nccl_comm_) return nranks_ == 1 ? 0 : 1;
  PTB_CUDA_OK(cudaSetDevice(device_));
  PTB_CUDA_OK(cudaDeviceSynchronize());
  PTB_CUDA_OK(cudaEventRecord(ev_ar0_, compute_));
  if (nccl_reduce_scatter_sum_f64(nccl_comm_, d_flux_, d_flux_global_ + size_t(rank_) * share_, share_, compute_)) return 1;
  PTB_CUDA_OK(cudaEventRecord(ev_ar1_, compute_));
  if (exchange_detectors()) return 1;
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, ev_ar0_, ev_ar1_) == cudaSuccess) allreduce_ms_ = ms;
  flux_global_valid_ = true;
  flux_owned_only_ = true;
  eval_valid_ = false;
  return 0;
}

// Collective: every rank contributes its share, every rank ends up with the whole (summed) array.
int Engine::gather_shares() {
  if (!flux_global_valid_ || !flux_owned_only_) return 0;
  PTB_CUDA_OK(cudaSetDevice(device_));
  if (nccl_all_gather_f64(nccl_comm_, d_flux_global_ + size_t(rank_) * share_, d_flux_global_, share_, compute_)) return 1;
  PTB_CUDA_OK(cudaStreamSynchronize(compute_));
  flux_owned_only_ = false;
  return 0;
}

}  // namespace ptb
