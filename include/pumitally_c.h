/*
 * pumitally_c.h -- C ABI of libpumitally.so (H100 track-length tally engine).
 *
 * Plain pointers and sizes only.  The first five entry points are one-to-one
 * with the reference's public interface, which is what any FFI for this path
 * binds (reference: src/pumitally/PumiTally.h, class pumitally::PumiTally);
 * the C++ facade in include/pumitally/PumiTally.h is a thin wrapper over them.
 * The rest are additive: accessors the reference's tests obtain by reaching
 * into PumiTallyImpl members, device-pointer entry points for callers whose
 * particle data already lives in HBM, and the multi-GPU exchange step.
 *
 * Error convention follows the reference (PumiTallyImpl.cpp:444-458, 558-565):
 * problems are printed to stderr and the call returns; functions that return
 * int give 0 on success and non-zero on failure so FFI callers can also check.
 * There is no CPU fallback: without a CUDA device pumitally_create* fails.
 */
#ifndef PUMITALLY_C_H
#define PUMITALLY_C_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pumitally_engine pumitally_engine;

/* ---- reference interface ------------------------------------------------ */

/* PumiTally::PumiTally(mesh_filename, num_particles, argc, argv)
 * (reference: PumiTally.h:50-51, PumiTallyImpl.cpp:31-52).  mesh_filename: an
 * Omega_h "<name>.osh" directory, a raw mesh file, or "box:nx,ny,nz[,lx,ly,lz]".
 * argc/argv may be NULL.  Returns NULL on failure. */
pumitally_engine *pumitally_create(const char *mesh_filename, int32_t num_particles,
                                   int *argc, char ***argv);

/* PumiTally::CopyInitialPosition(init_particle_positions, size)
 * (reference: PumiTally.h:66-67, PumiTallyImpl.cpp:54-64).  Host pointer,
 * x0,y0,z0,x1,...; size = 3 * num_particles.  Once per engine. */
int pumitally_copy_initial_position(pumitally_engine *e, const double *init_particle_positions,
                                    int32_t size);

/* PumiTally::MoveToNextLocation(origin, destinations, flying, weights, size)
 * (reference: PumiTally.h:87-89, PumiTallyImpl.cpp:66-149).  Host pointers;
 * size = 3 * num_particles; flying[] is overwritten with zeros
 * (PumiTallyImpl.cpp:169-172).  Inputs are fully consumed before return. */
int pumitally_move_to_next_location(pumitally_engine *e, const double *particle_origin,
                                    const double *particle_destinations, int8_t *flying,
                                    const double *weights, int32_t size);

/* PumiTally::WriteTallyResults() (reference: PumiTally.h:95,
 * PumiTallyImpl.cpp:151-157, 382-416): flux/volume -> "fluxresult.vtk". */
int pumitally_write_tally_results(pumitally_engine *e);

/* PumiTally::~PumiTally() (reference: PumiTally.h:103, PumiTally.cpp:16-19). */
void pumitally_destroy(pumitally_engine *e);

/* ---- additive: construction from arrays ---------------------------------- */

/* Same engine, mesh given in memory: coords double[3*nverts], tet2vert
 * int32[4*ntets] (what the reference gets from Omega_h::binary::read,
 * PumiTallyImpl.cpp:562).  device < 0 selects the current CUDA device. */
pumitally_engine *pumitally_create_from_arrays(const double *coords, int64_t nverts,
                                               const int32_t *tet2vert, int64_t ntets,
                                               int32_t num_particles, int32_t device);

/* ---- additive: accessors (reference tests read Impl members instead:
 * test_pumi_tally_impl_methods.cpp:153, 163, 232) ------------------------- */

int64_t pumitally_num_elements(const pumitally_engine *e);
int32_t pumitally_num_particles(const pumitally_engine *e);
/* raw (un-normalised) flux, double[num_elements] (handler->flux); with score bins also
 * n = nbins * num_elements, see pumitally_set_score_bins */
int pumitally_get_flux(pumitally_engine *e, double *out, int64_t n);
/* flux / volume and volume (NormalizeFlux, PumiTallyImpl.cpp:382-409); either may be NULL */
int pumitally_get_normalized_flux(pumitally_engine *e, double *out_flux, double *out_volume,
                                  int64_t n);
/* parent element of every particle, int32[num_particles] (tracer->getElementIds()) */
int pumitally_get_element_ids(pumitally_engine *e, int32_t *out, int64_t n);
/* current particle positions, double[3*num_particles] AoS (ptcls->get<0>()) */
int pumitally_get_positions(pumitally_engine *e, double *out, int64_t n3);
/* face adjacency derived by the engine, int32[4*num_elements], -1 = hull */
int pumitally_get_adjacency(const pumitally_engine *e, int32_t *out, int64_t n4);
/* zero the flux and the statistics (new batch) */
int pumitally_reset_tally(pumitally_engine *e);
/* Per-source-particle normalisation of the NORMALISED flux (pumitally_get_normalized_flux and
 * WriteTallyResults; the raw flux is unaffected).  The reference divides by tet volume only
 * (PumiTallyImpl.cpp:402) although PumiTally.h:93 promises "and total number of particles", and
 * carries an unused total_initial_weight "needed for normalization" (PumiTallyImpl.h:170-171).
 * mode 0: volume only (default = the reference's behaviour); 1: also by num_particles;
 * 2: also by `value` (> 0, e.g. the total source weight of the batch); 3: also by the total weight
 * of the first tracks after CopyInitialPosition / pumitally_reset_tally, summed by the engine. */
int pumitally_set_source_normalization(pumitally_engine *e, int32_t mode, double value);
/* the divisor currently in effect (1.0 for mode 0) */
double pumitally_get_source_normalization(pumitally_engine *e);

typedef struct pumitally_stats {
  uint64_t segments;      /* tally contributions issued in weighted phases (the metric's unit) */
  uint64_t tracks;        /* flying particles in weighted phases */
  uint64_t relocations;   /* tet crossings walked with tallying off (phase 1 + localisation) */
  uint64_t lost;          /* walks stopped by the iteration limit */
  uint64_t moves;         /* MoveToNextLocation calls */
  double kernel_ms;       /* device time of the walk kernels (CUDA events), cumulative */
  double h2d_bytes;       /* bytes uploaded by the host-pointer entry points, cumulative */
  uint64_t plane_fallbacks; /* compact-layout walk: rays coplanar with a mesh edge, finished on the plane records */
} pumitally_stats;
int pumitally_get_stats(pumitally_engine *e, pumitally_stats *out);

/* Per-call output file name for WriteTallyResults (default "fluxresult.vtk"). */
int pumitally_set_output_name(pumitally_engine *e, const char *filename);
/* Options: "variant" (-1 = the engine picks the walk kernel from the mesh size, the default; 0, 8,
 * 16, 24 = the kernels of this library), "block", "chunk" (particles per upload/compute pipeline
 * stage), "seed_grid", "morton", "claim_run", "host_path" (1 = host-pointer moves are staged
 * through pinned per-particle slots by a small worker pool and only the origins that differ from
 * the previous call's destinations travel; 0 = direct copies of all four arrays from the caller's
 * memory; 2 = default: staged, except that for page-locked caller arrays the engine times both and
 * keeps the faster), "host_threads" (workers of that pool, before the first host-pointer call;
 * default: CPU quota / ranks per node - 1; environment: PUMITALLY_HOST_THREADS,
 * PUMITALLY_HOST_PIN=0 keeps them off the GPU's NUMA node), "register_host" (direct path only:
 * 1 = page-lock the caller's pageable buffers with cudaHostRegister the first time they are
 * seen; the caller must then keep them alive; also PUMITALLY_REGISTER_HOST=1), "max_iters"
 * (crossing limit per walk; 0 = number of elements + 16, the default), "l2_fetch", "autotune"
 * (1 = default: while "variant" is automatic the engine times the streaming and the sorted/packed
 * kernel on moves 1-4 of every 64 and keeps the faster one).  Read-only: "launches", "staged",
 * "stage_host_us", "stage_sent_bytes", "scores", "time_bins", "moments", "walk_blocks_per_sm" (blocks
 * per SM of the last persistent walk kernel launched). */
int pumitally_set_option(pumitally_engine *e, const char *name, int64_t value);
int64_t pumitally_get_option(const pumitally_engine *e, const char *name);

/* ---- additive: device-pointer entry points -------------------------------
 * Same semantics as the host versions, but the arrays already live in device
 * memory (AoS positions, int8 flying, double weights).  Work is enqueued on
 * `stream` (a cudaStream_t passed as void*; NULL = the CUDA default stream,
 * which is also what PyTorch's default stream is) and the call returns
 * without synchronising.  d_flying is NOT zeroed. */
int pumitally_copy_initial_position_device(pumitally_engine *e, const double *d_xyz, int32_t size,
                                           void *stream);
int pumitally_move_to_next_location_device(pumitally_engine *e, const double *d_origin,
                                           const double *d_destinations, const int8_t *d_flying,
                                           const double *d_weights, int32_t size, void *stream);
/* Particle slots [first, first+count) <- positions d_xyz[3*count] in elements d_elem[count] (the
 * caller's element numbering), without walking there; and the reverse.  For drivers that place
 * particles themselves, e.g. the spatially partitioned multi-GPU driver
 * (pumiumtally_b200/partition.py), which hands particles from one picpart's engine to the next.
 * The elements are trusted to contain the positions.  Enqueued on `stream`, no synchronisation. */
int pumitally_set_state_device(pumitally_engine *e, const double *d_xyz, const int32_t *d_elem,
                               int32_t first, int32_t count, void *stream);
int pumitally_get_state_device(pumitally_engine *e, double *d_xyz, int32_t *d_elem, int32_t first,
                               int32_t count, void *stream);
/* raw flux in the caller's element numbering into device memory d_out[num_elements] (with score bins
 * and scores: every bin and score, [bin][score][element]) */
int pumitally_get_flux_device(pumitally_engine *e, double *d_out, void *stream);
/* device address of the raw flux array (double[num_elements]); NOTE: in the engine's internal
 * (spatially sorted) element order -- use pumitally_get_flux for the caller's numbering.  With score
 * bins and scores the array is [bin][element][stride], see pumitally_set_scores */
double *pumitally_flux_device_ptr(pumitally_engine *e);
int pumitally_synchronize(pumitally_engine *e);

/* ---- additive: multi-GPU exchange step -----------------------------------
 * One engine per GPU/process.  Every rank holds a picpart of the mesh and a
 * slice of the particles; at batch end the per-rank tallies of shared (ghost)
 * elements are summed with ncclAllReduce over NVLink.  The 128-byte unique id
 * is produced on rank 0 and distributed by the caller (MPI_Bcast in OpenMC,
 * torch.distributed in bench.py). */
int pumitally_nccl_unique_id(uint8_t out_id[128]);
int pumitally_comm_init(pumitally_engine *e, int32_t rank, int32_t nranks, const uint8_t id[128]);
int pumitally_allreduce_tally(pumitally_engine *e);
/* The cheaper batch-end exchange (half the NVLink traffic): ncclReduceScatter -- every rank receives
 * the sum over ranks of its own share of the elements only.  The shares are gathered (ncclAllGather,
 * COLLECTIVE: every rank must make the call) the first time pumitally_get_flux,
 * pumitally_get_normalized_flux, pumitally_get_flux_device or pumitally_write_tally_results needs
 * the whole array, i.e. normally once, at the end of the run. */
int pumitally_reduce_tally_to_owners(pumitally_engine *e);
/* Which of the two is quicker depends on the size of the flux array and on the algorithm NCCL picks for
 * it (either can be the quicker by a large factor), so
 * pumitally_comm_init times both on the engine's own mesh, agrees on the result across the ranks, and
 * this call -- the one a driver should make at batch end -- runs the quicker one.  Read the decision
 * with pumitally_get_option("exchange_choice") (0 all-reduce, 1 reduce-scatter) and the two times with
 * "exchange_allreduce_us" / "exchange_reduce_scatter_us". */
int pumitally_exchange_tally(pumitally_engine *e);

/* ---- additive: score filter (SURVEY section 8 f4) ---------------------------
 * The reference tallies one flux array (PumiTallyImpl.h:142, flux[elem] += length * weight,
 * PumiTallyImpl.cpp:376); an OpenMC tally usually carries a filter -- energy group, particle type,
 * material -- that sends a score to one of several bins.  pumitally_set_score_bins(e, nbins)
 * gives the engine nbins flux arrays (and resets the tally; on several GPUs call it before
 * pumitally_comm_init), and the *_binned moves take one more per-particle array: the bin particle i
 * scores into during this move.  A bin outside [0, nbins) means "no bin matches": the particle
 * flies and is clipped like any other, unscored.  bins == NULL or nbins == 1 is the plain move.
 * With nbins > 1, pumitally_get_flux / pumitally_get_normalized_flux accept n = num_elements (bin 0)
 * or n = nbins * num_elements (every bin, bin-major); pumitally_get_flux_device always writes every
 * bin; WriteTallyResults writes "flux" = the sum over the bins plus "flux_bin<k>" per bin; the
 * batch-end exchange moves all bins.  The walk kernels are the unfiltered ones: a binned move walks
 * the particle range once per bin with the flying flags masked to that bin (particles are independent
 * and a particle that does not fly is not touched), so it costs one extra pass over the particle
 * arrays per bin, not per segment. */
int pumitally_set_score_bins(pumitally_engine *e, int32_t nbins);
int32_t pumitally_get_score_bins(const pumitally_engine *e);
int pumitally_move_to_next_location_binned(pumitally_engine *e, const double *particle_origin,
                                           const double *particle_destinations, int8_t *flying,
                                           const double *weights, const int32_t *bins, int32_t size);
int pumitally_move_to_next_location_device_binned(pumitally_engine *e, const double *d_origin,
                                                  const double *d_destinations, const int8_t *d_flying,
                                                  const double *d_weights, const int32_t *d_bins,
                                                  int32_t size, void *stream);

/* ---- additive: scores (several responses per track, one walk) --------------
 * An OpenMC tally on a mesh filter usually carries several scores (flux, fission, heating, absorption,
 * ...).  The track-length estimate of score x in element e is the sum of l * w * Sigma_x(E) over the
 * segments in e, and within one move a particle keeps its material and energy, so Sigma_x is one number
 * per particle and move: a response.  pumitally_set_scores(e, nscores), 1 <= nscores <= 8, gives every
 * score bin nscores flux arrays (any other value returns non-zero and changes nothing); it resets the
 * tally, combines with pumitally_set_score_bins in either order and is refused after
 * pumitally_comm_init.  Read it back with pumitally_get_scores or the option "scores".
 * The scored moves take responses double[nscores * num_particles], particle-major (r[i*nscores + k],
 * never NULL), and bins int32[num_particles] or NULL with the score filter's meaning.  Each segment of
 * length l of particle i in element e adds l * w[i] * r[i*nscores + k] to score k of the particle's
 * bin, for every k; a bin outside [0, nbins) flies and scores nothing.  Everything else is the plain
 * move: relocation, clipping at the hull, flying[] zeroed by the host version, the same statistics, and
 * parent elements and positions identical to a plain move with the same origin, dest, flying and
 * weights.  A non-finite w * r is treated like a non-finite weight: zero-length flight, counted as
 * lost, nothing tallied.  With nscores = 1 a scored move equals a plain move with weights w * r.
 * One walk serves all scores (the record fetches, relocation and positions are shared; every further
 * score adds one reduction per crossing), where nscores engines would walk nscores times.
 * With nscores > 1 the plain and binned moves (and PumiTally::MoveToNextLocation) print an error,
 * return non-zero and touch nothing, flying[] included.
 * Results are [bin][score][element] in the caller's element numbering: pumitally_get_flux and
 * pumitally_get_normalized_flux accept n = num_elements (bin 0, score 0) or n = nbins * nscores *
 * num_elements (everything); pumitally_get_flux_device writes everything.  Volume and source
 * normalisation apply to every score alike (mode 3 still sums the weights, not the responses);
 * pumitally_reset_tally zeroes every score and the batch-end exchange moves all of them.
 * WriteTallyResults writes score 0 as "flux" / "flux_bin<b>", exactly as without scores, and every
 * score k >= 1 as "score<k>" (sum over the bins) and, with several bins, "score<k>_bin<b>".
 * The internal array behind pumitally_flux_device_ptr is [bin][element][stride] with stride = nscores
 * padded to 1, 2, 4 or 8 (internal element order). */
int pumitally_set_scores(pumitally_engine *e, int32_t nscores);
int32_t pumitally_get_scores(const pumitally_engine *e);
int pumitally_move_to_next_location_scored(pumitally_engine *e, const double *particle_origin,
                                           const double *particle_destinations, int8_t *flying,
                                           const double *weights, const double *responses,
                                           const int32_t *bins, int32_t size);
int pumitally_move_to_next_location_device_scored(pumitally_engine *e, const double *d_origin,
                                                  const double *d_destinations, const int8_t *d_flying,
                                                  const double *d_weights, const double *d_responses,
                                                  const int32_t *d_bins, int32_t size, void *stream);

/* ---- additive: time filter (track-length scores split between time bins) ----
 * Time advances along a flight, so one flight can span several bins of a pulsed-source or time-of-flight
 * tally.  pumitally_set_time_bins(e, edges, nedges) sets the edges T_0 < T_1 < ... < T_n, n = nedges - 1,
 * 1 <= n <= 1024; bin j is [T_j, T_{j+1}).  The edges must be finite and strictly increasing; anything else,
 * or a flux array that cannot be allocated (nelements * nbins * padded nscores * n doubles), returns
 * non-zero and changes nothing.  edges == NULL with nedges == 0 removes the filter.  The call resets the
 * tally, combines with pumitally_set_score_bins and pumitally_set_scores in any order and is refused after
 * pumitally_comm_init.  pumitally_get_time_bins (or the option "time_bins") returns n, 0 without a filter.
 * The timed moves take, besides the scored move's arguments, times double[num_particles] (particle i's
 * time at its origin) and speeds double[num_particles] (mesh length units per time unit), never NULL;
 * responses may be NULL only with one score (every response 1), bins may be NULL (no score filter).  A
 * segment of particle i in element e covers track distance [s_a, s_b], i.e. the times
 * [times[i] + s_a/speeds[i], times[i] + s_b/speeds[i]]; for every time bin j it overlaps it adds
 * w[i] * r[i,k] * speeds[i] * overlap_j (the track length spent in bin j) to score k of bin bins[i] in time
 * bin j.  A track starting exactly on an edge starts in the bin above it; a flight ending exactly on an
 * edge adds nothing to the next bin.  What lies before T_0 or at or after T_n is not tallied: the particle
 * flies, unscored there.  Relocation carries no time.  A non-finite time, or a speed that is not finite and
 * > 0, is treated like a non-finite weight: zero-length flight, counted as lost, nothing tallied.
 * Everything else is the plain move: parent elements, positions, clipping at the hull, flying[] zeroed by
 * the host version, and the statistics (segments are counted once per crossing, not once per piece).
 * While time bins are set the plain, binned and scored moves (and PumiTally::MoveToNextLocation) print an
 * error, return non-zero and touch nothing, flying[] included; a timed move without time bins is refused
 * the same way.
 * Results are [time][bin][score][element] in the caller's element numbering: pumitally_get_flux and
 * pumitally_get_normalized_flux accept n = num_elements (time bin 0, bin 0, score 0) or n = ntime * nbins
 * * nscores * num_elements; pumitally_get_flux_device writes everything.  Volume and source normalisation
 * are unchanged (nothing is divided by the bin width); pumitally_reset_tally and the batch-end exchange
 * cover every time bin.  WriteTallyResults writes every array it writes without time bins as the sum over
 * the time bins, under the same name, and for every time bin j the same arrays with "_t<j>" after the
 * score name: "flux_t<j>", "flux_t<j>_bin<b>", "score<k>_t<j>", "score<k>_t<j>_bin<b>".
 * The internal array behind pumitally_flux_device_ptr is [time][bin][element][stride]. */
int pumitally_set_time_bins(pumitally_engine *e, const double *edges, int32_t nedges);
int32_t pumitally_get_time_bins(const pumitally_engine *e);
int pumitally_move_to_next_location_timed(pumitally_engine *e, const double *particle_origin,
                                          const double *particle_destinations, int8_t *flying,
                                          const double *weights, const double *times, const double *speeds,
                                          const double *responses, const int32_t *bins, int32_t size);
int pumitally_move_to_next_location_device_timed(pumitally_engine *e, const double *d_origin,
                                                 const double *d_destinations, const int8_t *d_flying,
                                                 const double *d_weights, const double *d_times,
                                                 const double *d_speeds, const double *d_responses,
                                                 const int32_t *d_bins, int32_t size, void *stream);

/* ---- additive: linear flux moments (first spatial moments of every track-length score) ----
 * pumitally_set_moments(e, order): order 1 makes every move also tally, per element e, score, bin and
 * time bin, the first moment of the track-length estimate about the element's centroid c_e: a segment of
 * length l with midpoint x_mid adds w * r * l * (x_mid - c_e), an unbiased estimate of the integral of
 * (x - c_e) * phi over the element.  Order 0 (the default) stops it; any other order, or a flux array that
 * cannot be allocated (4 times the array without moments), returns non-zero and changes nothing.  The call
 * resets the tally, combines with pumitally_set_score_bins, pumitally_set_scores and
 * pumitally_set_time_bins in any order and is refused after pumitally_comm_init.
 * pumitally_get_moments (or the read-only option "moments") returns the order.
 * Every move tallies moments while they are set: the plain, binned, scored and timed moves, host and device,
 * and PumiTally::MoveToNextLocation (the plain and binned moves as one score with every response 1; the
 * rules that refuse a move with several scores or with time bins are unchanged).  Apart from the moments a
 * move does exactly what it does without them: parent elements, positions, clipping, flying[] and the
 * statistics are the same, and so is the flux (pumitally_get_flux, pumitally_get_normalized_flux,
 * pumitally_get_flux_device and the VTK arrays return what they return without moments, up to the order of
 * the reductions).
 * pumitally_get_flux_moments(e, out, n) writes the raw first moments m1; pumitally_get_flux_gradient(e,
 * out, n) writes g = M_e^-1 m1, M_e = integral over the element of (x - c_e)(x - c_e)^T, divided by the
 * source-normalisation divisor of pumitally_get_normalized_flux: normalized_flux + g . (x - c_e) is then
 * the L2 projection of the flux onto linear functions on the element (exact for a flux linear in it).
 * Both are [time][bin][score][element][3] in the caller's element numbering, n = 3 * num_elements (time
 * bin 0, bin 0, score 0) or 3 * ntime * nbins * nscores * num_elements; both follow the batch-end exchange
 * as pumitally_get_flux does, and both return non-zero without moments.  WriteTallyResults writes, after
 * every array it writes without moments, "<name>_grad": the normalised gradient, a 3-component cell array
 * (the gradient of a sum over bins or time bins is the sum of the gradients).
 * Behind pumitally_flux_device_ptr an element's record is [m0 of the S scores][Rx][Ry][Rz], S slots each
 * (S = nscores padded to 1, 2, 4 or 8; stride 4 S), [time][bin][element][4 S] overall; R is the first
 * moment about the mesh centre C (the middle of the bounding box), m1 = R - (c_e - C) * m0. */
int pumitally_set_moments(pumitally_engine *e, int32_t order);
int32_t pumitally_get_moments(const pumitally_engine *e);
int pumitally_get_flux_moments(pumitally_engine *e, double *out, int64_t n);
int pumitally_get_flux_gradient(pumitally_engine *e, double *out, int64_t n);

/* ---- additive: point queries (locate points in the mesh, evaluate the results there) ----
 * For consumers whose points are not the tally's elements (a thermal or CFD solver's quadrature points or nodes, a
 * collision estimator, a mesh source or weight-window lookup).  Points are npts AoS coordinates (x, y, z), caller's
 * frame; npts may exceed 2^31.  A query may be made at any time after construction (before CopyInitialPosition too)
 * and changes nothing: particle positions and elements, the tally, the statistics and the kernel auto-tuner are the
 * same before and after it.
 * pumitally_locate_points writes the element (caller's numbering) containing each point to out_elem[npts], -1 for a
 * point outside the mesh or with a non-finite coordinate.  This holds on convex and non-convex meshes (notches,
 * voids).  A point on a face, edge or vertex shared by several elements gets one of them.  A point within 1e-10 times
 * the mesh extent (the longest edge of its bounding box) of the hull may get a hull element or -1.
 * pumitally_locate_points_device does the same on device arrays, enqueued on `stream` (no synchronisation).
 * Host-pointer calls work through device buffers of the option "chunk" points, whatever npts is.
 * pumitally_evaluate_points writes the normalised result of every time bin, score bin and score at each point to
 * out, [time][bin][score][point]: n = npts (time bin 0, bin 0, score 0) or ntime * nbins * nscores * npts, anything
 * else returns non-zero.  The value is pumitally_get_normalized_flux's for the containing element e, plus, with
 * moments, g_e . (x - c_e) (g_e as pumitally_get_flux_gradient returns it, c_e the average of e's four vertices);
 * NaN outside the mesh.  It follows the batch-end exchange and the source normalisation as
 * pumitally_get_normalized_flux does (after pumitally_reduce_tally_to_owners it gathers the shares: collective) and
 * fails where it fails.  out_elem[npts] receives the elements as pumitally_locate_points does, or is NULL. */
int pumitally_locate_points(pumitally_engine *e, const double *xyz, int64_t npts, int32_t *out_elem);
int pumitally_locate_points_device(pumitally_engine *e, const double *d_xyz, int64_t npts, int32_t *d_elem,
                                   void *stream);
int pumitally_evaluate_points(pumitally_engine *e, const double *xyz, int64_t npts, double *out, int64_t n,
                              int32_t *out_elem);

/* ---- additive: collision estimator (events scored at collision sites) ----
 * Some scores can only be made at a collision (an analog absorption count, the energy a collision deposits) and only the
 * caller knows what happened there; OpenMC's combined k-eff also wants a collision estimate next to the track-length
 * one.  pumitally_set_collision_estimator(e, 1) adds a collision tally with the configuration of the track-length tally
 * (score bins, scores, time bins, moment order) in arrays of its own, so the same scores are estimated both ways; 0
 * (the default) removes it.  Any other value, or a flux array that cannot be allocated (twice the track-length one),
 * returns non-zero and changes nothing.  The call resets the tally, combines with the other pumitally_set_* calls in any
 * order and is refused after pumitally_comm_init.  pumitally_get_collision_estimator (or the read-only option
 * "collision_estimator") returns 1 or 0.  With it off nothing differs from an engine without it.
 * Event i in element e, score bin b = bins[i] and time bin j adds weights[i] * responses[i * nscores + k] to score k of
 * (j, b, e); with moments it also adds that amount times (x_i - C), C the mesh centre, to the first-moment slots, as a
 * move does for a segment's midpoint.  What weights carry is the caller's choice: w / Sigma_t for a collision
 * estimate, w with 0/1 responses for an analog count.
 * pumitally_tally_collisions: nevents events at AoS points xyz[3 * nevents], each located as pumitally_locate_points
 * locates it; host calls work through device buffers of the option "chunk" events.  The _device variant takes device
 * arrays and is enqueued on `stream`.
 * pumitally_tally_collisions_at_particles: an event for every particle i with collided[i] != 0, at its stored position,
 * in its parent element (no location step); n must be num_particles and collided is not zeroed.  Flag only flights that
 * ended at their destination: a flight clipped at the hull stored the hull point.  The _device variant is enqueued on
 * `stream` behind the last move, as a move on another stream is.
 * responses may be NULL only with one score (every response 1); bins may be NULL (every event in bin 0); times are
 * required while time bins are set and ignored otherwise.  A time on an edge belongs to the bin above it.  Not tallied:
 * a bin outside [0, nbins), a time before T_0 or at or after T_n, a located event outside the mesh (counted as outside),
 * and an event with a non-finite coordinate, weight * response or time (counted as rejected; this takes precedence).
 * The read-only options "collisions", "collisions_outside" and "collisions_rejected" count the events tallied, outside
 * and rejected since the last pumitally_reset_tally.  Refused (non-zero, nothing changes): the estimator is off,
 * responses NULL with several scores, times NULL while time bins are set, nevents < 0, n != num_particles.  nevents == 0
 * succeeds and does nothing.
 * A collision call changes no particle, flying flag, track-length result, statistic or kernel choice; like a move it
 * ends the validity of the last batch-end exchange.  Host calls have consumed their inputs when they return.
 * pumitally_get_collision_results(e, kind, out, n): kind 0 raw, 1 normalised, 2 first moments m1, 3 gradient -- what
 * pumitally_get_flux, _get_normalized_flux, _get_flux_moments and _get_flux_gradient return for the track-length tally,
 * with the same n, layout, caller's numbering, volume, source normalisation and batch-end exchange (collective after
 * pumitally_reduce_tally_to_owners).  Kinds 2 and 3 without moments, and any call with the estimator off, return
 * non-zero.  pumitally_reset_tally zeroes the collision tally; both batch-end exchanges sum it with the track-length
 * tally in the same collective.  WriteTallyResults writes, after the track-length arrays, every one of their names
 * prefixed "collision_" ("collision_flux", "collision_flux_bin<b>", "collision_score<k>_t<j>", "collision_flux_grad",
 * ...).  Behind pumitally_flux_device_ptr the collision tally directly follows the track-length one, same layout. */
int pumitally_set_collision_estimator(pumitally_engine *e, int32_t on);
int32_t pumitally_get_collision_estimator(const pumitally_engine *e);
int pumitally_tally_collisions(pumitally_engine *e, const double *xyz, int64_t nevents, const double *weights,
                               const double *responses, const int32_t *bins, const double *times);
int pumitally_tally_collisions_device(pumitally_engine *e, const double *d_xyz, int64_t nevents,
                                      const double *d_weights, const double *d_responses, const int32_t *d_bins,
                                      const double *d_times, void *stream);
int pumitally_tally_collisions_at_particles(pumitally_engine *e, const int8_t *collided, const double *weights,
                                            const double *responses, const int32_t *bins, const double *times,
                                            int32_t n);
int pumitally_tally_collisions_at_particles_device(pumitally_engine *e, const int8_t *d_collided,
                                                   const double *d_weights, const double *d_responses,
                                                   const int32_t *d_bins, const double *d_times, int32_t n,
                                                   void *stream);
int pumitally_get_collision_results(pumitally_engine *e, int32_t kind, double *out, int64_t n);

/* ---- additive: point detectors (next-event flux estimates at fixed points; MCNP's F5 tally) ----
 * pumitally_set_point_detectors(e, xyz, ndet, r0) sets D = ndet detectors, 1 <= D <= 256, at the AoS positions
 * xyz[3D], each located at set time as pumitally_locate_points locates it, with exclusion radii r0[D] (finite, >= 0;
 * required).  (NULL, 0, NULL) removes them.  Refused, changing nothing: a position outside the mesh or non-finite, a bad
 * r0, D out of range.  The call resets the tally, discards the folded batches, combines with the other pumitally_set_*
 * calls in any order and is refused after pumitally_comm_init.  pumitally_get_point_detectors and the read-only option
 * "point_detectors" return D.
 * pumitally_set_detector_cross_sections(e, sigma_t, n): the total cross sections Sigma_t[bin][element] in the caller's
 * numbering, n == nbins * num_elements, finite and >= 0 (or nothing changes); the score bin is the energy group.  The
 * call resets nothing and may come at any time; a later pumitally_set_score_bins that changes nbins drops the table.
 * Detector calls are refused while there is no table.
 * Scoring: event i (position x, element, weight w, responses r[k], score bin b, with time bins a time t and a speed v)
 * and detector d at x_d form one ray.  R = |x_d - x|; p = pdf[i * D + d], the angular density toward the detector per
 * steradian (pdf NULL: isotropic, 1 / (4 pi)).  If R >= r0_d and R > 0 the ray is traced through the mesh and scores
 * s_k = w r[k] p exp(-tau) / R^2, tau the sum over the tets it crosses of Sigma_t[b][tet] times the length inside.  If
 * R < r0_d nothing is traced and s_k = w r[k] p 3 g(Sigma_t[b][e_i] r0_d) / r0_d^2, g(x) = (1 - exp(-x)) / x (1 at 0):
 * the mean of exp(-Sigma r) / r^2 over the ball.  The arrival time t + R / v goes into the time bin that holds it (an
 * edge belongs to the bin above).  Results are laid out [time][bin][score][detector].
 * Ray outcomes: traced (the walk reaches the tet that contains the detector); shadowed (the ray leaves the mesh through
 * the hull first and scores 0: outside the mesh counts as a void of zero importance, which is exact for rays that stay
 * inside the mesh; with the detector void off, re-entry across a concave part of the hull is NOT followed: see
 * pumitally_set_detector_void below for the mode that follows it); lost (stopped by the option "max_iters"; scores 0).
 * Event outcomes, checked in this order and shared by all the event's rays: rejected (a non-finite coordinate, weight *
 * response, time or pdf value, a negative pdf value, a speed not > 0 with time bins, or R == 0 at a detector with
 * r0_d == 0); outside (a located event outside the mesh).  Then per ray, skipped (a bin outside [0, nbins) or an
 * arrival time outside [T_0, T_n): not traced, not counted).  With a pdf every ray reads the event's D values, and with
 * a detector of r0 == 0 every ray compares the event with the D positions.  A multigroup scattering matrix, whose outgoing group depends on the direction, is handled by the
 * caller passing one event per outgoing group g' with bin g' and pdf p(g -> g', mu_d).
 * pumitally_tally_detectors: nevents events at AoS points xyz[3 * nevents], each located as pumitally_locate_points
 * locates it; host calls work through device buffers of the option "chunk" events.  The _device variant takes device
 * arrays and is enqueued on `stream`.  pumitally_tally_detectors_at_particles: an event for every particle i with
 * flagged[i] != 0, at its stored position in its parent element (n must be num_particles); the _device variant is
 * enqueued behind the last move.  pdf may be NULL; responses may be NULL only with one score; bins may be NULL (bin 0);
 * times and speeds are required while time bins are set and ignored otherwise.
 * pumitally_get_detector_results(e, kind, out, n), n == ntime * nbins * nscores * D: kind 0 the open tally divided by
 * the per-source divisor (the sum over ranks after a batch-end exchange), 1 the batch mean, 2 its standard error, 3 its
 * relative error (kinds 1-3 need batch statistics, kinds 2-3 two batches).  end_batch folds the detector tally (summed
 * over the ranks) on every rank.
 * Read-only counters since the last pumitally_reset_tally: "detector_rays" (traced), "detector_rays_shadowed",
 * "detector_rays_lost", "detector_inside_r0" (rays inside an exclusion radius), "detector_crossings" (interior faces
 * the traced, shadowed and lost rays crossed), "detector_events_outside" (once per event) and
 * "detector_events_rejected" (once per event).  The four ray counters add up to D times the events neither rejected
 * nor outside, less the skipped rays.
 * A detector call changes no particle, flying flag, track-length or collision result, element statistic or kernel
 * choice; like a collision call it opens the batch a checkpoint then holds.  Checkpoints hold the open detector tally
 * and counters, and its batch mean and M2 (merged by Chan's update); the fingerprint holds D, the positions and r0 bit
 * for bit and the CRC-32 of the cross-section table as uploaded, so a file of other detectors or another table is
 * refused with a message that names them.  A file with detectors is written as format version 3; every other file
 * keeps its version and bytes. */
int pumitally_set_point_detectors(pumitally_engine *e, const double *xyz, int32_t ndet, const double *r0);
int32_t pumitally_get_point_detectors(const pumitally_engine *e);

/* ---- additive: the detector void (point-detector rays through the space outside the mesh) ----
 * pumitally_set_detector_void(e, on), on 0 or 1 (default 0), treats the space outside the mesh as a void (Sigma_t = 0)
 * that the detector rays cross.  pumitally_get_detector_void and the read-only option "detector_void" return the mode.
 * The call may come before or after pumitally_set_point_detectors and is refused after pumitally_comm_init.  Setting the
 * mode the engine has changes nothing; switching resets the tally and discards the folded batches.  Switching off while
 * a detector lies outside the mesh is refused and changes nothing.  Anything but 0 or 1 is refused.
 * With the mode on:
 * - tau is the sum over the tets of Sigma_t[b][tet] times the length of the segment event -> detector inside the tet,
 *   over the whole segment; its parts outside the mesh add 0.  A ray that leaves through the hull is followed to where
 *   it enters the mesh again (across a notch, a gap or a cavity), so no ray is shadowed.
 * - Detector positions may be any finite point: inside the mesh, in a notch or cavity, or outside the bounding box.
 *   They are still located, so a detector inside keeps its element.
 * - A located event outside the mesh (pumitally_tally_detectors) is traced from where it is and is not counted as
 *   outside ("detector_events_outside" stays 0).  Inside r0 such an event scores the ball
 *   formula with Sigma = 0: s_k = w r[k] p 3 / r0_d^2.
 * - Ray outcomes are traced, lost and inside r0; the four ray counters add up to D times the events not rejected, less
 *   the skipped rays.  Every entry into the mesh counts as one iteration against "max_iters", so every ray is bounded.
 * - The read-only counter "detector_hull_entries" counts the rays' entries into the mesh through the hull: the first
 *   entry of an outside event's ray and every re-entry after a hull exit (0 with the mode off; pumitally_reset_tally
 *   zeroes it).  On a convex hull a ray that has left the mesh cannot come back, so only outside events enter.
 * The entry search runs over lists of hull tets per seed-grid cell, built and uploaded at the mode's first detector
 * call ("detector_hull_candidates" returns their length).  With the mode off every result, counter, refusal and
 * checkpoint byte is what it was without the call.  A checkpoint of an engine with detectors and the mode on is written
 * as format version 4 (version 3's header, and the hull-entry counter with the others); the fingerprint holds the mode
 * while detectors are set, and a load or merge across the two settings is refused with a message that names the
 * detector void. */
int pumitally_set_detector_void(pumitally_engine *e, int32_t on);
int32_t pumitally_get_detector_void(const pumitally_engine *e);
int pumitally_set_detector_cross_sections(pumitally_engine *e, const double *sigma_t, int64_t n);
int pumitally_tally_detectors(pumitally_engine *e, const double *xyz, int64_t nevents, const double *weights,
                              const double *pdf, const double *responses, const int32_t *bins, const double *times,
                              const double *speeds);
int pumitally_tally_detectors_device(pumitally_engine *e, const double *d_xyz, int64_t nevents, const double *d_weights,
                                     const double *d_pdf, const double *d_responses, const int32_t *d_bins,
                                     const double *d_times, const double *d_speeds, void *stream);
int pumitally_tally_detectors_at_particles(pumitally_engine *e, const int8_t *flagged, const double *weights,
                                           const double *pdf, const double *responses, const int32_t *bins,
                                           const double *times, const double *speeds, int32_t n);
int pumitally_tally_detectors_at_particles_device(pumitally_engine *e, const int8_t *d_flagged, const double *d_weights,
                                                  const double *d_pdf, const double *d_responses, const int32_t *d_bins,
                                                  const double *d_times, const double *d_speeds, int32_t n,
                                                  void *stream);
int pumitally_get_detector_results(pumitally_engine *e, int32_t kind, double *out, int64_t n);

/* ---- additive: face currents (the weight crossing every element face, and the leakage through the hull) ----
 * pumitally_set_face_currents(e, 1) makes every move -- plain, binned, scored and timed, host and device pointers --
 * also tally, for each face a track crosses in the tally phase of a move, the particle's weight (weights[i], no
 * response) as the outgoing partial current of the face of the element it leaves, which is the incoming partial
 * current of the same face of the neighbour.  A flight that leaves through the hull counts as outgoing through that
 * hull face (leakage); nothing enters through the hull.  A relocation, the end of a flight, a face the iteration limit
 * stopped the walk at and a bad track add nothing.  Currents are kept per score bin (particles whose bin is outside
 * [0, nbins) add nothing) and per time bin (the bin that holds the crossing time; a crossing exactly on an edge belongs
 * to the bin below), not per score.  0 (the default) stops them; any other value is refused.  The call resets the tally
 * and discards the folded batches; refused after pumitally_comm_init.  Currents change no other result.
 *
 * pumitally_get_face_current_results(e, direction, kind, out, n): direction 0 outgoing, 1 incoming; kind 0 the open
 * tally divided by the per-source divisor of the source normalisation (not by an area or volume), 1 the batch mean,
 * 2 its standard error, 3 its relative error (kinds 1-3 need batch statistics, 2-3 two batches).  n = ntime * nbins *
 * E * 4, [time][bin][element][face] in the caller's numbering, face f opposite local vertex f of the element (the
 * convention of pumitally_get_adjacency).  pumitally_get_leakage(e, kind, out, n): the outgoing current summed over all
 * hull faces, summed on the device in a fixed order, kinds as above, n = ntime * nbins, [time][bin].  A wrong n or
 * kind is refused and changes nothing.  Both are collective after pumitally_reduce_tally_to_owners, as pumitally_get_flux.
 * Checkpoints carry the currents; a checkpoint saved with the other setting is refused. */
int pumitally_set_face_currents(pumitally_engine *e, int32_t on);
int32_t pumitally_get_face_currents(const pumitally_engine *e);
int pumitally_get_face_current_results(pumitally_engine *e, int32_t direction, int32_t kind, double *out, int64_t n);
int pumitally_get_leakage(pumitally_engine *e, int32_t kind, double *out, int64_t n);

/* ---- additive: cosine bins of the face currents ----
 * pumitally_set_current_cosine_bins(e, edges, nedges) sets edges mu_0 < mu_1 < ... < mu_C in [0, 1], C = nedges - 1
 * between 1 and 64, finite and strictly increasing; (NULL, 0) removes them; anything else is refused and changes
 * nothing.  Each crossing of the face currents then also goes to the bin of its cosine mu = min(bden * (1 / |u|), 1):
 * bden is n . u of the face the walk leaves through (n the stored unit normal, u = destination - origin of the flight)
 * and 1 / |u| is formed once per flight.  mu lies in (0, 1], measured against the face normal that points the way the
 * particle travels, and the same mu goes to the neighbour's incoming slot or the hull's outgoing one.  Against a face
 * with a fixed normal (OpenMC's MuSurfaceFilter), an outgoing partial current holds the crossings at +mu and an
 * incoming one those at -mu.  Bin k holds mu_k <= mu < mu_k+1 and mu == mu_C goes to the last bin; a crossing with mu
 * outside [mu_0, mu_C] adds nothing to any current, leakage included.  While bins are set and face currents are on:
 *   pumitally_get_face_current_results takes n = ntime * nbins * C * E * 4, [time][bin][cosine][element][face];
 *   pumitally_get_leakage takes n = ntime * nbins * C, [time][bin][cosine];
 *   pumitally_get_region_current_results takes n = ntime * nbins * C * P, [time][bin][cosine][pair];
 * with the same kinds.  A net current per cosine bin is the difference of the two partials in that bin, and summed over
 * the bins of edges that cover [0, 1] every result is the result without bins.  The call may come before or after
 * pumitally_set_face_currents; nothing changes while face currents are off.  It resets the tally and discards the
 * folded batches; refused after pumitally_comm_init.  pumitally_get_current_cosine_bins (or the option
 * "current_cosine_bins") returns C, 0 without bins.  A checkpoint saved with other cosine bins is refused. */
int pumitally_set_current_cosine_bins(pumitally_engine *e, const double *edges, int32_t nedges);
int32_t pumitally_get_current_cosine_bins(const pumitally_engine *e);

/* ---- additive: batch statistics (mean, standard and relative errors over batches, on the device) ----
 * A Monte Carlo tally is reported as mean +- standard error over batches.  pumitally_set_batch_statistics(e, 1) keeps,
 * for every reported result (the track-length tally and, with the estimator on, the collision tally: every time bin,
 * score bin and score), a running mean and sum of squared deviations M2 on the device; 0 (the default) frees them.  Any
 * other value, or statistics that cannot be allocated (2 doubles per double of the reported tallies), returns non-zero
 * and changes nothing.  The call resets the tally, combines with the other pumitally_set_* calls in any order and is
 * refused after pumitally_comm_init.  Calling it with 1 again discards the folded batches, and so does, while it is on,
 * every other pumitally_set_* call that changes the configuration (the statistics take the new layout); so does
 * pumitally_comm_init.  Read-only options: "batch_statistics" (0/1) and "batches" (batches folded).
 * pumitally_end_batch(e) closes the open batch.  Its divisor d_b is, on one rank, exactly what
 * pumitally_get_normalized_flux would divide by at that moment; on several ranks modes 1 and 3 use the sum of the ranks'
 * divisors (the whole batch's source), mode 2 uses `value` and mode 0 uses 1.  A d_b that is not > 0 refuses the call
 * and changes nothing.  Every reported double x of the batch tally is folded as x / d_b into its mean and M2 by Welford's
 * update (which, unlike sum and sum of squares, does not cancel when the relative error is small); then the call does
 * exactly what pumitally_reset_tally does, and synchronises as it does.  Refused while statistics are off.  With several
 * ranks the call is collective: the batch tally is reduce-scattered to the element owners (as by
 * pumitally_reduce_tally_to_owners) and every rank folds and keeps only its share.
 * pumitally_get_batch_results(e, tally, kind, out, n): tally 0 track length, 1 collision; kind 0 the mean divided by
 * volume (the per-source normalised result averaged over the batches), 1 its standard error sqrt(M2 / (B (B - 1))) /
 * volume, 2 the relative error (1) / |(0)|, 0 where the mean is 0, 3 the gradient of the mean (what
 * pumitally_get_flux_gradient computes, applied to the batch means; moments only).  n, the layout
 * [time][bin][score][element] (times 3 for kind 3) and the caller's numbering are those of
 * pumitally_get_normalized_flux / pumitally_get_flux_gradient.  Refused: no batch folded, fewer than two for kinds 1 and
 * 2, kind 3 without moments, tally 1 without the estimator, a wrong n.  Collective with several ranks (the shares are
 * gathered).  Statistics are of the m0 results only; moments and gradients get no variance (that needs covariances).
 * pumitally_get_batch_max_rel_err(e, tally, score, out_max, out_nonzero): for tally triggers, the largest relative error
 * of score `score` over every element, score bin and time bin with a nonzero mean, and how many such results there are,
 * reduced on the device; refused with fewer than two batches.  Collective with several ranks (max and sum over ranks).
 * WriteTallyResults with statistics on and at least one batch folded writes, after every array it writes without them,
 * "<name>_mean" for every scalar array (for a sum over bins or time bins, such as "flux" with bins, the sum of the
 * means) and, with two batches or more, "<name>_rel_err" for every scalar array that is exactly one (time bin, bin,
 * score) result: "flux" / "score<k>" without bins or time bins, otherwise the "_bin<b>" / "_t<j>" arrays.  Sums over bins
 * or time bins get no "_rel_err", their error needs covariances.  Collision arrays carry the same suffixes after their
 * "collision_" names.  The other arrays are unchanged and hold the open batch. */
int pumitally_set_batch_statistics(pumitally_engine *e, int32_t on);
int pumitally_end_batch(pumitally_engine *e);
int pumitally_get_batch_results(pumitally_engine *e, int32_t tally, int32_t kind, double *out, int64_t n);
int pumitally_get_batch_max_rel_err(pumitally_engine *e, int32_t tally, int32_t score, double *out_max,
                                    int64_t *out_nonzero);

/* ---- additive: region tallies (sums over caller-defined groups of elements, with batch statistics) ----
 * A region is a group of elements, such as a material or a CAD part (a Gmsh physical group, an Omega_h class id).
 * pumitally_set_regions(e, region_of_element, n, nregions): region_of_element holds one id per element in the caller's
 * numbering (n == pumitally_num_elements), each in [-1, nregions), -1 for an element in no region, and
 * 1 <= nregions <= n.  Regions may be empty.  region_of_element == NULL with nregions == 0 removes the regions; any
 * other input returns non-zero and changes nothing.  The call resets the tally and discards the folded batches, as
 * every pumitally_set_* call does, and is refused after pumitally_comm_init.  pumitally_get_regions returns nregions, 0
 * without regions.
 * pumitally_get_region_volumes(e, out, n == nregions): V_G, the sum of the region's element volumes.
 * pumitally_get_region_results(e, tally, kind, out, n): tally 0 track length, 1 collision (estimator on); kind 0 the raw
 * sum sum_{e in G} x_e of every result (m0 only: moments are not summed), kind 1 the normalised value sum / V_G / d,
 * d the divisor pumitally_get_normalized_flux uses.  Layout [time][bin][score][region]; n == nregions gives time bin 0,
 * bin 0, score 0, n == ntime * nbins * nscores * nregions everything.  It reads the tally the flux accessors read
 * (after a batch-end exchange the summed one; collective after pumitally_reduce_tally_to_owners, as they are).
 * Sums are formed on the device in a fixed order (ascending internal element id in chunks of 32, then the chunk sums
 * in chunks of 32, and so on), so the same tally gives the same bits; a one-element region gives exactly the element's
 * pumitally_get_flux / pumitally_get_normalized_flux value, and its volume is the element's.  An empty region has
 * volume 0 and sum 0; its kind 1 value and all of its batch results are NaN (0 / 0).
 * Batch statistics: while pumitally_set_batch_statistics is on and regions are set, pumitally_end_batch also sums the
 * batch's raw tally (both tallies) into regions before it is folded, adds those sums over the ranks (one
 * ncclAllReduce of nregions * results doubles) and folds sum / d_b as it folds every element.  The variance of a
 * region sum needs the covariances of its elements, which per-element statistics cannot give afterwards: this does.
 * pumitally_get_region_batch_results(e, tally, kind, out, n): kind 0 the mean / V_G, 1 the standard error / V_G, 2 the
 * relative error; layout and n as pumitally_get_region_results.  Refused as pumitally_get_batch_results is (kind 3 does
 * not exist here), and without regions.  Not collective: every rank holds the same region statistics. */
int pumitally_set_regions(pumitally_engine *e, const int32_t *region_of_element, int64_t n, int32_t nregions);
int32_t pumitally_get_regions(const pumitally_engine *e);
int pumitally_get_region_volumes(pumitally_engine *e, double *out, int64_t n);
int pumitally_get_region_results(pumitally_engine *e, int32_t tally, int32_t kind, double *out, int64_t n);
int pumitally_get_region_batch_results(pumitally_engine *e, int32_t tally, int32_t kind, double *out, int64_t n);

/* ---- additive: region currents (partial and net currents between adjacent regions and out through the hull) ----
 * pumitally_set_region_currents(e, 1), while regions are set and face currents are on, also reports, per time bin and
 * score bin, the partial current of every ordered pair of adjacent regions (the weight crossing from region A into
 * region B) and its net current.  Region ids are the caller's; -1 (elements in no region) is a region of its own and
 * -2 stands for outside the mesh.  The pairs come from the face-current slots (see pumitally_set_face_currents): an
 * interior face between element e in region A and element n in region B != A adds the weight entering n through it to
 * pair A -> B and the weight entering e to B -> A; a face with A == B belongs to no pair; a hull face of an element in
 * A adds the weight leaving through it to A -> -2.  The pair list holds every pair with at least one face, in
 * ascending (from, to) order as signed integers; it depends on the mesh and the region map only.  The partial current
 * of pair p is the sum of its faces' currents, formed on the device in the order of the region sums (so the same tally
 * gives the same bits); net[p] = partial[p] - partial[B -> A], the second term 0 when that pair does not exist (always
 * for to == -2).  The partials of the pairs into -2 add up to pumitally_get_leakage (up to summation order).
 * The call is refused, changing nothing, without regions, with face currents off, after pumitally_comm_init, when 4 * E
 * exceeds INT32_MAX, or for `on` other than 0 or 1.  Like every pumitally_set_* call it resets the tally and discards
 * the folded batches.  pumitally_set_regions(e, NULL, 0) and pumitally_set_face_currents(e, 0) switch region currents
 * off; pumitally_set_regions with a new map keeps them on with the new map's pairs (or fails, changing nothing).
 * pumitally_get_region_current_pair_count(e): P, 0 while region currents are off.
 * pumitally_get_region_current_pairs(e, from, to, n == P): the pair list.
 * pumitally_get_region_current_areas(e, out, n == P): the summed area of each pair's faces (fp64, summed in the order of
 * the partials), to divide by for a current per area such as a wall loading.
 * pumitally_get_region_current_results(e, which, kind, out, n): which 0 partial, 1 net; kind 0 the open tally divided
 * by the per-source divisor, 1 the batch mean, 2 its standard error, 3 its relative error.  Layout [time][bin][pair],
 * n == ntime * nbins * P.  Kind 0 reads the tally pumitally_get_region_results reads (collective after
 * pumitally_reduce_tally_to_owners); kinds 1-3 are refused as pumitally_get_batch_results refuses them and are not
 * collective.  While batch statistics are on, pumitally_end_batch forms every partial and net current of the batch next
 * to the region sums, before the exchange, and folds them with them: the error of a partial includes the covariances
 * of its faces, and the error of a net current the covariance of its two partials (a flight through a slab scores
 * both).  Checkpoints carry these statistics in their region sections; a checkpoint saved with the other setting is
 * refused. */
int pumitally_set_region_currents(pumitally_engine *e, int32_t on);
int32_t pumitally_get_region_currents(const pumitally_engine *e);
int64_t pumitally_get_region_current_pair_count(const pumitally_engine *e);
int pumitally_get_region_current_pairs(pumitally_engine *e, int32_t *from, int32_t *to, int64_t n);
int pumitally_get_region_current_areas(pumitally_engine *e, double *out, int64_t n);
int pumitally_get_region_current_results(pumitally_engine *e, int32_t which, int32_t kind, double *out, int64_t n);

/* ---- additive: checkpoints (save the tally state to a file, restart from it, merge independent runs) ----
 * A checkpoint holds the engine's tally state: the open batch (the raw tally, the first-track weight, the collision
 * counters, the pumitally_get_stats counts and the move counters), included only when something was moved, collided
 * or localised since the last reset (right after pumitally_end_batch it is the statistics alone); and, while batch
 * statistics are on, the number of folded batches, this rank's running mean and M2 of every reported double and the
 * region statistics.  It also holds a fingerprint of everything their layout and meaning depend on: the mesh (counts
 * and a hash of coordinates and t2v), the internal element order, score bins, scores, time-bin edges (bit for bit),
 * moment order, collision estimator, batch statistics on/off, the region map, the source-normalisation mode (and its
 * value in mode 2), and rank, number of ranks and rank share.  It holds no particle state, kernel or host-path option,
 * timer or output name: after a load the caller places the particles (CopyInitialPosition, as OpenMC does at every
 * batch start) before the next move.  All three calls return 0 on success; a refusal returns 1, prints the reason and
 * changes nothing in the engine.  None is collective: with several ranks every rank saves, loads or merges its own
 * share under a path the caller makes unique per rank (the region statistics, the same on every rank, are in each).
 * pumitally_save_checkpoint(e, path) synchronises, writes path + ".tmp", flushes, fsyncs and renames it over path: a
 * failed or killed save leaves the previous file at path intact.  It changes nothing in the engine, and the same state
 * always gives the same bytes.
 * pumitally_load_checkpoint(e, path) replaces the tally state with the file's.  It never reconfigures: set up the
 * configuration the file was saved with first (then pumitally_comm_init with several ranks, which discards folded
 * batches), then load.  The header and fingerprint are checked before anything is allocated; every section is
 * checked against its CRC-32 before the engine's buffers are replaced.
 * pumitally_merge_checkpoint(e, path) adds the file's folded batches to the engine's (Chan's parallel update of mean
 * and M2, on the device; element and region statistics): B becomes B_a + B_b.  It needs batch statistics on and the
 * same fingerprint, except the mode-2 normalisation value (the folded values are already per source), and refuses a
 * file that holds an open batch (save it at a batch end).  The engine's open batch, particles and counters are left
 * alone.
 * Device memory: load and merge hold a second copy of what they read until the swap or the merge is done, up to
 * 2 * (statistics doubles) + (tally doubles); when that cannot be allocated they refuse. */
int pumitally_save_checkpoint(pumitally_engine *e, const char *path);
int pumitally_load_checkpoint(pumitally_engine *e, const char *path);
int pumitally_merge_checkpoint(pumitally_engine *e, const char *path);

/* ---- additive: weight windows (MAGIC generation from the batch statistics, lookups on the GPU) ----
 * Deep-penetration and shielding tallies converge only with weight windows, and the usual way to get them is the MAGIC
 * method: run, turn the mesh flux tally into per-element, per-energy-group bounds, run again with those bounds.  The
 * engine holds one window table: ngroups (lower, upper) pairs per element, 16 * ngroups * num_elements bytes of device
 * memory; a call that cannot allocate it is refused.  Windows are not tally state: pumitally_reset_tally,
 * pumitally_end_batch, every pumitally_set_* call, pumitally_comm_init and checkpoint save, load and merge leave them
 * alone, and checkpoints do not hold them (get them and set them back).  A missing window reads (-1, -1).  Refusals
 * print the reason, return non-zero and change nothing.
 * pumitally_set_weight_windows(e, lower, upper, n, ngroups): host arrays [group][element] in the caller's numbering,
 * n == ngroups * num_elements.  An entry with lower <= 0 means no window; any other entry must be finite with
 * upper > lower, or (a NaN, an infinity, upper <= lower) the whole call is refused.  lower == NULL with ngroups == 0
 * removes the windows.  Not collective.  pumitally_get_weight_window_groups returns ngroups (0 without windows);
 * pumitally_get_weight_windows(e, lower, upper, n) returns what set stored, in the same layout (n == ngroups *
 * num_elements; 0 without windows).
 * pumitally_generate_weight_windows(e, tally, score, time_bin, ratio, max_rel_err) replaces the table with the MAGIC
 * windows of one result, the score bins as energy groups (ngroups = nbins).  It needs batch statistics on and at least
 * two folded batches; tally is 0 (track length) or 1 (collision, estimator on), 0 <= score < nscores,
 * 0 <= time_bin < max(ntime, 1), ratio finite and > 1, max_rel_err > 0 (+inf accepts every error).  For group b and
 * element e, phi and r are what pumitally_get_batch_results kinds 0 and 2 return for (time_bin, b, score, e).  The
 * element is eligible when phi is finite and > 0 and r <= max_rel_err; phimax_b is the largest eligible phi of group b.
 * An eligible element gets lower = (phi / phimax_b) * c with c = 2 / (ratio + 1), and upper = lower * ratio, in that
 * order of operations: the window's centre is phi / phimax_b, weight 1 where the flux is largest.  Every other element,
 * and every element of a group without an eligible one, gets (-1, -1).  Collective with several ranks: every rank
 * gathers the whole statistics and computes the same table.
 * pumitally_get_weight_windows_at_particles(e, groups, lower, upper, n): the window of each particle's current parent
 * element, n == num_particles; groups int32[n] is each particle's energy group, NULL for group 0.  A group outside
 * [0, ngroups) or an element without a window gives (-1, -1).  Refused before CopyInitialPosition.  The _device variant
 * takes device arrays and is enqueued on `stream` behind the last move, as pumitally_tally_collisions_at_particles_device.
 * pumitally_get_weight_windows_at_points(e, xyz, npts, groups, lower, upper): the window at each of npts AoS points,
 * located as pumitally_locate_points locates them; a point outside the mesh or with a non-finite coordinate gives
 * (-1, -1).  Host calls work through device buffers of the option "chunk" points; the _device variant is enqueued on
 * `stream`.  No lookup changes a particle, the tally, a statistic, a counter or the kernel auto-tuner.
 * WriteTallyResults with windows set writes, after every other array, "ww_lower" and "ww_upper" (one group) or
 * "ww_lower_g<g>" and "ww_upper_g<g>" for every group g. */
int pumitally_set_weight_windows(pumitally_engine *e, const double *lower, const double *upper, int64_t n,
                                 int32_t ngroups);
int32_t pumitally_get_weight_window_groups(const pumitally_engine *e);
int pumitally_get_weight_windows(pumitally_engine *e, double *lower, double *upper, int64_t n);
int pumitally_generate_weight_windows(pumitally_engine *e, int32_t tally, int32_t score, int32_t time_bin, double ratio,
                                      double max_rel_err);
int pumitally_get_weight_windows_at_particles(pumitally_engine *e, const int32_t *groups, double *lower, double *upper,
                                              int32_t n);
int pumitally_get_weight_windows_at_particles_device(pumitally_engine *e, const int32_t *d_groups, double *d_lower,
                                                     double *d_upper, int32_t n, void *stream);
int pumitally_get_weight_windows_at_points(pumitally_engine *e, const double *xyz, int64_t npts, const int32_t *groups,
                                           double *lower, double *upper);
int pumitally_get_weight_windows_at_points_device(pumitally_engine *e, const double *d_xyz, int64_t npts,
                                                  const int32_t *d_groups, double *d_lower, double *d_upper,
                                                  void *stream);

/* ---- additive: mesh source (per-element, per-group strengths sampled on the GPU, with source biasing) ----
 * A volumetric source on the tally mesh, e.g. the decay photons of a shutdown-dose-rate run: one strength per element
 * and group.  A sample picks an entry in proportion to its (biased) strength and then a uniform point inside the
 * element.  The engine holds one source table: 8 bytes per entry (16 with bias) and, from the first set on, the
 * elements' vertices (96 bytes per element).  The source is not tally state: pumitally_reset_tally, pumitally_end_batch,
 * every other pumitally_set_* call, pumitally_comm_init and checkpoints leave it alone, and checkpoints do not hold it.
 * Refusals print the reason, return non-zero and change nothing.
 * pumitally_set_source(e, strength, bias, n, ngroups, per_volume): host arrays [group][element] in the caller's
 * numbering, n == ngroups * num_elements; bias may be NULL.  Entry k = g * E + e gets p[k] = (q[k] * V[e] if per_volume
 * else q[k]) * (b[k] if bias else 1), each product rounded separately, V the element's volume; the CDF is the
 * sequential sum C[k] = C[k-1] + p[k], T = C[K-1], and Q the same sum of the unbiased q V (or q).  Refused: a strength
 * or bias that is negative or not finite, a bias of 0 where the strength is > 0, T or Q 0 or not finite, ngroups < 1
 * or a wrong n.  strength == NULL with ngroups == 0 removes the source.  pumitally_get_source_groups returns ngroups
 * (0 without a source); pumitally_get_source_strength returns Q, by which the caller normalises.
 * pumitally_sample_source(e, seed, first, n, xyz, elem, group, weight, place): samples i = first .. first + n - 1.
 * Sample i takes four uniforms u_k = ((z_k >> 12) + 0.5) * 2^-52, z_k the SplitMix64 mix of (seed, i, stream k), so it
 * depends on (seed, i) alone.  Its entry k is the first with C[k] > u_0 * T (the last entry with p > 0 if x rounded up
 * to T): group k / E, element k % E.  Its point is the Rocchini-Cignoni fold of (u_1, u_2, u_3) applied to the
 * element's vertices in the caller's local order, every operation rounded separately.  Its weight is 1 without bias and
 * (T / Q) / b[k] with bias (mean 1).  The outputs -- AoS xyz [3n], elem (caller's numbering), group, weight -- may each
 * be NULL.  place != 0 needs n == num_particles: sample j becomes particle j's position and parent element, without a
 * walk, as pumitally_set_state_device stores them; it counts as the initial placement (CopyInitialPosition is refused
 * afterwards).  Without place nothing in the engine changes.  The host call works through device buffers of the option
 * "chunk" samples and synchronises; the _device variant takes device arrays and is enqueued on `stream`, behind the
 * last work on the particle state.
 * WriteTallyResults with a source set writes, after every other array, "source" (one group) or "source_g<g>" for every
 * group g: the strengths as the caller gave them. */
int pumitally_set_source(pumitally_engine *e, const double *strength, const double *bias, int64_t n, int32_t ngroups,
                         int32_t per_volume);
int32_t pumitally_get_source_groups(const pumitally_engine *e);
int pumitally_get_source_strength(pumitally_engine *e, double *total);
int pumitally_sample_source(pumitally_engine *e, uint64_t seed, int64_t first, int64_t n, double *xyz, int32_t *elem,
                            int32_t *group, double *weight, int32_t place);
int pumitally_sample_source_device(pumitally_engine *e, uint64_t seed, int64_t first, int64_t n, double *d_xyz,
                                   int32_t *d_elem, int32_t *d_group, double *d_weight, int32_t place, void *stream);

/* test hook: processing order produced by the last binning pass (ids of flying particles
 * grouped by seed-grid cell); returns the number of entries, copies at most n of them */
int64_t pumitally_debug_order(pumitally_engine *e, int32_t *out, int64_t n);

/* test hook, needs no GPU: one stage pass of the host-pointer path (csrc/host_stage.hpp) over
 * particles [0, n) with `threads` workers.  b_dest/b_w/b_fly are the staging slots (b_dest also the
 * mirror the origins are compared against when compare != 0); out_patches receives 32-byte entries
 * {x, y, z, int32 index, int32 0}.  Returns the number of entries, or -1 if they exceed cap. */
int64_t pumitally_debug_stage(const double *origin, const double *dest, int8_t *flying,
                              const double *weights, double *b_dest, double *b_w, int8_t *b_fly,
                              int64_t n, int32_t compare, int32_t threads, void *out_patches,
                              int64_t cap);

const char *pumitally_version(void);

#ifdef __cplusplus
}
#endif
#endif /* PUMITALLY_C_H */
