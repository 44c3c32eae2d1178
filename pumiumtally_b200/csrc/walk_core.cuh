// Per-tet step of the adjacency walk: decode a packed TetRecord, find the exit
// face of the ray, decide reached / crossed / left-the-hull.
//
// This is the arithmetic the reference delegates to the external pumi-pic
// tracer (call site PumiTallyImpl.cpp:454; contract PumiTallyImpl.h:74-85)
// fused with the reference's own per-iteration functor
// (PumiTallyImpl.cpp:297-316): tally the piece inside the current tet
// (EvaluateFlux :352-380), clip at the hull (ApplyVacuumBC :256-286), advance
// (UpdateCurrentElement :243-254).  prev_xpoint (:322-350) is the register
// `tcur`.
//
// The functions are __host__ __device__ only so that tests/ can compile them
// with g++ and check the logic on a machine without a GPU; the library never
// runs them on the host.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define PTB_HD __host__ __device__ __forceinline__
#if defined(__CUDA_ARCH__)
#define PTB_UNROLL _Pragma("unroll")
#else
#define PTB_UNROLL  // nvcc's host pass hands the pragma to g++, which does not know it
#endif
#else
#define PTB_HD inline
#define PTB_UNROLL
#include <cmath>
#include <cstring>
#endif

#if defined(__CUDA_ARCH__)
#define PTB_LDG(p) __ldg(p)
// RED.E.ADD.F64 (Kokkos::atomic_add, Impl.cpp:376) carrying the same L2 evict_last priority as
// the tet records: with the default priority the (small, extremely hot) flux lines are the first
// victims of the evict_last tet stream and every second reduction misses in L2.
__device__ __forceinline__ void tally_add(double *ptr, double v) {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  asm volatile("red.global.add.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(ptr), "d"(v), "l"(pol) : "memory");
}
#define PTB_TALLY_ADD(ptr, v) tally_add((ptr), (v))
// Experiment (north_star: "warp-aggregated atomicAdd to cut contention"): lanes of the warp that tally
// into the same tet in this step are found with match.any, their contributions are summed with
// shuffles and one lane issues the reduction.  Called by every converged lane; `on` = this lane has
// something to add.  Experiment variants 28, 29; not used by the product kernels.
__device__ __forceinline__ void tally_add_aggregated(double *flux, int32_t e, double v, bool on) {
  const unsigned act = __activemask();
  const int lane = threadIdx.x & 31;
  unsigned peers = __match_any_sync(act, on ? e : -1 - lane);  // lanes with nothing to add match only themselves
  const int leader = __ffs(peers) - 1;
  double sum = 0.0;
  unsigned m = peers;
  while (__any_sync(act, m != 0)) {
    const int src = m ? __ffs(m) - 1 : lane;
    const double x = __shfl_sync(act, v, src);
    if (m) { sum += x; m &= m - 1; }
  }
  if (on && lane == leader) tally_add(flux + e, sum);
}
#else
#define PTB_LDG(p) (*(p))
#define PTB_TALLY_ADD(ptr, v) (*(ptr) += (v))  // test-only host build is single threaded
#endif

namespace ptb {

// low/high 32-bit halves of a double, portable between nvcc device code and g++
PTB_HD uint32_t dlo(double x) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__double2loint(x);
#else
  uint64_t u; memcpy(&u, &x, 8); return (uint32_t)u;
#endif
}
// Tet ids are 30-bit; the all-ones id marks the hull.
constexpr uint32_t kIdMask = 0x3fffffffu;

// byte 0 of four words -> one word (b0 | b1<<8 | b2<<16 | b3<<24)
PTB_HD uint32_t pack_low_bytes(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(__byte_perm(w0, w1, 0x0040), __byte_perm(w2, w3, 0x0040), 0x5410);
#else
  return (w0 & 0xffu) | ((w1 & 0xffu) << 8) | ((w2 & 0xffu) << 16) | ((w3 & 0xffu) << 24);
#endif
}

// Payload of one face of tet `self` (the four doubles a,b,c,d of local face f): the id of the
// neighbour across it (-1 = hull) and `back`, the neighbour's local index of the shared face.
// Stored symmetrically -- bits 0..29 = self XOR neighbour, bits 30..31 = f XOR back -- so the
// payload, and with it the plane, is bit-identical in the two records that share the face.
PTB_HD void face_payload(double a, double b, double c, double d, int32_t self, int f, int32_t &nbr,
                         int32_t &back) {
  const uint32_t pay = pack_low_bytes(dlo(a), dlo(b), dlo(c), dlo(d));
  const uint32_t x = (pay ^ (uint32_t)self) & kIdMask;
  nbr = (int32_t)((x + 1u) & kIdMask) - 1;  // kIdMask -> -1 (hull), everything else unchanged
  back = (int32_t)((pay >> 30) ^ (uint32_t)f);
}

// Running minimum of the exit parameter over the faces scanned so far.  Ray x(t) = o + t*u,
// t in [0,1]; a face is a candidate when the ray leaves through it (n.u > 0).  Numerator and
// denominator depend only on the plane and the ray, never on the tet, so both tets sharing a
// face compute the identical quotient.  The minimum is selected by cross-multiplication
// (num_a*den_b < num_b*den_a, both den > 0): one fp64 division per crossing instead of one per
// face; ties within rounding pick either face, which only reorders a zero-length piece.
constexpr double kParallelTol = 1e-12;

struct ExitScan {
  double bnum = 1.0, bden = 0.0;  // t = +inf
  int32_t nbr = -2, back = -1;
};

PTB_HD void scan_face(ExitScan &s, double nx, double ny, double nz, double c, int32_t nbr,
                      int32_t back, double ox, double oy, double oz, double ux, double uy,
                      double uz) {
  const double den = nx * ux + ny * uy + nz * uz;
  const double num = c - (nx * ox + ny * oy + nz * oz);
  // A face counts as an exit candidate only if the ray leaves through it at a real angle:
  // n.u > kParallelTol*|u|_1, not n.u > 0.  (a) A plane component that is exactly zero carries the
  // payload byte as a denormal, so a ray exactly parallel to the face would see n.u = +-1e-321*|u|.
  // (b) A ray that runs inside a face plane or along a mesh edge sees n.u = rounding noise for the faces
  // that contain it, and num/den of such a face is an arbitrary number that can win the minimum.  No ray
  // that is not parallel to the face within 1e-12 rad is affected.
  const bool take = (den > kParallelTol * (fabs(ux) + fabs(uy) + fabs(uz))) && (num * s.bden < s.bnum * den);
  s.bnum = take ? num : s.bnum;
  s.bden = take ? den : s.bden;
  s.nbr = take ? nbr : s.nbr;
  s.back = take ? back : s.back;
}

// Lean flavour of the scan: instead of decoding the neighbour of every face and selecting among the
// decoded values, the raw payload word and the face index of the best face are kept and decoded once
// after the last face (6 integer instructions per face less).  Same selection rule, same result.
struct LeanScan {
  double bnum = 1.0, bden = 0.0;  // t = +inf
  uint32_t pay = 0;
  int32_t f = -1;  // -1: no exit candidate yet
};

PTB_HD void scan_face_lean(LeanScan &s, double nx, double ny, double nz, double c, int f, double tol, double ox,
                           double oy, double oz, double ux, double uy, double uz) {
  const double den = nx * ux + ny * uy + nz * uz;
  const double num = c - (nx * ox + ny * oy + nz * oz);
  const bool take = (den > tol) && (num * s.bden < s.bnum * den);  // tol = kParallelTol * |u|_1, see scan_face()
  const uint32_t pay = pack_low_bytes(dlo(nx), dlo(ny), dlo(nz), dlo(c));
  s.bnum = take ? num : s.bnum;
  s.bden = take ? den : s.bden;
  s.pay = take ? pay : s.pay;
  s.f = take ? f : s.f;
}

PTB_HD void decode_lean(const LeanScan &s, int32_t self, int32_t &nbr, int32_t &back) {
  const uint32_t x = (s.pay ^ (uint32_t)self) & kIdMask;
  nbr = s.f < 0 ? -2 : (int32_t)((x + 1u) & kIdMask) - 1;
  back = s.f < 0 ? -1 : (int32_t)((s.pay >> 30) ^ (uint32_t)s.f);
}

// bnum >= bden  <=>  t >= 1: the destination lies in this tet, no division needed
PTB_HD double exit_parameter(const ExitScan &s) {
  return (s.bnum < s.bden) ? s.bnum / s.bden : __builtin_huge_val();
}
PTB_HD double exit_parameter(const LeanScan &s) {
  return (s.bnum < s.bden) ? s.bnum / s.bden : __builtin_huge_val();
}

// All four faces of a record held as 16 raw doubles (variants that fetch the whole line).
PTB_HD void scan_record(const double (&r)[16], int32_t self, double ox, double oy, double oz,
                        double ux, double uy, double uz, ExitScan &s) {
PTB_UNROLL
  for (int f = 0; f < 4; ++f) {
    int32_t nb, bk;
    face_payload(r[4 * f], r[4 * f + 1], r[4 * f + 2], r[4 * f + 3], self, f, nb, bk);
    scan_face(s, r[4 * f], r[4 * f + 1], r[4 * f + 2], r[4 * f + 3], nb, bk, ox, oy, oz, ux, uy, uz);
  }
}


// ---------------------------------------------------------------------------
// Per-ray state machine shared by every kernel variant.
// ---------------------------------------------------------------------------

struct DeviceStats {
  unsigned long long segments;     // tally contributions (weighted phase, flying particles)
  unsigned long long tracks;       // flying particles in weighted phases
  unsigned long long relocations;  // crossings walked with tallying off
  unsigned long long lost;         // walks stopped by the iteration limit
  unsigned long long fallbacks;    // compact layout: rays handed to the plane records (coplanar edge)
};

struct TetRecord;
struct TetLinks;
struct VertexRec;
struct TetStart;

// Persistent per-particle state: position + parent element in one 32-byte, 32-byte aligned
// record = one DRAM/L2 sector.  A particle is read with two 128-bit loads of the same sector and
// written back with two 128-bit stores that cover the whole sector (no read-modify-write fill), in
// whatever order particles are processed.  (Reference: DPS members origin + the tracer's elem_ids,
// PumiTallyImpl.h:39-41.)
struct alignas(32) ParticleState {
  double x, y, z;
  int32_t elem;
  int32_t pad;
};
static_assert(sizeof(ParticleState) == 32, "ParticleState must be one sector");

PTB_HD ParticleState load_state(const ParticleState *p) {
#if defined(__CUDA_ARCH__)
  unsigned long long a, b, c, d;
  asm volatile(
      "ld.global.L1::no_allocate.v2.b64 {%0,%1}, [%4];\n\t"
      "ld.global.L1::no_allocate.v2.b64 {%2,%3}, [%4+16];"
      : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p));
  ParticleState s;
  s.x = __longlong_as_double((long long)a);
  s.y = __longlong_as_double((long long)b);
  s.z = __longlong_as_double((long long)c);
  s.elem = (int32_t)(d & 0xffffffffull);
  s.pad = 0;
  return s;
#else
  return *p;
#endif
}
PTB_HD void store_state(ParticleState *p, double x, double y, double z, int32_t elem) {
#if defined(__CUDA_ARCH__)
  asm volatile(
      "st.global.L1::no_allocate.v2.b64 [%0], {%1,%2};\n\t"
      "st.global.L1::no_allocate.v2.b64 [%0+16], {%3,%4};" ::"l"(p),
               "l"((unsigned long long)__double_as_longlong(x)), "l"((unsigned long long)__double_as_longlong(y)),
               "l"((unsigned long long)__double_as_longlong(z)), "l"((unsigned long long)(uint32_t)elem)
               : "memory");
#else
  p->x = x; p->y = y; p->z = z; p->elem = elem; p->pad = 0;
#endif
}

// Uniform background grid over the mesh bounding box: cell -> the tet that
// contains the cell centre (-1 if the centre is outside the mesh).  A far
// relocation (re-sampled particle, initial localisation) starts its tally-off
// walk at the centre of the target's cell instead of at the particle's old
// position.  For a target inside the mesh both walks end in the tet that
// contains it, so the result is the reference's; if the seeded walk meets the
// hull the kernel falls back to the reference walk from the old position,
// which also reproduces the clip point of an out-of-mesh target.
struct SeedGrid {
  const int32_t *cell_tet;  // [nx*ny*nz]; nullptr = grid disabled
  const int32_t *cell_rank; // [nx*ny*nz] position of the cell along a Morton curve (binning key)
  double x0, y0, z0;        // low corner of the bounding box
  double h, inv_h;          // cell edge and its reciprocal
  double far2;              // seed only when |target - position|^2 exceeds this
  int32_t nx, ny, nz;
};

// Seed point of cell (cx,cy,cz): deliberately off-centre so that structured
// meshes whose cell centres lie on tet faces/edges do not start every seeded
// walk in a degenerate position.  Explicit fma: identical on host and device.
PTB_HD void seed_point(const SeedGrid &g, int cx, int cy, int cz, double &x, double &y, double &z) {
  x = fma(cx + 0.41421356237, g.h, g.x0);
  y = fma(cy + 0.57735026919, g.h, g.y0);
  z = fma(cz + 0.31830988618, g.h, g.z0);
}

// One entry of the origin patch list (host-pointer path, delta upload): particle idx starts this
// move at (x,y,z) instead of at the previous move's destination.  32 bytes = one sector.
struct alignas(32) PatchEntry {
  double x, y, z;
  int32_t idx;
  int32_t pad;
};

// One row of the packed, spatially sorted particle batch (variant "packed"): everything a flying
// particle needs for this move in one 64-byte line, written by the binning pass in cell order and
// streamed by the walk kernel with one bulk copy per chunk.  The stored position is not carried:
// for every continuing particle it equals `origin` bit for bit; the others (bit 31 of `elem` set)
// read their ParticleState when they start.
struct alignas(64) PackedRow {
  double ox, oy, oz;  // origin (= position before the move unless the relocate bit is set)
  double dx, dy, dz;  // destination
  double w;
  int32_t id;         // particle index in the caller's arrays
  uint32_t elem;      // bits 0..29 parent element, bit 31: origin differs from the stored position
};
static_assert(sizeof(PackedRow) == 64, "PackedRow must be one 64-byte line");

// One launch = one particle range of one MoveToNextLocation / CopyInitialPosition.
struct WalkParams {
  const TetRecord *tets;   // [E] packed records
  const TetLinks *links;   // [E] compact layout (walk_compact.cuh); nullptr when not uploaded
  const VertexRec *verts;  // [V]
  const TetStart *starts;  // [E]
  double *flux;            // [E] raw tally
  ParticleState *state;    // [N] persistent particle position + parent element
  const double *origin;    // [3N] AoS relocation target (phase 1), nullptr = skip phase
  const double *dest;      // [3N] AoS flight target (phase 2), nullptr = skip phase
  const int8_t *flying;    // [N], nullptr = every particle flies (localisation)
  const double *weights;   // [N]
  int32_t begin, end;      // particle range
  int32_t max_iters;       // crossing limit per walk ("May need more loops in search")
  int32_t bulk_ok;         // all particle arrays 16-byte aligned: cp.async.bulk staging allowed
  unsigned int *work_counter;  // chunk ticket of the persistent kernel (zeroed per launch)
  const int32_t *order;        // gather mode: ids of the flying particles in processing order
  const unsigned int *work_count;  // gather mode: number of entries in order[] (device scalar)
  int32_t claim_run;           // gather mode: chunks per ticket (1, 2 or 4)
  const PackedRow *rows;       // packed mode: work_count rows in processing order
  DeviceStats *stats;
  SeedGrid grid;
  double cx, cy, cz;           // mesh centre: the planes are stored relative to it (tet_mesh.hpp)
  // Sorted (gather / packed) modes, optional: the SMs of each L2 partition work on their own end of the sorted
  // particle sequence (walk_persist.cuh, "die split").  die_mask bit s = partition of SM s; die0_sms of nsms SMs
  // are in partition 0; work_counter2 is the second partition's chunk ticket.  die0_sms == 0: off.
  uint32_t die_mask[8];
  int32_t die0_sms, nsms;
  unsigned int *work_counter2;
};

// ---- scored walk: several responses per track ------------------------------------------------------
// Within one move a particle keeps its material and energy, so every cross section is constant along
// the track: the caller passes one response r[i,k] per particle and score (e.g. the macroscopic cross
// sections) and a segment of length l in element e adds l * w[i] * r[i,k] to score k of e.  One walk
// serves all scores: the record fetches, the relocation and the positions are shared, each score costs
// one more reduction per crossing.
constexpr int kMaxScores = 8;

// Doubles per element of the internal flux array ([bin][element][score]): nscores padded to 1, 2, 4 or 8,
// so that the scores of one element share one 32-byte sector (nscores <= 4) or one 64-byte half line and
// the reductions of a crossing all land in one L2 line.
PTB_HD int score_stride(int nscores) { return nscores <= 1 ? 1 : nscores <= 2 ? 2 : nscores <= 4 ? 4 : 8; }

struct ScoreParams {
  const double *responses;  // [N * nscores], particle-major: r[i * nscores + k]
  int32_t nscores;          // 1..kMaxScores
  int32_t stride;           // score_stride(nscores)
};

// Parameters of a scored launch: the plain ones, unchanged, followed by the scores.
struct ScoredWalkParams : WalkParams {
  ScoreParams sc;
};

// One lane's scores.  wl[k * step] = w * r[i,k] * |u| of the lane's current track: written when the tally
// phase starts, read at every crossing (on the device a per-lane shared-memory slot, lane-contiguous per k).
struct ScoreLane {
  const double *responses;
  double *wl;
  int32_t n, stride, step;
};

// ---- timed walk: a time filter that splits every segment between time bins ------------------------
// Time advances along a flight (t = times[i] + s / speeds[i] at track distance s), so one segment can span
// several bins [T_j, T_j+1) of a time filter.  The timed walk is the scored one plus time: a segment adds
// w * r[i,k] * |u| * (ray-parameter overlap with bin j) to score k of time bin j, which is the track length
// spent in the bin.  Only the walk knows where a segment lies along the flight, so the split happens here:
// the common crossing (exit before the bin's upper edge) costs one comparison and issues exactly the scored
// step's reductions; each edge crossed costs one division.
constexpr int kMaxTimeBins = 1024;

struct TimeParams {
  const double *edges;   // [nt + 1], finite, strictly increasing
  const double *times;   // [N] time of particle i at its origin
  const double *speeds;  // [N] mesh length units per time unit, finite and > 0
  int32_t nt;            // time bins, 1..kMaxTimeBins
  int64_t slice;         // doubles from time bin j to j + 1 of the same array (0: every bin into one array)
};

// Parameters of a timed launch: the scored ones, unchanged, followed by the time filter.
struct TimedWalkParams : ScoredWalkParams {
  TimeParams tm;
};

// One lane's scores and time state.  Next to the score slots, at wl[(NS + m) * step]: m = 0 the time at ray
// parameter 0, m = 1 the time per unit ray parameter (|u| / v), m = 2 the upper edge of the current bin;
// *bin is the current bin (-1: before T_0, nt: at or after T_nt; neither is tallied).
struct TimeLane : ScoreLane {
  int32_t *bin;
};

// ---- face currents: the weight crossing every face --------------------------------------------------
// Each crossing of the tally phase adds the particle's weight w (not a response) to one double per (element, local
// face): for an interior face, the slot (next, back) of the element entered, so the slot holds the weight *entering*
// through it; for a hull face, the slot (e, f) of the element left, so the slot holds the weight *leaving* through it
// (nothing enters through the hull: the tally phase ends there).  Four doubles per element are one 32-byte sector; a
// crossing costs one more reduction and no fetch, since the neighbour and `back` are already decoded.  With a time
// filter the crossing goes to the bin that holds its time (time_tally's bin after the segment: a crossing exactly on
// an edge stays in the bin below).
//
// Cosine bins (MU): a crossing also goes to the bin of its cosine mu = fmin(bden * inv, 1.0), one rounded product and
// a clamp (crossing_cosine).  bden is the exit scan's n.u of the face the walk leaves through: the normal exactly as the
// record stores it, payload byte included, and the products summed as scan_face() sums them.  inv = 1.0 / len, one
// rounded division formed once per flight when the tally phase starts, where len = sqrt(ux * ux + uy * uy + uz * uz) is
// the length start_tally_to() forms for the weights (nvcc may contract that sum of squares into fmas; the host build,
// compiled without contraction, rounds each operation as written).  The face is an exit face, so mu lies in (0, 1], measured against the normal that points the way the particle travels; the same mu goes
// to whichever slot the crossing adds to (the neighbour's incoming slot or the hull's outgoing one).  Against a face
// with a fixed normal, an outgoing partial current holds the crossings at +mu and an incoming one those at -mu.  Bin k
// holds edges[k] <= mu < edges[k + 1], and mu == edges[nmu] goes to the last bin (OpenMC's MuFilter rule); a crossing
// with mu outside [edges[0], edges[nmu]] adds nothing.
constexpr int kMaxCosineBins = 64;

struct CurrentParams {
  double *cur;            // [E][4] of time bin 0 of the score bin (and cosine bin 0)
  int64_t slice;          // doubles from time bin j to j + 1 of cur (0: every time bin into one array)
  const double *edges;    // MU: [nmu + 1] cosine-bin edges in [0, 1], strictly increasing
  int32_t nmu;            // MU: cosine bins, 1..kMaxCosineBins
  int64_t mu_stride;      // MU: doubles from cosine bin k to k + 1 of cur (0: every cosine bin into one array)
};

// Parameters of a launch with face currents: the timed ones, unchanged, followed by the currents.
struct CurrentWalkParams : TimedWalkParams {
  CurrentParams cu;
};

// The lane slot that holds w, after the scores and the time slots: written when the tally phase starts (0 for a bad
// track), read at every crossing.
template <int NS, bool TM>
constexpr int kCurrentSlot = NS + (TM ? 3 : 0);

// ---- linear flux moments: the first spatial moment of every score ---------------------------------
// A segment of length l from ray parameter p to q adds w * r * l to score k and, with moments, w * r * l * (mid - C)
// to its first moment, mid = o + (p + q) / 2 * u the segment midpoint: the integral of (x - C) along a straight
// segment is exactly l * (mid - C).  The kernel accumulates about the mesh centre C (Ray::ox.., WalkParams::cx..),
// where the midpoint is already in registers; the host centres each element's record on its centroid c_e once at
// read time (m1 = R - (c_e - C) * m0, linear_moments() in tet_mesh.cpp).  An element's record is
// [m0 of scores 0..S-1][Rx 0..S-1][Ry 0..S-1][Rz 0..S-1], S = score_stride(nscores): its stride is 4 S doubles and
// m0 of score k stays at slot k, so with one score the four reductions of a crossing are one 32-byte sector.
constexpr int kMomentSlots = 4;

// The moments of one segment: a = (q - p) * wl[k] of every score is the tally step's own operand, unchanged.
template <int NS>
PTB_HD void moment_tally(double *f, const ScoreLane *sl, double p, double q, double ox, double oy, double oz, double ux,
                         double uy, double uz) {
  const double s = 0.5 * (p + q);
  const double mx = fma(s, ux, ox), my = fma(s, uy, oy), mz = fma(s, uz, oz);
  const int S = sl->stride / kMomentSlots;
  const double dt = q - p;
PTB_UNROLL
  for (int k = 0; k < NS; ++k)
    if (k < sl->n) {
      const double a = dt * sl->wl[k * sl->step];
      PTB_TALLY_ADD(f + k, a);
      PTB_TALLY_ADD(f + S + k, a * mx);
      PTB_TALLY_ADD(f + 2 * S + k, a * my);
      PTB_TALLY_ADD(f + 3 * S + k, a * mz);
    }
}

constexpr int kStageReloc = 0;  // phase 1: move to caller's origin, tally off
constexpr int kStageTally = 1;  // phase 2: fly to destination, tally on
constexpr int kStageDone = 2;
constexpr int kStageSeed = 3;   // phase 1 started from a seed-grid cell centre

struct Ray {
  double ox, oy, oz;  // ray origin (fixed for the whole walk), in mesh-centred coordinates
  double ux, uy, uz;  // target - origin
  double tx, ty, tz;  // target (stored exactly as given: it becomes the position when reached)
  double tcur;        // parameter of the last crossing (the reference's prev_xpoint)
  double wl;          // weight * |u|  (tally phase)
  int32_t e;          // current tet
  int32_t entry;      // local face of `e` the ray came in through (-1 at the start of a ray):
                      // it can never be the exit, so its sector need not be fetched
  int32_t stage;
  int32_t iters;
};

struct Counters {
  unsigned segs = 0, tracks = 0, relocs = 0, lost = 0, fallbacks = 0;
};

// (x,y,z) and the target are the caller's (absolute) coordinates; only the ray origin is translated,
// once: the direction is a difference and the target is kept as given (it becomes the stored position)
PTB_HD void set_ray(const WalkParams &P, Ray &r, double x, double y, double z, double tx, double ty, double tz) {
  r.ox = x - P.cx; r.oy = y - P.cy; r.oz = z - P.cz;
  r.ux = tx - x; r.uy = ty - y; r.uz = tz - z;
  r.tx = tx; r.ty = ty; r.tz = tz;
  r.tcur = 0.0;
  r.iters = 0;
  r.entry = -1;
}

// NaN or infinity in the caller's numbers must not reach the tally or the stored state: x*0 is 0 for
// every finite x and NaN otherwise.
PTB_HD bool all_finite(double a, double b, double c) { return (a * 0.0 + b * 0.0 + c * 0.0) == 0.0; }

// Tally phase towards (tx,ty,tz) with weight w.  A non-finite destination or weight turns the flight
// into a zero-length one (the particle stays where it is, nothing is tallied) and counts as lost.
// Timed walk, start of a track: the lane's time state for a flight that is at time t0 at ray parameter 0 and
// spends tpp time units per unit ray parameter.  The starting bin is found by binary search over the edges
// (a start exactly on an edge belongs to the bin above it); a bad track gets bin nt, which tallies nothing.
template <int NS>
PTB_HD void time_start(const TimedWalkParams &T, const TimeLane *tl, double t0, double tpp, bool bad) {
  const double *ed = T.tm.edges;
  const int nt = T.tm.nt;
  int lo = 0, hi = nt + 1;  // lo: number of edges <= t0
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (PTB_LDG(ed + mid) <= t0) lo = mid + 1;
    else hi = mid;
  }
  const int j = bad ? nt : lo - 1;
  double *wl = tl->wl;
  wl[NS * tl->step] = bad ? 0.0 : t0;
  wl[(NS + 1) * tl->step] = bad ? 0.0 : tpp;
  wl[(NS + 2) * tl->step] = j < nt ? PTB_LDG(ed + j + 1) : __builtin_huge_val();
  *tl->bin = j;
}

// Time bin of t: the number of edges <= t, minus one (-1 before T_0, nt at or after T_nt): a time on an edge belongs
// to the bin above it, as a track that starts there does (time_start).
PTB_HD int time_bin(const double *ed, int nt, double t) {
  int lo = 0, hi = nt + 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (PTB_LDG(ed + mid) <= t) lo = mid + 1;
    else hi = mid;
  }
  return lo - 1;
}

// MU: the cosine of a crossing whose exit face has n.u == bden, for a flight with 1 / |u| == inv.
PTB_HD double crossing_cosine(double bden, double inv) { return fmin(bden * inv, 1.0); }

// MU: the cosine bin of mu, -1 outside the edges.  time_bin() over edges[0..nmu - 1] gives the bin whose lower edge is
// the last one <= mu; mu == edges[nmu] stays in the last bin.
PTB_HD int cosine_bin(const CurrentParams &cu, double mu) {
  const int k = time_bin(cu.edges, cu.nmu - 1, mu);
  return (k >= 0 && mu <= PTB_LDG(cu.edges + cu.nmu)) ? k : -1;
}

// Timed walk, one crossing: the segment [tcur, tnew] (ray parameters) of element e.  While the exit time lies
// beyond the current bin's upper edge, the segment is cut at the edge's ray parameter and the bins are walked
// forward (time only increases along a ray).  A flight that ends exactly on an edge stays in the bin below.
// MO: every piece [p, pe] also adds its first moment (moment_tally), with the ray's origin o and direction u.
template <int NS, bool MO = false>
PTB_HD void time_tally(const TimedWalkParams &T, int32_t e, double tcur, double tnew, const TimeLane *tl,
                       const Ray *ray = nullptr) {
  const int step = tl->step;
  double *wl = tl->wl;
  const double t0 = wl[NS * step], tpp = wl[(NS + 1) * step];
  double tup = wl[(NS + 2) * step];
  int j = *tl->bin;
  double *f = T.flux + (size_t)e * tl->stride;
  double p = tcur;
  for (;;) {
    const bool split = fma(tnew, tpp, t0) > tup;
    const double pe = split ? fmin(fmax((tup - t0) / tpp, p), tnew) : tnew;
    if (j >= 0 && j < T.tm.nt) {
      const double dt = pe - p;
      double *fj = f + (size_t)j * (size_t)T.tm.slice;
      if constexpr (MO) {
        moment_tally<NS>(fj, tl, p, pe, ray->ox, ray->oy, ray->oz, ray->ux, ray->uy, ray->uz);
      } else {
PTB_UNROLL
        for (int k = 0; k < NS; ++k)
          if (k < tl->n) PTB_TALLY_ADD(fj + k, dt * wl[k * step]);
      }
    }
    if (!split) return;
    p = pe;
    ++j;
    tup = j < T.tm.nt ? PTB_LDG(T.tm.edges + j + 1) : __builtin_huge_val();
    wl[(NS + 2) * step] = tup;
    *tl->bin = j;
  }
}

// NS > 0: scored walk of up to NS scores (sl->n of them); particle i's responses are read here, once per
// track, and w * r[i,k] follows the rule for the weight.  w * r is exactly the weight a plain move with
// weights w * r[:,k] carries, so every score is that move's tally.
// TM: timed walk (NS > 0, sl is a TimeLane): particle i's time and speed are read here too; a non-finite time
// or a speed that is not finite and > 0 is a bad track like a non-finite weight.  No responses (nullptr):
// every r[i,k] is 1.
// MO: moment walk (NS > 0); responses may be nullptr here too (every r[i,k] 1), for the plain and binned moves.
// CU: face currents (NS > 0; P is a CurrentWalkParams): w goes to the lane's kCurrentSlot, 0 for a bad track; responses may
// be nullptr as with MO.
// MU: cosine bins (CU): 1 / |u| (1.0 / len, 0 for a bad track) goes to the slot after kCurrentSlot.
template <int NS = 0, bool TM = false, bool MO = false, bool CU = false, bool MU = false>
PTB_HD void start_tally_to(const WalkParams &P, Ray &r, double x, double y, double z, double tx, double ty,
                           double tz, double w, Counters &c, bool writer, int i = 0,
                           const ScoreLane *sl = nullptr) {
  static_assert(!CU || NS > 0, "face currents run on the tallied walk");
  static_assert(!MU || CU, "cosine bins split the face currents");
  if constexpr (NS == 0) {
    if (!all_finite(tx, ty, tz) || !all_finite(w, 0.0, 0.0)) {
      tx = x; ty = y; tz = z;
      w = 0.0;
      if (writer) c.lost++;
    }
    set_ray(P, r, x, y, z, tx, ty, tz);
    const double len = sqrt(r.ux * r.ux + r.uy * r.uy + r.uz * r.uz);
    r.wl = w * len;
  } else {
    bool bad = !all_finite(tx, ty, tz) || !all_finite(w, 0.0, 0.0);
    double t0 = 0.0, v = 1.0;
    if constexpr (TM) {
      const TimedWalkParams &T = static_cast<const TimedWalkParams &>(P);
      t0 = PTB_LDG(T.tm.times + i);
      v = PTB_LDG(T.tm.speeds + i);
      bad = bad || !all_finite(t0, v, 0.0) || !(v > 0.0);
    }
    const double *rp = sl->responses + (size_t)i * sl->n;
PTB_UNROLL
    for (int k = 0; k < NS; ++k)
      if (k < sl->n) {
        const double wr = w * ((!(TM || MO || CU) || sl->responses) ? PTB_LDG(rp + k) : 1.0);
        bad = bad || !all_finite(wr, 0.0, 0.0);
        sl->wl[k * sl->step] = wr;
      }
    if (bad) {
      tx = x; ty = y; tz = z;
      if (writer) c.lost++;
    }
    set_ray(P, r, x, y, z, tx, ty, tz);
    const double len = sqrt(r.ux * r.ux + r.uy * r.uy + r.uz * r.uz);
    r.wl = 0.0;  // (unused: the scores carry the weights)
PTB_UNROLL
    for (int k = 0; k < NS; ++k)
      if (k < sl->n) sl->wl[k * sl->step] = bad ? 0.0 : sl->wl[k * sl->step] * len;
    if constexpr (TM)
      time_start<NS>(static_cast<const TimedWalkParams &>(P), static_cast<const TimeLane *>(sl), t0, len / v, bad);
    if constexpr (CU) sl->wl[kCurrentSlot<NS, TM> * sl->step] = bad ? 0.0 : w;
    if constexpr (MU) sl->wl[(kCurrentSlot<NS, TM> + 1) * sl->step] = bad ? 0.0 : 1.0 / len;
  }
  r.stage = kStageTally;
  if (writer) c.tracks++;
}

template <int NS = 0, bool TM = false, bool MO = false, bool CU = false, bool MU = false>
PTB_HD void start_tally(const WalkParams &P, int i, Ray &r, double x, double y, double z,
                        Counters &c, bool writer, const ScoreLane *sl = nullptr) {
  start_tally_to<NS, TM, MO, CU, MU>(P, r, x, y, z, PTB_LDG(P.dest + 3 * (size_t)i), PTB_LDG(P.dest + 3 * (size_t)i + 1),
                     PTB_LDG(P.dest + 3 * (size_t)i + 2), PTB_LDG(P.weights + i), c, writer, i, sl);
}

// Phase 1 for a particle at (x,y,z) in tet r.e whose caller-side origin is (tx,ty,tz).
PTB_HD void start_reloc(const WalkParams &P, Ray &r, double x, double y, double z, double tx,
                        double ty, double tz) {
  r.wl = 0.0;  // p_wgt = 0 during relocation (Impl.cpp:105)
  const SeedGrid &g = P.grid;
  if (g.cell_tet) {
    const double dx = tx - x, dy = ty - y, dz = tz - z;
    const double fx = (tx - g.x0) * g.inv_h, fy = (ty - g.y0) * g.inv_h, fz = (tz - g.z0) * g.inv_h;
    if (dx * dx + dy * dy + dz * dz > g.far2 && fx >= 0.0 && fy >= 0.0 && fz >= 0.0 &&
        fx < (double)g.nx && fy < (double)g.ny && fz < (double)g.nz) {
      const int cx = (int)fx, cy = (int)fy, cz = (int)fz;
      const int32_t seed = PTB_LDG(g.cell_tet + ((size_t)cz * g.ny + cy) * g.nx + cx);
      if (seed >= 0) {
        double sx, sy, sz;
        seed_point(g, cx, cy, cz, sx, sy, sz);
        set_ray(P, r, sx, sy, sz, tx, ty, tz);
        r.e = seed;
        r.stage = kStageSeed;
        return;
      }
    }
  }
  set_ray(P, r, x, y, z, tx, ty, tz);
  r.stage = kStageReloc;
}

// K1/K2/K3 of the reference folded into the prologue: pick the walk target.
template <int NS = 0, bool TM = false, bool MO = false, bool CU = false, bool MU = false>
PTB_HD void begin_particle(const WalkParams &P, int i, Ray &r, Counters &c, bool writer,
                           const ScoreLane *sl = nullptr) {
  r.stage = kStageDone;
  const bool fly = P.flying ? (P.flying[i] == 1) : true;  // only the value 1 flies (Impl.cpp:95)
  if (!fly) return;  // dest := own origin => zero-length walk, nothing changes (Impl.cpp:100-102)
  const ParticleState s0 = load_state(P.state + i);
  const double x = s0.x, y = s0.y, z = s0.z;
  r.e = s0.elem;
  if (P.origin) {
    const double tx = PTB_LDG(P.origin + 3 * (size_t)i), ty = PTB_LDG(P.origin + 3 * (size_t)i + 1),
                 tz = PTB_LDG(P.origin + 3 * (size_t)i + 2);
    if (tx != x || ty != y || tz != z) {
      if (!all_finite(tx, ty, tz)) {  // unusable origin: the particle sits this move out
        if (writer) c.lost++;
        return;
      }
      start_reloc(P, r, x, y, z, tx, ty, tz);
      return;
    }
  }
  if (P.dest) start_tally<NS, TM, MO, CU, MU>(P, i, r, x, y, z, c, writer, sl);
}

// The current ray ended (target reached, hull hit, or iteration limit).
// kReloadTarget: the caller does not keep Ray::tx,ty,tz alive in registers (the compact-layout
// kernel); the target is read back from the caller's array, where it came from: dest[] in the
// tally phase, origin[] in phase 1.  Same values, six registers fewer in the crossing loop.
template <bool kReloadTarget = false, int NS = 0, bool TM = false, bool MO = false, bool CU = false, bool MU = false>
PTB_HD void end_ray(const WalkParams &P, int i, Ray &r, bool reached, double tnew, Counters &c,
                    bool writer, const ScoreLane *sl = nullptr) {
  // crossings of the ray that just ended: tally contributions in the tally phase, relocation crossings
  // otherwise (counted here, once per ray, instead of once per crossing)
  if (writer) {
    if (r.stage == kStageTally) c.segs += (unsigned)r.iters;
    else c.relocs += (unsigned)r.iters;
  }
  double x, y, z;
  if (kReloadTarget && (reached || r.stage == kStageSeed)) {
    const double *t = (r.stage == kStageTally ? P.dest : P.origin) + 3 * (size_t)i;
    r.tx = PTB_LDG(t); r.ty = PTB_LDG(t + 1); r.tz = PTB_LDG(t + 2);
  }
  if (r.stage == kStageSeed && !reached) {
    // the target is not reachable from the seed inside the mesh (it lies outside the hull):
    // redo phase 1 exactly as the reference does, from the particle's stored position
    const ParticleState s0 = load_state(P.state + i);
    x = s0.x; y = s0.y; z = s0.z;
    r.e = s0.elem;
    set_ray(P, r, x, y, z, r.tx, r.ty, r.tz);
    r.stage = kStageReloc;
    return;
  }
  if (reached) {  // tracer commit: origin <- dest, exactly (test lines 323-346)
    x = r.tx; y = r.ty; z = r.tz;
  } else {  // vacuum BC: dest <- intersection point (Impl.cpp:275-281)
    x = fma(tnew, r.ux, r.ox) + P.cx; y = fma(tnew, r.uy, r.oy) + P.cy; z = fma(tnew, r.uz, r.oz) + P.cz;
  }
  if (r.stage != kStageTally && P.dest) {
    start_tally<NS, TM, MO, CU, MU>(P, i, r, x, y, z, c, writer, sl);  // phase 2 starts where phase 1 ended
  } else {
    if (writer) {
      store_state(P.state + i, x, y, z, r.e);
    }
    r.stage = kStageDone;
  }
}

// Functor body for one crossing, given the tracer's answer (texit, next).
// NS > 0: scored walk (start_tally_to); one reduction per score into the element's scores.
// TM: timed walk (time_tally); the same reductions, into the time bins the segment spans.
// MO: moment walk (NS > 0): each of those reductions comes with the three of its first moment (moment_tally).
// CU: face currents (NS > 0): a crossing of the tally phase -- not the end of a flight, not a face the iteration limit
// stopped the walk at -- adds w to the slot of the face (CurrentParams).
// MU: cosine bins (CU): bden is the exit scan's n.u of that face, and the crossing goes to the slot of its cosine bin
// (cosine_bin), or nowhere outside the edges.  Without MU, bden is not read.
template <bool kReloadTarget = false, bool kAggregateTally = false, int NS = 0, bool TM = false, bool MO = false,
          bool CU = false, bool MU = false>
PTB_HD void advance(const WalkParams &P, int i, Ray &r, double texit, int32_t next, int32_t back,
                    Counters &c, bool writer, const ScoreLane *sl = nullptr, double bden = 0.0) {
  const bool reached = !(texit < 1.0);  // last_exit == -1: destination inside this tet
  const double tnew = reached ? 1.0 : fmax(texit, r.tcur);
  // MU: the crossing's cosine bin (-1: none) waits in the lane's second MU slot while the flux is tallied, so that
  // neither bden nor the bin is held in registers across it.  It is found for every step, relocation and the end of a
  // flight included, and read only for a crossing of the tally phase (where the 1 / |u| slot is the flight's own): a
  // guard on the tally phase here made ptxas spill 8 B more in the timed walks of variants 8 and 24.
  if constexpr (MU)
    sl->wl[(kCurrentSlot<NS, TM> + 2) * sl->step] = cosine_bin(static_cast<const CurrentWalkParams &>(P).cu,
        crossing_cosine(bden, sl->wl[(kCurrentSlot<NS, TM> + 1) * sl->step]));
  if constexpr (TM) {
    if (r.stage == kStageTally && writer)
      time_tally<NS, MO>(static_cast<const TimedWalkParams &>(P), r.e, r.tcur, tnew, static_cast<const TimeLane *>(sl), &r);
  } else if constexpr (MO) {
    if (r.stage == kStageTally && writer)
      moment_tally<NS>(P.flux + (size_t)r.e * sl->stride, sl, r.tcur, tnew, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz);
  } else if constexpr (NS > 0) {
    if (r.stage == kStageTally && writer) {
      const double dt = tnew - r.tcur;
      double *f = P.flux + (size_t)r.e * sl->stride;
PTB_UNROLL
      for (int k = 0; k < NS; ++k)
        if (k < sl->n) PTB_TALLY_ADD(f + k, dt * sl->wl[k * sl->step]);
    }
  } else {
#if defined(__CUDA_ARCH__)
  if constexpr (kAggregateTally) {
    tally_add_aggregated(P.flux, r.e, (tnew - r.tcur) * r.wl, r.stage == kStageTally && writer);
  } else
#endif
  if (r.stage == kStageTally && writer)  // EvaluateFlux (Impl.cpp:362-379)
    PTB_TALLY_ADD(P.flux + r.e, (tnew - r.tcur) * r.wl);
  }
  const bool hull = !reached && next < 0;  // next_elems == -1 (Impl.cpp:270-271)
  r.iters++;
  const bool over = r.iters >= P.max_iters;
  if constexpr (CU) {
    if (r.stage == kStageTally && writer && !reached && (hull || !over)) {
      const CurrentWalkParams &Q = static_cast<const CurrentWalkParams &>(P);
      int j = 0;
      if constexpr (TM) j = *static_cast<const TimeLane *>(sl)->bin;
      const double w = sl->wl[kCurrentSlot<NS, TM> * sl->step];
      if constexpr (MU) {
        const int kmu = (int)sl->wl[(kCurrentSlot<NS, TM> + 2) * sl->step];
        if ((!TM || (j >= 0 && j < Q.tm.nt)) && kmu >= 0)
          PTB_TALLY_ADD(Q.cu.cur + (size_t)j * (size_t)Q.cu.slice + (size_t)kmu * (size_t)Q.cu.mu_stride +
                            (size_t)(hull ? r.e : next) * 4 + back,
                        w);
      } else if (!TM || (j >= 0 && j < Q.tm.nt)) {
        PTB_TALLY_ADD(Q.cu.cur + (size_t)j * (size_t)Q.cu.slice + (size_t)(hull ? r.e : next) * 4 + back, w);
      }
    }
  }
  if (reached || hull || over) {
    if (over && !reached && !hull && writer && r.stage != kStageSeed) c.lost++;
    end_ray<kReloadTarget, NS, TM, MO, CU, MU>(P, i, r, reached, tnew, c, writer, sl);
  } else {
    r.e = next;  // UpdateCurrentElement (Impl.cpp:247-253)
    r.entry = back;
    r.tcur = tnew;
  }
}

// ---- point location: the element that contains an arbitrary point ---------------------------------
// The walk of a relocation with tallying off, without a particle.  The point's seed-grid cell gives the start: the
// cell's seed point and tet, or, for a cell without a seed on a convex hull, the centroid of the start element (where
// localisation starts).  The walk runs over the plane records to the point and the tet it ends in contains it; on a
// convex hull a walk that meets the hull proves the point outside.  On any other hull, a point whose walk meets the
// hull, whose cell has no seed, or whose walk is stopped by the iteration limit is tested against the cell's candidate
// tets instead (every tet whose bounding box overlaps the cell, a CSR list built on the host: cell_candidates() in
// seed_grid.hpp) with the four face planes of each record.
//
// Hull band: a point closer than kLocateBand * extent to the hull (extent = the longest edge of the bounding box) may
// get a hull tet or -1.  The walk decides such points on the hull planes, which are stored ~1e-13 * extent outwards
// (tet_mesh.cpp); the candidate test accepts a point within kLocateSlack * extent of a tet when no tet contains it
// strictly.  A point outside the bounding box, or with a non-finite coordinate, gets -1.
constexpr double kLocateBand = 1e-10;
constexpr double kLocateSlack = 1e-12;

struct LocateParams : WalkParams {  // uses tets, grid (cell_tet), max_iters and the mesh centre cx, cy, cz
  double sx, sy, sz;                // centroid of the start element (caller's coordinates)
  int32_t start_elem;               // internal id of the start element
  int32_t convex;                   // HostMesh::hull_convex
  const int64_t *cand_off;          // [ncell + 1] candidate list of each cell; nullptr on a convex hull
  const int32_t *cand;              // internal tet ids
  double slack;                     // kLocateSlack * extent
};

// Face planes of record r against the mesh-centred point p: is n.p <= c + slack for all four?
PTB_HD bool record_contains(const double (&r)[16], double px, double py, double pz, double slack) {
  bool in = true;
PTB_UNROLL
  for (int f = 0; f < 4; ++f)
    in = in && (r[4 * f + 3] - (r[4 * f] * px + r[4 * f + 1] * py + r[4 * f + 2] * pz) >= -slack);
  return in;
}

// Exact fallback: the first of the cell's candidates that contains the point strictly, else the first within the
// slack, else -1.  fetch(e, r) loads record e into r[16].
template <class Fetch>
PTB_HD int32_t locate_candidates(const LocateParams &P, int64_t cell, double px, double py, double pz, Fetch &&fetch) {
  if (!P.cand_off) return -1;
  const int64_t a = PTB_LDG(P.cand_off + cell), b = PTB_LDG(P.cand_off + cell + 1);
  int32_t near = -1;
  for (int64_t k = a; k < b; ++k) {
    const int32_t t = PTB_LDG(P.cand + k);
    double r[16];
    fetch(t, r);
    if (record_contains(r, px, py, pz, 0.0)) return t;
    if (near < 0 && record_contains(r, px, py, pz, P.slack)) near = t;
  }
  return near;
}

// Internal id of the element containing (x, y, z) (caller's coordinates), -1 outside the mesh.  Touches no particle.
template <class Fetch>
PTB_HD int32_t locate_point(const LocateParams &P, double x, double y, double z, Fetch &&fetch) {
  if (!all_finite(x, y, z)) return -1;
  const SeedGrid &g = P.grid;
  const double fx = (x - g.x0) * g.inv_h, fy = (y - g.y0) * g.inv_h, fz = (z - g.z0) * g.inv_h;
  if (!(fx >= 0.0 && fy >= 0.0 && fz >= 0.0 && fx < (double)g.nx && fy < (double)g.ny && fz < (double)g.nz)) return -1;
  const int cx = (int)fx, cy = (int)fy, cz = (int)fz;
  const int64_t cell = ((int64_t)cz * g.ny + cy) * g.nx + cx;
  const int32_t seed = PTB_LDG(g.cell_tet + cell);
  Ray r;
  if (seed >= 0) {
    double sx, sy, sz;
    seed_point(g, cx, cy, cz, sx, sy, sz);
    set_ray(P, r, sx, sy, sz, x, y, z);
    r.e = seed;
  } else if (P.convex) {
    set_ray(P, r, P.sx, P.sy, P.sz, x, y, z);
    r.e = P.start_elem;
  } else {
    return locate_candidates(P, cell, x - P.cx, y - P.cy, z - P.cz, fetch);
  }
  for (;;) {
    double rec[16];
    fetch(r.e, rec);
    ExitScan sc;
    scan_record(rec, r.e, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz, sc);
    if (!(exit_parameter(sc) < 1.0)) return r.e;  // the point lies in this tet
    const bool hull = sc.nbr < 0;
    if (hull && P.convex) return -1;  // left a convex mesh on the way to the point: it is outside
    if (hull || ++r.iters >= P.max_iters) break;
    r.e = sc.nbr;
  }
  return locate_candidates(P, cell, x - P.cx, y - P.cy, z - P.cz, fetch);
}

// ---- collision estimator: events scored at a point --------------------------------------------------
// The caller knows what happened at a collision (absorbed, scattered, the energy deposited), so it passes every event's
// weight w, responses r[k], score bin and time, and the event adds w * r[k] to score k of its element, in a region of
// d_flux_ laid out as the track-length tally ([time][bin][element][stride]).  With moments it also adds w * r[k] *
// (x - C) to the moment slots, C the mesh centre, as moment_tally does for a segment's midpoint.
struct CollisionParams {
  double *flux;              // time bin 0, bin 0, element 0 of the collision region
  const double *edges;       // [nt + 1] time bin edges (nt > 0)
  int32_t nt;                // time bins (0: no time filter; times are not read)
  int32_t nbins;             // score bins
  int32_t nscores, stride;   // stride: score_stride(nscores), times kMomentSlots with moments
  int32_t moments;           // 1: tally the first moments
  int64_t bin_stride;        // doubles from one score bin to the next (E * stride)
  int64_t slice;             // doubles from one time bin to the next (nbins * E * stride)
  double cx, cy, cz;         // mesh centre
};

// What became of an event; the first three are counted.
constexpr int kEventTallied = 0;
constexpr int kEventOutside = 1;   // located outside the mesh
constexpr int kEventRejected = 2;  // non-finite coordinate, weight * response or time
constexpr int kEventSkipped = 3;   // bin outside [0, nbins), or time before T_0 or at or after T_nt

// One event in element e (internal id, -1: outside the mesh) at (x, y, z) (caller's coordinates) with weight w,
// responses resp[0..nscores) (nullptr: every response 1), score bin `bin` and time t (read only with time bins).
// Rejected takes precedence over outside, outside over skipped.
PTB_HD int collision_event(const CollisionParams &P, int32_t e, double x, double y, double z, double w,
                           const double *resp, int32_t bin, double t) {
  double wr[kMaxScores];
  bool bad = !all_finite(x, y, z) || (P.nt > 0 && !all_finite(t, 0.0, 0.0));
PTB_UNROLL
  for (int k = 0; k < kMaxScores; ++k)
    if (k < P.nscores) {
      wr[k] = w * (resp ? PTB_LDG(resp + k) : 1.0);
      bad = bad || !all_finite(wr[k], 0.0, 0.0);
    }
  if (bad) return kEventRejected;
  if (e < 0) return kEventOutside;
  const int j = P.nt > 0 ? time_bin(P.edges, P.nt, t) : 0;
  if (bin < 0 || bin >= P.nbins || j < 0 || (P.nt > 0 && j >= P.nt)) return kEventSkipped;
  double *f = P.flux + (size_t)j * (size_t)P.slice + (size_t)bin * (size_t)P.bin_stride + (size_t)e * (size_t)P.stride;
  if (P.moments) {
    const int S = P.stride / kMomentSlots;
    const double dx = x - P.cx, dy = y - P.cy, dz = z - P.cz;
PTB_UNROLL
    for (int k = 0; k < kMaxScores; ++k)
      if (k < P.nscores) {
        PTB_TALLY_ADD(f + k, wr[k]);
        PTB_TALLY_ADD(f + S + k, wr[k] * dx);
        PTB_TALLY_ADD(f + 2 * S + k, wr[k] * dy);
        PTB_TALLY_ADD(f + 3 * S + k, wr[k] * dz);
      }
  } else {
PTB_UNROLL
    for (int k = 0; k < kMaxScores; ++k)
      if (k < P.nscores) PTB_TALLY_ADD(f + k, wr[k]);
  }
  return kEventTallied;
}

// ---- point detectors: next-event estimates of the flux at fixed points ------------------------------------------------
// Event i at x in element e and detector d at x_d form one ray.  Its score is w * r[k] * p * exp(-tau) / R^2, R = |x_d -
// x| and tau the line integral of Sigma_t from x to x_d over the mesh (detector_ray).  Inside the exclusion radius r0
// (R < r0) nothing is traced and the ray scores the mean of exp(-Sigma r) / r^2 over the ball instead, with Sigma the
// event element's: w * r[k] * p * 3 g(Sigma r0) / r0^2, g(x) = -expm1(-x) / x.
constexpr int kRayTraced = 0;    // the walk reached the tet that contains the detector
constexpr int kRayShadowed = 1;  // the ray left the mesh through the hull first: it scores 0
constexpr int kRayLost = 2;      // stopped by the iteration limit: it scores 0
constexpr int kRayInsideR0 = 3;  // R < r0: the ball formula, no walk
// the outcomes of detector_event that are not one of the four above
constexpr int kDetOutside = 4;   // the event lies outside the mesh (counted once per event)
constexpr int kDetRejected = 5;  // a non-finite coordinate, w * r[k], time or pdf value, a negative pdf value, a speed
                                 // not > 0, or R == 0 at a detector with r0 == 0 (counted once per event)
constexpr int kDetSkipped = 6;   // bin outside [0, nbins), or arrival time outside [T_0, T_nt): not traced, not counted

constexpr int kMaxDetectors = 256;

struct DetectorParams {
  double *tally;          // [time][bin][score][D]
  const double *sigma;    // [nbins][E] Sigma_t in internal element order
  const double *pos;      // [3D] detector positions (caller's coordinates)
  const double *r0;       // [D] exclusion radii
  const double *edges;    // [nt + 1] time bin edges (nt > 0)
  int32_t nt;             // time bins (0: times and speeds are not read)
  int32_t nbins, nscores, ndet;
  int32_t zero_r0;        // some detector has r0 == 0 (an event exactly on it is rejected)
  int64_t E;
};

// ---- detector void: the space outside the mesh is a void the rays cross (pumitally_set_detector_void) -------------
// With the void on, a ray that leaves the mesh through the hull is not shadowed: hull_entry() finds the first tet it
// enters again, and a ray from an event outside the mesh starts there.  The candidates are the hull tets (a tet with a
// face on the hull) of every seed-grid cell, CSR lists built by cell_candidates() (seed_grid.hpp) with a hull filter.
struct HullGrid {
  SeedGrid g;           // the seed grid's geometry (h, inv_h, nx, ny, nz); cell_tet is not read
  double ox, oy, oz;    // the grid's low corner (x0, y0, z0) in mesh-centred coordinates, as the rays' origins are
  const int64_t *off;   // [ncell + 1] hull-tet list of each cell
  const int32_t *tets;  // internal tet ids
  int32_t convex;       // HostMesh::hull_convex: a ray that has left the mesh cannot come back
};

// Entry parameter of the ray into the record's tet: the largest num / den over the faces the ray enters through (den <
// -tol, with num and den as scan_face forms them), -inf when there is none, +inf when a face parallel to the ray within
// tol has the ray outside its plane (num < 0).
PTB_HD double entry_parameter(const double (&r)[16], const Ray &ray) {
  const double tol = kParallelTol * (fabs(ray.ux) + fabs(ray.uy) + fabs(ray.uz));
  double tin = -__builtin_huge_val();
PTB_UNROLL
  for (int f = 0; f < 4; ++f) {
    const double nx = r[4 * f], ny = r[4 * f + 1], nz = r[4 * f + 2];
    const double den = nx * ray.ux + ny * ray.uy + nz * ray.uz;
    const double num = r[4 * f + 3] - (nx * ray.ox + ny * ray.oy + nz * ray.oz);
    if (den < -tol) tin = fmax(tin, num / den);
    else if (!(den > tol) && num < 0.0) tin = __builtin_huge_val();
  }
  return tin;
}

// The first tet the ray enters at or after tcur.  [tcur, 1] is clipped to the grid's box and the cells along it are
// visited in order (Amanatides-Woo).  Every candidate of a cell is clipped against its record's four planes: [tin,
// tout], tout from scan_record and exit_parameter exactly as the walk forms its exit, tin from entry_parameter.  A
// candidate with tout > tcur and tin <= tout enters at max(tin, tcur); the smallest wins, ties to the first found, and
// the search stops once it lies within the cell being visited.  Returns the tet (-1: the ray enters no tet before t =
// 1) and *tenter.  The walk then leaves the tet at its own exit parameter, which is this tout > tcur, through the same
// planes: it stays monotone and watertight.  A cell missed by rounding at a cell boundary is covered by the lists'
// padding (kLocateBand * extent, Engine::ensure_hull_grid).  fetch(e, r) loads record e.
template <class Fetch>
PTB_HD int32_t hull_entry(const HullGrid &H, const Ray &ray, double tcur, double *tenter, Fetch &&fetch) {
  const SeedGrid &g = H.g;
  const double inf = __builtin_huge_val();
  // position in cell units: f + t df
  const double fx = (ray.ox - H.ox) * g.inv_h, fy = (ray.oy - H.oy) * g.inv_h, fz = (ray.oz - H.oz) * g.inv_h;
  const double dfx = ray.ux * g.inv_h, dfy = ray.uy * g.inv_h, dfz = ray.uz * g.inv_h;
  double t0 = tcur, t1 = 1.0;
  auto clip = [&](double f, double df, int n) {
    if (df == 0.0) {
      if (!(f >= 0.0 && f <= (double)n)) t1 = -inf;
    } else {
      const double a = -f / df, b = ((double)n - f) / df;
      t0 = fmax(t0, fmin(a, b));
      t1 = fmin(t1, fmax(a, b));
    }
  };
  clip(fx, dfx, g.nx);
  clip(fy, dfy, g.ny);
  clip(fz, dfz, g.nz);
  if (!(t0 <= t1)) return -1;
  auto cell_of = [&](double f, double df, int n) { return (int)fmin(fmax(floor(f + t0 * df), 0.0), (double)(n - 1)); };
  auto next_of = [&](int c, double f, double df) { return df == 0.0 ? inf : ((double)(c + (df > 0.0)) - f) / df; };
  int cx = cell_of(fx, dfx, g.nx), cy = cell_of(fy, dfy, g.ny), cz = cell_of(fz, dfz, g.nz);
  double nxt = next_of(cx, fx, dfx), nyt = next_of(cy, fy, dfy), nzt = next_of(cz, fz, dfz);
  int32_t best = -1;
  double bt = inf;
  for (;;) {
    const double tfar = fmin(fmin(nxt, nyt), fmin(nzt, t1));
    const int64_t cell = ((int64_t)cz * g.ny + cy) * g.nx + cx;
    const int64_t a = PTB_LDG(H.off + cell), b = PTB_LDG(H.off + cell + 1);
    for (int64_t k = a; k < b; ++k) {
      const int32_t t = PTB_LDG(H.tets + k);
      double rec[16];
      fetch(t, rec);
      ExitScan sc;
      scan_record(rec, t, ray.ox, ray.oy, ray.oz, ray.ux, ray.uy, ray.uz, sc);
      const double tout = exit_parameter(sc), tin = entry_parameter(rec, ray);
      const double te = fmax(tin, tcur);
      if (tout > tcur && tin <= tout && te < bt) {
        bt = te;
        best = t;
      }
    }
    if (bt <= tfar || !(tfar < t1)) break;
    if (nxt <= nyt && nxt <= nzt) {
      cx += dfx > 0.0 ? 1 : -1;
      if (cx < 0 || cx >= g.nx) break;
      nxt = next_of(cx, fx, dfx);
    } else if (nyt <= nzt) {
      cy += dfy > 0.0 ? 1 : -1;
      if (cy < 0 || cy >= g.ny) break;
      nyt = next_of(cy, fy, dfy);
    } else {
      cz += dfz > 0.0 ? 1 : -1;
      if (cz < 0 || cz >= g.nz) break;
      nzt = next_of(cz, fz, dfz);
    }
  }
  if (!(bt < 1.0)) return -1;
  *tenter = bt;
  return best;
}

// tau / R of the straight line from (x, y, z) in element e to (tx, ty, tz): the sum over the tets the walk crosses of
// sig[tet] times the ray parameter spent in it.  The loop is locate_point's (record, scan_record, exit_parameter), the
// step rule advance()'s.  Returns kRayTraced, kRayShadowed or kRayLost; crossings += the interior faces crossed.
// VOID (the detector void, with H its hull grid): an event outside the mesh (e == -1) starts at its ray's first entry,
// a hull exit searches for the next entry from the exit instead of shadowing the ray, and a ray that enters no tet
// again is traced: the void adds nothing to tau.  On a convex hull a ray that has left never comes back, so only the
// first entry is searched for.  Every entry counts one iteration against max_iters and one in *entries.
template <bool VOID = false, class Fetch>
PTB_HD int detector_ray(const WalkParams &P, const double *sig, int32_t e, double x, double y, double z, double tx,
                        double ty, double tz, double &tau_over_r, uint32_t &crossings, Fetch &&fetch,
                        const HullGrid *H = nullptr, uint32_t *entries = nullptr) {
  Ray r;
  set_ray(P, r, x, y, z, tx, ty, tz);
  r.e = e;
  double s = 0.0;
  if constexpr (VOID) {
    // one search site, so that the search and the walk share their registers
    tau_over_r = 0.0;
    bool search = e < 0;
    for (;;) {
      if (search) {
        r.e = hull_entry(*H, r, r.tcur, &r.tcur, fetch);
        if (r.e < 0) return kRayTraced;  // the rest of the ray lies in the void
        if (++r.iters >= P.max_iters) return kRayLost;
        ++*entries;
      }
      double rec[16];
      fetch(r.e, rec);
      ExitScan sc;
      scan_record(rec, r.e, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz, sc);
      const double texit = exit_parameter(sc);
      const bool reached = !(texit < 1.0);
      const double tnew = reached ? 1.0 : fmax(texit, r.tcur);
      s += PTB_LDG(sig + r.e) * (tnew - r.tcur);
      tau_over_r = s;
      if (reached) return kRayTraced;
      search = sc.nbr < 0;  // out through the hull: on to the next entry, if the hull lets there be one
      if (search && H->convex) return kRayTraced;
      if (!search) {
        if (++r.iters >= P.max_iters) return kRayLost;
        ++crossings;
        r.e = sc.nbr;
      }
      r.tcur = tnew;
    }
  } else {
    for (;;) {
      double rec[16];
      fetch(r.e, rec);
      ExitScan sc;
      scan_record(rec, r.e, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz, sc);
      const double texit = exit_parameter(sc);
      const bool reached = !(texit < 1.0);
      const double tnew = reached ? 1.0 : fmax(texit, r.tcur);
      s += PTB_LDG(sig + r.e) * (tnew - r.tcur);
      tau_over_r = s;
      if (reached) return kRayTraced;
      if (sc.nbr < 0) return kRayShadowed;  // graveyard outside the hull: re-entry across a concave notch is not followed
      if (++r.iters >= P.max_iters) return kRayLost;
      ++crossings;
      r.e = sc.nbr;
      r.tcur = tnew;
    }
  }
}

// g(x) = (1 - exp(-x)) / x, 1 at x = 0, through expm1 so that small x keeps its digits
PTB_HD double ball_g(double x) { return x > 0.0 ? -expm1(-x) / x : 1.0; }

// Event (x, y, z) in element e (internal id, -1 outside) with weight w, responses resp (nullptr: 1), score bin `bin`,
// time t and speed v (read only with time bins), and pdf[0..D) the event's angular densities toward the detectors (per
// steradian; nullptr: 1 / (4 pi)).  Every ray of an event checks the whole event, pdf row and R == 0 == r0 at every
// detector included (kDetRejected), before whether it lies in the mesh (kDetOutside): rejection takes precedence, and
// all the rays of an event share its outcome, which the kernels count once per event.  On a scoring outcome (traced,
// inside r0) val[k] = the score of score k and *slot = its [time][bin][0][d] index (score k at slot + k D).
// Shadowed and lost rays return val 0.  crossings += the interior faces the walk crossed.
// VOID (the detector void, detector_ray): an event outside the mesh is not kDetOutside but traced from where it is, and
// inside r0 it takes the ball formula with Sigma = 0 (3 / r0^2); *entries += the ray's entries through the hull.
template <bool VOID = false, class Fetch>
PTB_HD int detector_event(const WalkParams &W, const DetectorParams &P, int d, int32_t e, double x, double y, double z,
                          double w, const double *resp, int32_t bin, double t, double v, const double *pdf,
                          double *val, int64_t *slot, uint32_t &crossings, Fetch &&fetch, const HullGrid *H = nullptr,
                          uint32_t *entries = nullptr) {
  bool bad = !all_finite(x, y, z) || (P.nt > 0 && (!all_finite(t, 0.0, 0.0) || !(v > 0.0)));
PTB_UNROLL
  for (int k = 0; k < kMaxScores; ++k)
    if (k < P.nscores) {
      val[k] = w * (resp ? PTB_LDG(resp + k) : 1.0);
      bad = bad || !all_finite(val[k], 0.0, 0.0);
    }
  if (pdf)
    for (int q = 0; q < P.ndet; ++q) {
      const double p = PTB_LDG(pdf + q);
      bad = bad || !all_finite(p, 0.0, 0.0) || p < 0.0;
    }
  if (P.zero_r0 && !bad)
    for (int q = 0; q < P.ndet; ++q) {
      const double ax = PTB_LDG(P.pos + 3 * q) - x, ay = PTB_LDG(P.pos + 3 * q + 1) - y, az = PTB_LDG(P.pos + 3 * q + 2) - z;
      bad = bad || (PTB_LDG(P.r0 + q) == 0.0 && sqrt(ax * ax + ay * ay + az * az) == 0.0);
    }
  if (bad) return kDetRejected;
  if constexpr (!VOID)
    if (e < 0) return kDetOutside;
  const double pd = pdf ? PTB_LDG(pdf + d) : 0.25 / M_PI;
  const double dx = PTB_LDG(P.pos + 3 * d), dy = PTB_LDG(P.pos + 3 * d + 1), dz = PTB_LDG(P.pos + 3 * d + 2);
  const double ux = dx - x, uy = dy - y, uz = dz - z;
  const double R = sqrt(ux * ux + uy * uy + uz * uz);
  const double r0 = PTB_LDG(P.r0 + d);
  const int j = P.nt > 0 ? time_bin(P.edges, P.nt, t + R / v) : 0;
  if (bin < 0 || bin >= P.nbins || j < 0 || (P.nt > 0 && j >= P.nt)) return kDetSkipped;
  const double *sig = P.sigma + (size_t)bin * (size_t)P.E;
  double f;
  int outcome;
  if (R < r0) {
    f = pd * 3.0 * ball_g((VOID && e < 0 ? 0.0 : PTB_LDG(sig + e)) * r0) / (r0 * r0);
    outcome = kRayInsideR0;
  } else {
    double tr = 0.0;
    outcome = detector_ray<VOID>(W, sig, e, x, y, z, dx, dy, dz, tr, crossings, fetch, H, entries);
    f = outcome == kRayTraced ? pd * exp(-(tr * R)) / (R * R) : 0.0;
  }
PTB_UNROLL
  for (int k = 0; k < kMaxScores; ++k)
    if (k < P.nscores) val[k] *= f;
  *slot = ((int64_t)j * P.nbins + bin) * (int64_t)P.nscores * P.ndet + d;
  return outcome;
}

}  // namespace ptb
