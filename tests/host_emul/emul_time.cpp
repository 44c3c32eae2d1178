// TEST-ONLY host build of the timed tally step (walk_core.cuh, NS > 0 with TM).
//
// The same per-ray state machine as emul_scores.cpp, instantiated for kMaxScores scores and a time filter the way
// the timed kernels instantiate it, with the lane's score and time slots in ordinary arrays.  Compiled by g++ so
// that the time split can be checked against the oracle on a machine without a GPU; never linked into
// libpumitally.so.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "tet_mesh.hpp"
#include "walk_core.cuh"

using namespace ptb;

namespace {
struct TimedEmul {
  HostMesh mesh;
  std::vector<TetRecord> recs;
  std::vector<double> flux;  // [time][element][stride], internal order
  std::vector<double> edges;
  std::vector<ParticleState> state;
  DeviceStats stats{};
  int n = 0, nscores = 1, stride = 1, nt = 1;

  // times == nullptr: localisation (no tally phase)
  void walk(const double *origin, const double *dest, const int8_t *flying, const double *weights,
            const double *responses, const double *times, const double *speeds) {
    TimedWalkParams P{};
    P.tets = recs.data();
    P.flux = flux.data();
    P.state = state.data();
    P.origin = origin; P.dest = dest; P.flying = flying; P.weights = weights;
    P.begin = 0; P.end = n;
    P.max_iters = int32_t(mesh.ntets + 16);
    P.stats = &stats;
    P.cx = mesh.center[0]; P.cy = mesh.center[1]; P.cz = mesh.center[2];
    P.sc = ScoreParams{responses, nscores, stride};
    P.tm = TimeParams{edges.data(), times, speeds, nt, int64_t(mesh.ntets) * stride};
    double wl[kMaxScores + 3];
    int32_t bin = 0;
    TimeLane tl;
    tl.responses = responses;
    tl.wl = wl;
    tl.n = nscores;
    tl.stride = stride;
    tl.step = 1;
    tl.bin = &bin;
    for (int i = 0; i < n; ++i) {
      Counters c;
      Ray r;
      if (times) begin_particle<kMaxScores, true>(P, i, r, c, true, &tl);
      else begin_particle(P, i, r, c, true);
      while (r.stage != kStageDone) {
        // the persistent kernels' fetch: the entry face's sector is never read
        const double *rec = recs[r.e].d;
        const int en = r.entry;
        ExitScan sc;
        for (int k = 0; k < (en < 0 ? 4 : 3); ++k) {
          const int fk = k + ((en >= 0 && k >= en) ? 1 : 0);
          int32_t nb, bk;
          face_payload(rec[4 * fk], rec[4 * fk + 1], rec[4 * fk + 2], rec[4 * fk + 3], r.e, fk, nb, bk);
          scan_face(sc, rec[4 * fk], rec[4 * fk + 1], rec[4 * fk + 2], rec[4 * fk + 3], nb, bk, r.ox, r.oy, r.oz,
                    r.ux, r.uy, r.uz);
        }
        if (times) advance<false, false, kMaxScores, true>(P, i, r, exit_parameter(sc), sc.nbr, sc.back, c, true, &tl);
        else advance(P, i, r, exit_parameter(sc), sc.nbr, sc.back, c, true);
      }
      stats.segments += c.segs; stats.tracks += c.tracks;
      stats.relocations += c.relocs; stats.lost += c.lost;
    }
  }
};
}  // namespace

extern "C" {
void *ptb_timed_create(const double *coords, int64_t nverts, const int32_t *t2v, int64_t ntets, int n, int nscores,
                       const double *edges, int nedges) {
  if (nscores < 1 || nscores > kMaxScores || nedges < 2 || nedges - 1 > kMaxTimeBins) return nullptr;
  auto *e = new TimedEmul;
  std::string err;
  if (!e->mesh.from_arrays(coords, nverts, t2v, ntets, &err)) { delete e; return nullptr; }
  e->recs = e->mesh.records;
  e->n = n;
  e->nscores = nscores;
  e->stride = score_stride(nscores);
  e->nt = nedges - 1;
  e->edges.assign(edges, edges + nedges);
  e->flux.assign(size_t(e->nt) * size_t(ntets) * size_t(e->stride), 0.0);
  e->state.assign(size_t(n), ParticleState{e->mesh.centroid0[0], e->mesh.centroid0[1], e->mesh.centroid0[2], e->mesh.start_elem, 0});
  return e;
}
void ptb_timed_destroy(void *h) { delete static_cast<TimedEmul *>(h); }
void ptb_timed_localize(void *h, const double *xyz) {
  static_cast<TimedEmul *>(h)->walk(xyz, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
}
// r == nullptr: every response 1 (one score)
void ptb_timed_move(void *h, const double *origin, const double *dest, int8_t *flying, const double *w, const double *r,
                    const double *times, const double *speeds) {
  auto *e = static_cast<TimedEmul *>(h);
  e->walk(origin, dest, flying, w, r, times, speeds);
  std::memset(flying, 0, size_t(e->n));
}
// flux: [time][score][E] in the caller's numbering
void ptb_timed_get(void *h, double *flux, int32_t *elem, double *pos, unsigned long long *stats) {
  auto *e = static_cast<TimedEmul *>(h);
  const int64_t E = e->mesh.ntets;
  for (int t = 0; t < e->nt; ++t)
    for (int k = 0; k < e->nscores; ++k)
      for (int64_t i = 0; i < E; ++i)
        flux[(int64_t(t) * e->nscores + k) * E + e->mesh.orig_of_internal[i]] =
            e->flux[(size_t(t) * size_t(E) + size_t(i)) * e->stride + k];
  for (int i = 0; i < e->n; ++i) {
    elem[i] = e->mesh.orig_of_internal[e->state[i].elem];
    pos[3 * i] = e->state[i].x; pos[3 * i + 1] = e->state[i].y; pos[3 * i + 2] = e->state[i].z;
  }
  stats[0] = e->stats.segments; stats[1] = e->stats.tracks; stats[2] = e->stats.relocations; stats[3] = e->stats.lost;
}
}
