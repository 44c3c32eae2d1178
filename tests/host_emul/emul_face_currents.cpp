// TEST-ONLY host build of the face-current crossing step (walk_core.cuh, CU with and without TM and MO).
//
// The same per-ray state machine as emul_moments.cpp, instantiated for kMaxScores scores with face currents, with or
// without a time filter and moments, the way the CU kernels instantiate it.  The internal slots are read out with the
// engine's convention (4 * neighbour + back of the record's payload; the hull slot is the element's own).  Compiled by
// g++ so that the crossing rule can be checked against an exact reference on a machine without a GPU; never linked
// into libpumitally.so.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "tet_mesh.hpp"
#include "walk_core.cuh"

using namespace ptb;

namespace {
struct CurrentEmul {
  HostMesh mesh;
  std::vector<TetRecord> recs;
  std::vector<double> flux;  // [time][element][stride], internal order
  std::vector<double> cur;   // [time][element][4], internal order
  std::vector<double> edges;
  std::vector<ParticleState> state;
  DeviceStats stats{};
  int n = 0, nscores = 1, stride = 1, nt = 0, max_iters = 0;
  bool mo = false;

  template <bool TM, bool MO>
  void walk(const double *origin, const double *dest, const int8_t *flying, const double *weights,
            const double *responses, const double *times, const double *speeds) {
    CurrentWalkParams P{};
    P.tets = recs.data();
    P.flux = flux.data();
    P.state = state.data();
    P.origin = origin; P.dest = dest; P.flying = flying; P.weights = weights;
    P.begin = 0; P.end = n;
    P.max_iters = max_iters > 0 ? max_iters : int32_t(mesh.ntets + 16);
    P.stats = &stats;
    P.cx = mesh.center[0]; P.cy = mesh.center[1]; P.cz = mesh.center[2];
    P.sc = ScoreParams{responses, nscores, stride};
    P.tm = TimeParams{edges.data(), times, speeds, nt, int64_t(mesh.ntets) * stride};
    P.cu = CurrentParams{cur.data(), int64_t(mesh.ntets) * 4};
    double wl[kMaxScores + 4];
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
      if (dest) begin_particle<kMaxScores, TM, MO, true>(P, i, r, c, true, &tl);
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
        if (dest)
          advance<false, false, kMaxScores, TM, MO, true>(P, i, r, exit_parameter(sc), sc.nbr, sc.back, c, true, &tl);
        else
          advance(P, i, r, exit_parameter(sc), sc.nbr, sc.back, c, true);
      }
      stats.segments += c.segs; stats.tracks += c.tracks;
      stats.relocations += c.relocs; stats.lost += c.lost;
    }
  }
};
}  // namespace

extern "C" {
// nedges == 0: no time filter; moments: 0 or 1; max_iters 0: the engine's default (ntets + 16)
void *ptb_currents_create(const double *coords, int64_t nverts, const int32_t *t2v, int64_t ntets, int n, int nscores,
                          const double *edges, int nedges, int moments, int max_iters) {
  if (nscores < 1 || nscores > kMaxScores || nedges == 1 || nedges - 1 > kMaxTimeBins) return nullptr;
  auto *e = new CurrentEmul;
  std::string err;
  if (!e->mesh.from_arrays(coords, nverts, t2v, ntets, &err)) { delete e; return nullptr; }
  e->recs = e->mesh.records;
  e->n = n;
  e->nscores = nscores;
  e->mo = moments != 0;
  e->stride = score_stride(nscores) * (e->mo ? kMomentSlots : 1);
  e->nt = nedges > 0 ? nedges - 1 : 0;
  e->max_iters = max_iters;
  if (nedges > 0) e->edges.assign(edges, edges + nedges);
  const size_t T = size_t(e->nt > 0 ? e->nt : 1);
  e->flux.assign(T * size_t(ntets) * size_t(e->stride), 0.0);
  e->cur.assign(T * size_t(ntets) * 4, 0.0);
  e->state.assign(size_t(n), ParticleState{e->mesh.centroid0[0], e->mesh.centroid0[1], e->mesh.centroid0[2], e->mesh.start_elem, 0});
  return e;
}
void ptb_currents_destroy(void *h) { delete static_cast<CurrentEmul *>(h); }
void ptb_currents_localize(void *h, const double *xyz) {
  static_cast<CurrentEmul *>(h)->walk<false, false>(xyz, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
}
// r == nullptr: every response 1 (one score); times/speeds only with time bins
void ptb_currents_move(void *h, const double *origin, const double *dest, int8_t *flying, const double *w, const double *r,
                       const double *times, const double *speeds) {
  auto *e = static_cast<CurrentEmul *>(h);
  if (e->nt > 0) {
    if (e->mo) e->walk<true, true>(origin, dest, flying, w, r, times, speeds);
    else e->walk<true, false>(origin, dest, flying, w, r, times, speeds);
  } else {
    if (e->mo) e->walk<false, true>(origin, dest, flying, w, r, nullptr, nullptr);
    else e->walk<false, false>(origin, dest, flying, w, r, nullptr, nullptr);
  }
  std::memset(flying, 0, size_t(e->n));
}
// out, in: [time][E][4] in the caller's numbering; adj: [E][4] (adjacency_original); elem, pos: particles; stats[4]
void ptb_currents_get(void *h, double *out, double *in, int32_t *adj, int32_t *elem, double *pos,
                      unsigned long long *stats) {
  auto *e = static_cast<CurrentEmul *>(h);
  const int64_t E = e->mesh.ntets;
  const int T = e->nt > 0 ? e->nt : 1;
  const std::vector<int32_t> &t2t = e->mesh.t2t;
  for (int t = 0; t < T; ++t)
    for (int64_t i = 0; i < E; ++i)
      for (int f = 0; f < 4; ++f) {
        const int32_t nb = t2t[size_t(4 * i + f)];
        int back = f;
        if (nb >= 0)
          for (int q = 0; q < 4; ++q)
            if (t2t[4 * size_t(nb) + q] == int32_t(i)) back = q;
        const double *c = e->cur.data() + size_t(t) * size_t(E) * 4;
        const size_t o = (size_t(t) * size_t(E) + size_t(e->mesh.orig_of_internal[i])) * 4 + size_t(f);
        out[o] = nb >= 0 ? c[4 * size_t(nb) + size_t(back)] : c[4 * size_t(i) + size_t(f)];
        in[o] = nb >= 0 ? c[4 * size_t(i) + size_t(f)] : 0.0;
      }
  const std::vector<int32_t> a = e->mesh.adjacency_original();
  std::memcpy(adj, a.data(), a.size() * sizeof(int32_t));
  for (int i = 0; i < e->n; ++i) {
    elem[i] = e->mesh.orig_of_internal[e->state[i].elem];
    pos[3 * i] = e->state[i].x; pos[3 * i + 1] = e->state[i].y; pos[3 * i + 2] = e->state[i].z;
  }
  stats[0] = e->stats.segments; stats[1] = e->stats.tracks; stats[2] = e->stats.relocations; stats[3] = e->stats.lost;
}
}
