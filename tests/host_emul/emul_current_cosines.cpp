// TEST-ONLY host build of the cosine-binned face-current crossing step (walk_core.cuh, CU and MU, with and without TM
// and MO).
//
// The per-ray state machine of emul_face_currents.cpp with cosine bins, instantiated the way the MU kernels instantiate
// it: the exit scan's bden is handed to advance(), and 1 / |u| and the crossing's cosine bin sit in the lane's two slots
// after the weight.  The packed records, the internal order and the mesh centre are exported, so that the test can
// restate the cosine of every crossing from the stored normals.  Compiled by g++ without contraction; never linked into
// libpumitally.so.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "tet_mesh.hpp"
#include "walk_core.cuh"

using namespace ptb;

namespace {
struct CosineEmul {
  HostMesh mesh;
  std::vector<TetRecord> recs;
  std::vector<double> flux;  // [time][element][stride], internal order
  std::vector<double> cur;   // [time][cosine][element][4], internal order
  std::vector<double> edges, mu_edges;
  std::vector<ParticleState> state;
  DeviceStats stats{};
  int n = 0, stride = 1, nt = 0, nmu = 0;
  bool mo = false;

  template <bool TM, bool MO>
  void walk(const double *origin, const double *dest, const int8_t *flying, const double *weights, const double *times,
            const double *speeds) {
    CurrentWalkParams P{};
    P.tets = recs.data();
    P.flux = flux.data();
    P.state = state.data();
    P.origin = origin; P.dest = dest; P.flying = flying; P.weights = weights;
    P.begin = 0; P.end = n;
    P.max_iters = int32_t(mesh.ntets + 16);
    P.stats = &stats;
    P.cx = mesh.center[0]; P.cy = mesh.center[1]; P.cz = mesh.center[2];
    P.sc = ScoreParams{nullptr, 1, stride};
    P.tm = TimeParams{edges.data(), times, speeds, nt, int64_t(mesh.ntets) * stride};
    const int64_t E4 = int64_t(mesh.ntets) * 4;
    P.cu = CurrentParams{cur.data(), E4 * nmu, mu_edges.data(), nmu, E4};
    double wl[kMaxScores + 6];
    int32_t bin = 0;
    TimeLane tl;
    tl.responses = nullptr;
    tl.wl = wl;
    tl.n = 1;
    tl.stride = stride;
    tl.step = 1;
    tl.bin = &bin;
    for (int i = 0; i < n; ++i) {
      Counters c;
      Ray r;
      if (dest) begin_particle<kMaxScores, TM, MO, true, true>(P, i, r, c, true, &tl);
      else begin_particle(P, i, r, c, true);
      while (r.stage != kStageDone) {
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
          advance<false, false, kMaxScores, TM, MO, true, true>(P, i, r, exit_parameter(sc), sc.nbr, sc.back, c, true,
                                                                &tl, sc.bden);
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
// nedges == 0: no time filter; nmu_edges: 2..kMaxCosineBins + 1
void *ptb_cosines_create(const double *coords, int64_t nverts, const int32_t *t2v, int64_t ntets, int n,
                         const double *edges, int nedges, const double *mu_edges, int nmu_edges, int moments) {
  if (nedges == 1 || nedges - 1 > kMaxTimeBins || nmu_edges < 2 || nmu_edges - 1 > kMaxCosineBins) return nullptr;
  auto *e = new CosineEmul;
  std::string err;
  if (!e->mesh.from_arrays(coords, nverts, t2v, ntets, &err)) { delete e; return nullptr; }
  e->recs = e->mesh.records;
  e->n = n;
  e->mo = moments != 0;
  e->stride = e->mo ? kMomentSlots : 1;
  e->nt = nedges > 0 ? nedges - 1 : 0;
  e->nmu = nmu_edges - 1;
  if (nedges > 0) e->edges.assign(edges, edges + nedges);
  e->mu_edges.assign(mu_edges, mu_edges + nmu_edges);
  const size_t T = size_t(e->nt > 0 ? e->nt : 1);
  e->flux.assign(T * size_t(ntets) * size_t(e->stride), 0.0);
  e->cur.assign(T * size_t(e->nmu) * size_t(ntets) * 4, 0.0);
  e->state.assign(size_t(n), ParticleState{e->mesh.centroid0[0], e->mesh.centroid0[1], e->mesh.centroid0[2], e->mesh.start_elem, 0});
  return e;
}
void ptb_cosines_destroy(void *h) { delete static_cast<CosineEmul *>(h); }
void ptb_cosines_localize(void *h, const double *xyz) {
  static_cast<CosineEmul *>(h)->walk<false, false>(xyz, nullptr, nullptr, nullptr, nullptr, nullptr);
}
// times/speeds only with time bins
void ptb_cosines_move(void *h, const double *origin, const double *dest, int8_t *flying, const double *w,
                      const double *times, const double *speeds) {
  auto *e = static_cast<CosineEmul *>(h);
  if (e->nt > 0) {
    if (e->mo) e->walk<true, true>(origin, dest, flying, w, times, speeds);
    else e->walk<true, false>(origin, dest, flying, w, times, speeds);
  } else {
    if (e->mo) e->walk<false, true>(origin, dest, flying, w, nullptr, nullptr);
    else e->walk<false, false>(origin, dest, flying, w, nullptr, nullptr);
  }
  std::memset(flying, 0, size_t(e->n));
}
// out, in: [time][cosine][E][4] in the caller's numbering; elem, pos: particles
void ptb_cosines_get(void *h, double *out, double *in, int32_t *elem, double *pos) {
  auto *e = static_cast<CosineEmul *>(h);
  const int64_t E = e->mesh.ntets;
  const int A = (e->nt > 0 ? e->nt : 1) * e->nmu;
  const std::vector<int32_t> &t2t = e->mesh.t2t;
  for (int a = 0; a < A; ++a)
    for (int64_t i = 0; i < E; ++i)
      for (int f = 0; f < 4; ++f) {
        const int32_t nb = t2t[size_t(4 * i + f)];
        int back = f;
        if (nb >= 0)
          for (int q = 0; q < 4; ++q)
            if (t2t[4 * size_t(nb) + q] == int32_t(i)) back = q;
        const double *c = e->cur.data() + size_t(a) * size_t(E) * 4;
        const size_t o = (size_t(a) * size_t(E) + size_t(e->mesh.orig_of_internal[i])) * 4 + size_t(f);
        out[o] = nb >= 0 ? c[4 * size_t(nb) + size_t(back)] : c[4 * size_t(i) + size_t(f)];
        in[o] = nb >= 0 ? c[4 * size_t(i) + size_t(f)] : 0.0;
      }
  for (int i = 0; i < e->n; ++i) {
    elem[i] = e->mesh.orig_of_internal[e->state[i].elem];
    pos[3 * i] = e->state[i].x; pos[3 * i + 1] = e->state[i].y; pos[3 * i + 2] = e->state[i].z;
  }
}
// adj: [E][4] (adjacency_original)
void ptb_cosines_adjacency(void *h, int32_t *adj) {
  const std::vector<int32_t> a = static_cast<CosineEmul *>(h)->mesh.adjacency_original();
  std::memcpy(adj, a.data(), a.size() * sizeof(int32_t));
}
// recs: [E][16] packed records in the caller's numbering (the stored planes, payload bytes included)
void ptb_cosines_records(void *h, double *recs) {
  auto *e = static_cast<CosineEmul *>(h);
  for (int64_t i = 0; i < e->mesh.ntets; ++i)
    std::memcpy(recs + 16 * size_t(e->mesh.orig_of_internal[i]), e->recs[size_t(i)].d, 16 * sizeof(double));
}
}
