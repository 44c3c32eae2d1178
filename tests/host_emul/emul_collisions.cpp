// TEST-ONLY host build of the collision estimator's per-event step (walk_core.cuh, collision_event) behind the point
// location of the located events (locate_point, with the seed grid and candidate lists emul_locate.cpp builds as the
// engine does).  Compiled by g++ so that the event rules can be checked against a numpy reference on a machine without a
// GPU; never linked into libpumitally.so.
#include "emul_locate.cpp"

extern "C" {
// The mesh centre C the moments are accumulated about.
void ptb_collide_centre(void *h, double *c) {
  auto *e = static_cast<LocateEmul *>(h);
  for (int a = 0; a < 3; ++a) c[a] = e->mesh.center[a];
}

// n located events into a fresh collision tally of nt time bins (0: none; edges[nt + 1]), nbins score bins and nscores
// scores, with moments or not.  m0 [T][B][S][E] and R [T][B][S][E][3] (first moment about C) in the caller's element
// numbering, T = max(nt, 1); counts[3] = events tallied, outside, rejected.  resp, bins and times may be nullptr.
void ptb_collide(void *h, const double *xyz, int64_t n, const double *w, const double *resp, const int32_t *bins,
                 const double *times, int32_t nscores, int32_t nbins, const double *edges, int32_t nt, int32_t moments,
                 double *m0, double *R, uint64_t *counts) {
  auto *e = static_cast<LocateEmul *>(h);
  const LocateParams L = e->params();
  auto fetch = [&](int32_t t, double (&r)[16]) { std::memcpy(r, e->recs[t].d, sizeof(r)); };
  const int64_t E = e->mesh.ntets;
  const int T = nt > 0 ? nt : 1, S = score_stride(nscores), stride = S * (moments ? kMomentSlots : 1);
  std::vector<double> flux(size_t(T) * nbins * E * stride, 0.0);
  CollisionParams P{};
  P.flux = flux.data();
  P.edges = edges;
  P.nt = nt;
  P.nbins = nbins;
  P.nscores = nscores;
  P.stride = stride;
  P.moments = moments;
  P.bin_stride = E * stride;
  P.slice = int64_t(nbins) * E * stride;
  P.cx = e->mesh.center[0]; P.cy = e->mesh.center[1]; P.cz = e->mesh.center[2];
  counts[0] = counts[1] = counts[2] = 0;
  for (int64_t i = 0; i < n; ++i) {
    const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const int32_t el = locate_point(L, x, y, z, fetch);
    const int c = collision_event(P, el, x, y, z, w[i], resp ? resp + i * nscores : nullptr, bins ? bins[i] : 0,
                                  nt > 0 ? times[i] : 0.0);
    if (c < 3) ++counts[c];
  }
  for (int j = 0; j < T; ++j)
    for (int b = 0; b < nbins; ++b)
      for (int64_t t = 0; t < E; ++t) {
        const double *f = flux.data() + ((size_t(j) * nbins + b) * E + t) * stride;
        const int64_t o = e->mesh.orig_of_internal[t];
        for (int k = 0; k < nscores; ++k) {
          const size_t q = ((size_t(j) * nbins + b) * nscores + k) * E + o;
          m0[q] = f[k];
          for (int a = 0; a < 3; ++a) R[3 * q + a] = moments ? f[(a + 1) * S + k] : 0.0;
        }
      }
}
}
