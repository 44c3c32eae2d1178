// TEST-ONLY host build of the detector void (walk_core.cuh, detector_event<true> / detector_ray<true> / hull_entry)
// behind the point location of the events (locate_point, with the seed grid and candidate lists emul_locate.cpp builds
// as the engine does) and the engine's own hull grid (seed_grid.hpp, hull_grid).  Compiled by g++ so that the void
// mode can be checked against a numpy reference on a machine without a GPU; never linked into libpumitally.so.
#include "emul_locate.cpp"

extern "C" {
// As ptb_detect (emul_detectors.cpp) with the void on: counts[8], the last the hull entries.
void ptb_detect_void(void *h, const double *xyz, int64_t n, const double *w, const double *pdf, const double *resp,
                     const int32_t *bins, const double *times, const double *speeds, int32_t nscores, int32_t nbins,
                     const double *edges, int32_t nt, const double *sigma, const double *det, int32_t ndet,
                     const double *r0, int32_t max_iters, double *out, uint64_t *counts) {
  auto *e = static_cast<LocateEmul *>(h);
  LocateParams L = e->params();
  if (max_iters > 0) L.max_iters = max_iters;
  auto fetch = [&](int32_t t, double (&r)[16]) { std::memcpy(r, e->recs[t].d, sizeof(r)); };
  std::vector<int64_t> hoff;
  std::vector<int32_t> htets;
  HullGrid H = hull_grid(e->mesh, e->grid, kLocateBand * e->extent, &hoff, &htets);
  H.off = hoff.data();
  H.tets = htets.data();
  const int64_t E = e->mesh.ntets;
  std::vector<double> sig(size_t(nbins) * E);
  for (int64_t b = 0; b < nbins; ++b)
    for (int64_t i = 0; i < E; ++i) sig[b * E + i] = sigma[b * E + e->mesh.orig_of_internal[i]];
  const int T = nt > 0 ? nt : 1;
  std::fill(out, out + size_t(T) * nbins * nscores * ndet, 0.0);
  DetectorParams P{};
  P.tally = out;
  P.sigma = sig.data();
  P.pos = det;
  P.r0 = r0;
  P.edges = edges;
  P.nt = nt;
  P.nbins = nbins;
  P.nscores = nscores;
  P.ndet = ndet;
  P.zero_r0 = std::count(r0, r0 + ndet, 0.0) > 0 ? 1 : 0;
  P.E = E;
  for (int c = 0; c < 8; ++c) counts[c] = 0;
  for (int d = 0; d < ndet; ++d)
    for (int64_t i = 0; i < n; ++i) {
      const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
      const int32_t el = locate_point(L, x, y, z, fetch);
      double val[kMaxScores];
      int64_t slot = 0;
      uint32_t cross = 0, entries = 0;
      const int o = detector_event<true>(L, P, d, el, x, y, z, w[i], resp ? resp + i * nscores : nullptr,
                                         bins ? bins[i] : 0, nt > 0 ? times[i] : 0.0, nt > 0 ? speeds[i] : 1.0,
                                         pdf ? pdf + i * ndet : nullptr, val, &slot, cross, fetch, &H, &entries);
      counts[4] += cross;
      counts[7] += entries;
      if (o == kRayTraced || o == kRayInsideR0)
        for (int k = 0; k < nscores; ++k) out[slot + int64_t(k) * ndet] += val[k];
      if (o <= kRayInsideR0) ++counts[o == kRayInsideR0 ? 3 : o];
      else if (o == kDetOutside && d == 0) ++counts[5];
      else if (o == kDetRejected && d == 0) ++counts[6];
    }
}

// Entries of the hull-tet lists, and how many tets have a face on the hull.
int64_t ptb_hull_candidates(void *h, int64_t *nhull) {
  auto *e = static_cast<LocateEmul *>(h);
  std::vector<int64_t> off;
  std::vector<int32_t> tets;
  hull_grid(e->mesh, e->grid, kLocateBand * e->extent, &off, &tets);
  const std::vector<uint8_t> keep = hull_tets(e->mesh);
  *nhull = std::count(keep.begin(), keep.end(), uint8_t(1));
  return int64_t(tets.size());
}
}
