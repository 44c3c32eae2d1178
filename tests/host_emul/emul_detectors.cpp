// TEST-ONLY host build of the point detectors' per-ray step (walk_core.cuh, detector_event / detector_ray) behind the
// point location of the events (locate_point, with the seed grid and candidate lists emul_locate.cpp builds as the engine
// does).  Compiled by g++ so that the scoring, the walk to the detector and the outcome ranking can be checked against
// a numpy reference on a machine without a GPU; never linked into libpumitally.so.
#include "emul_locate.cpp"

extern "C" {
// n located events scored at ndet detectors (det [3 ndet], r0 [ndet]) through Sigma_t sigma [nbins][E] (caller's
// numbering), with nt time bins (0: none; edges [nt + 1]).  out [T][nbins][nscores][ndet], T = max(nt, 1); counts[7]
// as the kernels count them (walk_kernels.hpp, kDetCount*).  pdf, resp, bins, times and speeds may be nullptr.
void ptb_detect(void *h, const double *xyz, int64_t n, const double *w, const double *pdf, const double *resp,
                const int32_t *bins, const double *times, const double *speeds, int32_t nscores, int32_t nbins,
                const double *edges, int32_t nt, const double *sigma, const double *det, int32_t ndet, const double *r0,
                double *out, uint64_t *counts) {
  auto *e = static_cast<LocateEmul *>(h);
  const LocateParams L = e->params();
  auto fetch = [&](int32_t t, double (&r)[16]) { std::memcpy(r, e->recs[t].d, sizeof(r)); };
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
  for (int c = 0; c < 7; ++c) counts[c] = 0;
  for (int d = 0; d < ndet; ++d)
    for (int64_t i = 0; i < n; ++i) {
      const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
      const int32_t el = locate_point(L, x, y, z, fetch);
      double val[kMaxScores];
      int64_t slot = 0;
      uint32_t cross = 0;
      const int o = detector_event(L, P, d, el, x, y, z, w[i], resp ? resp + i * nscores : nullptr, bins ? bins[i] : 0,
                                   nt > 0 ? times[i] : 0.0, nt > 0 ? speeds[i] : 1.0,
                                   pdf ? pdf + i * ndet : nullptr, val, &slot, cross, fetch);
      counts[4] += cross;
      if (o == kRayTraced || o == kRayInsideR0)
        for (int k = 0; k < nscores; ++k) out[slot + int64_t(k) * ndet] += val[k];
      if (o <= kRayInsideR0) ++counts[o == kRayInsideR0 ? 3 : o];
      else if (o == kDetOutside && d == 0) ++counts[5];
      else if (o == kDetRejected && d == 0) ++counts[6];
    }
}

double ptb_ball_g(double x) { return ball_g(x); }
}
