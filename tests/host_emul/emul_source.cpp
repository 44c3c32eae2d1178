// TEST-ONLY host build of the mesh source (source_sample.cuh), the code source_kernels.cu runs per sample and
// set_source runs to build the table.  Compiled by g++ with -ffp-contract=off so that it can be checked against numpy
// bit for bit on a machine without a GPU; never linked into libpumitally.so.
#include <cstdint>

#include "source_sample.cuh"

extern "C" {
uint64_t ptb_src_mix(uint64_t seed, uint64_t i, uint64_t stream) { return ptb::source_mix(seed, i, stream); }
double ptb_src_uniform(uint64_t z) { return ptb::source_uniform(z); }
int64_t ptb_src_entry(const double *cdf, int64_t K, int64_t klast, double x) {
  return ptb::source_entry(cdf, K, klast, x);
}

// source_build: nullptr (ok) or the refusal; cdf [ngroups * E], out3 = (T, Q), out_k = (klast, bad)
const char *ptb_src_build(const double *q, const double *bias, const double *volume, int64_t E, int32_t ngroups,
                          int32_t per_volume, double *cdf, double *out2, int64_t *out_k) {
  return ptb::source_build(q, bias, volume, E, ngroups, per_volume != 0, cdf, &out2[0], &out2[1], &out_k[0], &out_k[1]);
}

// samples first .. first + n - 1 exactly as source_sample_kernel stores them; verts [E][4][3]
void ptb_src_sample(const double *cdf, const double *bias, const double *verts, int64_t K, int64_t E, int64_t klast,
                    double T, double Q, uint64_t seed, uint64_t first, int64_t n, double *xyz, int32_t *elem,
                    int32_t *group, double *weight) {
  ptb::SourceTable S;
  S.cdf = cdf;
  S.bias = bias;
  S.verts = verts;
  S.K = K;
  S.E = E;
  S.klast = klast;
  S.total = T;
  S.ratio = T / Q;
  for (int64_t j = 0; j < n; ++j) {
    int64_t k;
    double p[3], w;
    ptb::source_sample(S, seed, first + uint64_t(j), k, p, w);
    const int64_t g = k / E;
    for (int d = 0; d < 3; ++d) xyz[3 * j + d] = p[d];
    elem[j] = int32_t(k - g * E);
    group[j] = int32_t(g);
    weight[j] = w;
  }
}
}
