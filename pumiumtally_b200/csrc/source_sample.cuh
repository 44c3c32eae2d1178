// Mesh source (engine.cu, set_source / sample_source; source_kernels.cu): a table of per-element, per-group strengths,
// optionally biased, sampled by a CDF search, with a uniform point inside the chosen element.
//
// __host__ __device__ so that tests/ can compile the same arithmetic with g++ (tests/host_emul/emul_source.cpp).  Every
// product and sum of the point is rounded separately (no FMA): the device and the g++ build must agree bit for bit.
#pragma once
#include <cfloat>
#include <cstdint>

#include "walk_core.cuh"

namespace ptb {

// SplitMix64 of workload.py (_NumpyOps.uniform) at step 0: the mix of sample i's stream k.
constexpr uint64_t kSrcGold = 0x9E3779B97F4A7C15ull, kSrcM1 = 0xBF58476D1CE4E5B9ull, kSrcM2 = 0x94D049BB133111EBull,
                   kSrcStream = 0x8CB92BA72F3D8DD7ull;

PTB_HD uint64_t source_mix(uint64_t seed, uint64_t i, uint64_t stream) {
  uint64_t z = i * kSrcGold + (seed + stream * kSrcStream);
  z = (z ^ (z >> 30)) * kSrcM1;
  z = (z ^ (z >> 27)) * kSrcM2;
  return z ^ (z >> 31);
}

// The open interval (0, 1), exactly: ((z >> 12) + 0.5) * 2^-52 <= 1 - 2^-53.  (((z >> 11) + 0.5) * 2^-53 would round
// to 1.0 for the largest z.)
PTB_HD double source_uniform(uint64_t z) { return (double(z >> 12) + 0.5) * 0x1p-52; }

PTB_HD double src_add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
PTB_HD double src_sub(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
PTB_HD double src_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

// The entry of x = u_0 T: the first k with C[k] > x, or klast (the last k with p[k] > 0) when there is none because x
// rounded up to T.  An entry with p[k] == 0 has C[k] == C[k-1] and is never the first above x.
PTB_HD int64_t source_entry(const double *cdf, int64_t K, int64_t klast, double x) {
  int64_t lo = 0, hi = K;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (PTB_LDG(cdf + mid) > x) hi = mid;
    else lo = mid + 1;
  }
  return lo < K ? lo : klast;
}

// The Rocchini-Cignoni fold of (s, t, u) in the unit cube into the unit simplex s, t, u >= 0, s + t + u <= 1.
PTB_HD void source_fold(double &s, double &t, double &u) {
  if (src_add(s, t) > 1.0) {
    s = src_sub(1.0, s);
    t = src_sub(1.0, t);
  }
  if (src_add(t, u) > 1.0) {
    const double t0 = t;
    t = src_sub(1.0, u);
    u = src_sub(src_sub(1.0, s), t0);
  } else if (src_add(src_add(s, t), u) > 1.0) {
    const double s0 = s;
    s = src_sub(src_sub(1.0, t), u);
    u = src_sub(src_add(src_add(s0, t), u), 1.0);
  }
}

// v0 + ((s (v1 - v0) + t (v2 - v0)) + u (v3 - v0)) of one coordinate
PTB_HD double source_coord(double v0, double v1, double v2, double v3, double s, double t, double u) {
  return src_add(v0, src_add(src_add(src_mul(s, src_sub(v1, v0)), src_mul(t, src_sub(v2, v0))),
                             src_mul(u, src_sub(v3, v0))));
}

// The device copy of the source: K = ngroups * E entries k = g * E + e, e in the caller's numbering.
struct SourceTable {
  const double *cdf = nullptr;    // [K] C[k] = C[k-1] + p[k]
  const double *bias = nullptr;   // [K] b[k]; nullptr: unbiased (every weight 1)
  const double *verts = nullptr;  // [E][4][3] each element's vertices, the caller's local order
  int64_t K = 0, E = 0, klast = 0;
  double total = 0.0;             // T = C[K-1]
  double ratio = 1.0;             // T / Q
};

// Sample i (seed): entry k, point p, birth weight w.  Four uniforms u_0..u_3, streams 0..3.
PTB_HD void source_sample(const SourceTable &S, uint64_t seed, uint64_t i, int64_t &k, double p[3], double &w) {
  const double u0 = source_uniform(source_mix(seed, i, 0));
  k = source_entry(S.cdf, S.K, S.klast, u0 * S.total);
  double s = source_uniform(source_mix(seed, i, 1)), t = source_uniform(source_mix(seed, i, 2)),
         u = source_uniform(source_mix(seed, i, 3));
  source_fold(s, t, u);
  const int64_t e = k % S.E;
  const double *v = S.verts + 12 * e;
  double r[12];
#if defined(__CUDA_ARCH__)
  // 96 B per element, 16-byte aligned: six 128-bit loads of three sectors
PTB_UNROLL
  for (int q = 0; q < 6; ++q) {
    const double2 a = __ldg(reinterpret_cast<const double2 *>(v) + q);
    r[2 * q] = a.x;
    r[2 * q + 1] = a.y;
  }
#else
  for (int q = 0; q < 12; ++q) r[q] = v[q];
#endif
PTB_UNROLL
  for (int d = 0; d < 3; ++d) p[d] = source_coord(r[d], r[3 + d], r[6 + d], r[9 + d], s, t, u);
  w = S.bias ? S.ratio / PTB_LDG(S.bias + k) : 1.0;
}

// ---- host side of set_source (engine.cu and the g++ build share it) ----

// p[k] = (q[k] V[e] if per_volume else q[k]) * (b[k] if bias else 1), each product rounded separately; C is their
// sequential sum, T = C[K-1], *Q the same sum of the unbiased q V (or q), *klast the last k with p[k] > 0.  nullptr, or
// why the table is refused (with the offending entry in *bad, -1 for the totals); nothing is valid then.
inline const char *source_build(const double *q, const double *bias, const double *volume, int64_t E, int32_t ngroups,
                                bool per_volume, double *cdf, double *T, double *Q, int64_t *klast, int64_t *bad) {
  double c = 0.0, qs = 0.0;
  *klast = -1;
  *bad = -1;
  for (int64_t g = 0; g < ngroups; ++g)
    for (int64_t e = 0; e < E; ++e) {
      const int64_t k = g * E + e;
      *bad = k;
      if (!(q[k] >= 0.0 && q[k] <= DBL_MAX)) return "a strength is negative or not finite";
      if (bias && !(bias[k] >= 0.0 && bias[k] <= DBL_MAX))
        return "a bias is negative or not finite";
      if (bias && bias[k] == 0.0 && q[k] > 0.0) return "a bias is 0 where the strength is > 0";
      const double qv = per_volume ? q[k] * volume[e] : q[k];
      const double p = qv * (bias ? bias[k] : 1.0);
      if (p > 0.0) *klast = k;
      c += p;
      qs += qv;
      cdf[k] = c;
    }
  *bad = -1;
  *T = c;
  *Q = qs;
  if (!(c > 0.0 && c <= DBL_MAX)) return "the total (biased) strength is 0 or not finite";
  if (!(qs > 0.0 && qs <= DBL_MAX)) return "the total strength is 0 or not finite";
  return nullptr;
}

}  // namespace ptb
