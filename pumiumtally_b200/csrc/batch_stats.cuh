// Batch statistics of the tally results (engine.cu, end_batch; stats_kernels.cu): a running mean and sum of squared
// deviations per result, folded one batch at a time by Welford's update.  Sum and sum of squares would cost the same
// memory traffic, but S2 - S1^2 / B cancels catastrophically when the relative error is small; Welford does not.
//
// __host__ __device__ so that tests/ can compile the same arithmetic with g++ (tests/host_emul/emul_batch_stats.cpp).
#pragma once
#include "walk_core.cuh"

#if !defined(__CUDACC__)
#include <cmath>
#endif
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

namespace ptb {

// Folds batch value x into (mean, m2) of the batches before it; nb is the number of batches including this one.
PTB_HD void welford_fold(double x, double nb, double &mean, double &m2) {
  const double d = x - mean;
  mean += d / nb;
  m2 += d * (x - mean);
}

// Combines the statistics (mean_b, m2_b) of nb batches into (mean, m2) of na other batches (Chan et al.'s parallel
// update): with n = na + nb and d = mean_b - mean, mean + d (nb / n) and m2 + m2_b + d^2 na nb / n.  An empty side
// gives the other side's values bit for bit (engine.cu, merge_checkpoint).
PTB_HD void welford_merge(double mean_b, double m2_b, double na, double nb, double &mean, double &m2) {
  const double n = na + nb, d = mean_b - mean;
  const double mu = mean + d * (nb / n), q = m2 + m2_b + d * d * (na * nb / n);
  mean = nb == 0.0 ? mean : na == 0.0 ? mean_b : mu;
  m2 = nb == 0.0 ? m2 : na == 0.0 ? m2_b : q;
}

// Standard error of the mean of nb >= 2 batches: sqrt(m2 / (nb (nb - 1))).
PTB_HD double batch_std_err(double m2, double nb) { return sqrt(m2 / (nb * (nb - 1.0))); }

// Relative error: std_err / |mean|, 0 where the mean is 0.
PTB_HD double batch_rel_err(double mean, double std_err) { return mean != 0.0 ? std_err / fabs(mean) : 0.0; }

// What pumitally_get_batch_results returns for one result of an element of volume `volume`: kind 0 the mean, 1 its
// standard error (both divided by the volume), 2 the relative error.
PTB_HD double batch_readout(double mean, double m2, double nb, double volume, int kind) {
  const double m = mean / volume;
  if (kind == 0) return m;
  const double s = batch_std_err(m2, nb) / volume;
  return kind == 1 ? s : batch_rel_err(m, s);
}

// ---- region sums (engine.cu, set_regions / get_region_results / end_batch; stats_kernels.cu, launch_region_sums) ----
// A region's sum is formed in levels.  Level 0 cuts the region's elements (ascending internal id) into chunks of at most
// kRegionChunk consecutive elements and sums each chunk left to right; every later level does the same to the region's
// chunk sums of the level before, until one sum per region is left.  The order depends on the region sizes only: the
// same tally always gives the same bits, and a one-element region's sum is its element's value itself.
constexpr int kRegionChunk = 32;

// Chunks a region of n inputs is cut into at one level; an empty region keeps one empty chunk, whose sum is 0.
PTB_HD int64_t region_chunks(int64_t n) { return n > kRegionChunk ? (n + kRegionChunk - 1) / kRegionChunk : 1; }

// acc[k] = x(0, k) + x(1, k) + ... + x(n - 1, k), left to right, for k < nscores: 0 for n == 0, x(0, k) for n == 1.
// (x is a device lambda in the kernel and a host one in region_sums_host)
#if defined(__CUDACC__)
#pragma nv_exec_check_disable
#endif
template <class F>
PTB_HD void chunk_sum(int64_t n, int nscores, F x, double (&acc)[kMaxScores]) {
  PTB_UNROLL
  for (int k = 0; k < kMaxScores; ++k) acc[k] = (k < nscores && n > 0) ? x(0, k) : 0.0;
  for (int64_t i = 1; i < n; ++i) {
    PTB_UNROLL
    for (int k = 0; k < kMaxScores; ++k)
      if (k < nscores) acc[k] += x(i, k);
  }
}

// One level of the plan: its chunk c covers inputs [starts[start_off + c], starts[start_off + c + 1]).
struct RegionLevel {
  int64_t start_off;  // first of its chunks + 1 entries in RegionPlan::starts
  int64_t chunks;     // the last level has one chunk per region, in region order
  int64_t inputs;     // level 0: the elements in a region; later levels: the chunks of the level before
};

struct RegionPlan {
  std::vector<int32_t> elems;   // level 0's inputs: internal element ids, ascending region, then ascending id
  std::vector<int32_t> starts;  // every level's chunk starts
  std::vector<RegionLevel> levels;
};

// Cuts p.elems, already grouped (group g holds n[g] consecutive inputs, in group order), into the plan's levels.
inline void cut_region_levels(std::vector<int64_t> n, RegionPlan &p) {
  for (bool done = false; !done;) {
    RegionLevel l{int64_t(p.starts.size()), 0, 0};
    done = true;
    for (int64_t &m : n) {
      const int64_t c = region_chunks(m);
      for (int64_t j = 0; j < c; ++j) p.starts.push_back(int32_t(l.inputs + std::min<int64_t>(j * kRegionChunk, m)));
      l.inputs += m;
      l.chunks += c;
      m = c;
      done = done && c == 1;
    }
    p.starts.push_back(int32_t(l.inputs));
    p.levels.push_back(l);
  }
}

// The plan of region_of_internal[e] in [-1, nregions) for e < E (-1: in no region).
inline RegionPlan build_region_plan(const int32_t *region_of_internal, int64_t E, int32_t nregions) {
  RegionPlan p;
  std::vector<int64_t> n(size_t(nregions), 0), off(size_t(nregions) + 1, 0);
  for (int64_t e = 0; e < E; ++e)
    if (region_of_internal[e] >= 0) ++n[size_t(region_of_internal[e])];
  for (size_t g = 0; g < n.size(); ++g) off[g + 1] = off[g] + n[g];
  p.elems.resize(size_t(off.back()));
  for (int64_t e = 0; e < E; ++e)  // ascending id within each region
    if (region_of_internal[e] >= 0) p.elems[size_t(off[size_t(region_of_internal[e])]++)] = int32_t(e);
  cut_region_levels(std::move(n), p);
  return p;
}

// Doubles of the scratch launch_region_sums needs for narrays arrays of nscores results: two buffers of the largest
// level output before the last.
inline int64_t region_scratch_len(const RegionPlan &p, int64_t narrays, int32_t nscores) {
  int64_t m = 0;
  for (size_t l = 0; l + 1 < p.levels.size(); ++l) m = std::max(m, p.levels[l].chunks);
  return 2 * m * narrays * nscores;
}

// The region sums of one value per element, values[internal id], in the order above: what launch_region_sums computes,
// on the host (the region volumes; tests/host_emul/emul_regions.cpp).
inline std::vector<double> region_sums_host(const RegionPlan &p, const double *values) {
  std::vector<double> in, out;
  for (size_t l = 0; l < p.levels.size(); ++l) {
    const RegionLevel &v = p.levels[l];
    out.assign(size_t(v.chunks), 0.0);
    for (int64_t c = 0; c < v.chunks; ++c) {
      const int32_t lo = p.starts[size_t(v.start_off + c)], hi = p.starts[size_t(v.start_off + c + 1)];
      double acc[kMaxScores];
      chunk_sum(hi - lo, 1, [&](int64_t i, int) { return l == 0 ? values[p.elems[size_t(lo + i)]] : in[size_t(lo + i)]; },
                acc);
      out[size_t(c)] = acc[0];
    }
    in.swap(out);
  }
  return in;
}

// ---- region currents (engine.cu, set_region_currents / get_region_current_results / end_batch) ----
// The face-current slots (walk_core.cuh, CurrentParams) grouped by ordered pair of regions.  Slot 4 n + b holds the
// weight entering element n through its face b; a hull slot 4 e + f holds the weight leaving e through f.  With reg()
// the region of an element, -1 for none and kOutside for outside the mesh: the interior slot 4 n + b, across from
// element e, belongs to pair reg(e) -> reg(n) when the two differ (and to no pair when they are equal); the hull slot
// 4 e + f belongs to pair reg(e) -> kOutside.  The pairs with at least one slot are listed in ascending (from, to)
// order as signed integers.  A pair's partial current is the sum of its slots in the RegionPlan order (its slots
// ascending, in chunks of kRegionChunk, level by level), its net current that minus the partial of the reverse pair.
constexpr int32_t kOutside = -2;

struct RegionCurrentPlan {
  RegionPlan sums;                 // elems: the slots, ascending pair, then ascending slot
  std::vector<int64_t> first;      // [P + 1] pair p's slots are sums.elems[first[p], first[p + 1])
  std::vector<int32_t> from, to;   // [P] the pairs
  std::vector<int32_t> rev;        // [P] the pair to -> from, -1 when there is none (always for to == kOutside)
  std::vector<double> area;        // [P] the pair's slot areas summed in the plan's order
};

// The area of face f (opposite local vertex f) of element e, from its three other vertices a, b, c in local order:
// |(b - a) x (c - a)| / 2, every operation rounded separately.
inline double face_area(const double *coords, const int32_t *t2v, int64_t e, int f) {
  const double *v[3];
  for (int q = 0, j = 0; q < 4; ++q)
    if (q != f) v[j++] = coords + 3 * int64_t(t2v[4 * e + q]);
  const double u0 = v[1][0] - v[0][0], u1 = v[1][1] - v[0][1], u2 = v[1][2] - v[0][2];
  const double w0 = v[2][0] - v[0][0], w1 = v[2][1] - v[0][1], w2 = v[2][2] - v[0][2];
  const double x = u1 * w2 - u2 * w1, y = u2 * w0 - u0 * w2, z = u0 * w1 - u1 * w0;
  const double s = x * x + y * y;
  return sqrt(s + z * z) * 0.5;
}

// The plan of region_of_internal[e] in [-1, nregions) for e < E, with t2t [4E] the neighbour across each face (-1 on
// the hull) and slot_area [4E] the area of each slot's face.  Needs 4E <= INT32_MAX (slot ids are int32).
inline RegionCurrentPlan build_region_current_plan(const int32_t *region_of_internal, const int32_t *t2t, int64_t E,
                                                   const double *slot_area) {
  RegionCurrentPlan p;
  // (pair key, slot) of every slot in a pair; the key orders (from, to) as signed integers
  auto key = [](int32_t a, int32_t b) { return int64_t(a) * (int64_t(1) << 32) + int64_t(uint32_t(b) ^ 0x80000000u); };
  std::vector<std::pair<int64_t, int32_t>> ks;
  for (int64_t e = 0; e < E; ++e)
    for (int f = 0; f < 4; ++f) {
      const int32_t nb = t2t[4 * e + f], a = region_of_internal[e];
      if (nb < 0) {
        ks.emplace_back(key(a, kOutside), int32_t(4 * e + f));
        continue;
      }
      const int32_t b = region_of_internal[nb];
      if (a == b) continue;
      int back = 0;
      for (int q = 0; q < 4; ++q)
        if (t2t[4 * int64_t(nb) + q] == int32_t(e)) back = q;
      ks.emplace_back(key(a, b), int32_t(4 * int64_t(nb) + back));  // e -> nb enters nb through its face back
    }
  std::sort(ks.begin(), ks.end());
  std::vector<int64_t> n;
  p.sums.elems.resize(ks.size());
  for (size_t i = 0; i < ks.size(); ++i) {
    if (i == 0 || ks[i].first != ks[i - 1].first) {
      n.push_back(0);
      p.from.push_back(int32_t(ks[i].first >> 32));
      p.to.push_back(int32_t(uint32_t(ks[i].first) ^ 0x80000000u));
    }
    ++n.back();
    p.sums.elems[i] = ks[i].second;
  }
  p.first.assign(1, 0);
  for (int64_t m : n) p.first.push_back(p.first.back() + m);
  cut_region_levels(std::move(n), p.sums);
  const size_t P = p.from.size();
  p.rev.assign(P, -1);
  for (size_t q = 0; q < P; ++q) {
    const int32_t a = p.to[q], b = p.from[q];  // the reverse pair, found by binary search in the sorted list
    size_t lo = 0, hi = P;
    while (lo < hi) {
      const size_t m = (lo + hi) / 2;
      if (key(p.from[m], p.to[m]) < key(a, b)) lo = m + 1; else hi = m;
    }
    if (lo < P && p.from[lo] == a && p.to[lo] == b) p.rev[q] = int32_t(lo);
  }
  p.area = region_sums_host(p.sums, slot_area);
  return p;
}

}  // namespace ptb
