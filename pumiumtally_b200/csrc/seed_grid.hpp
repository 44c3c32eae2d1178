// Geometry of the relocation seed grid (see SeedGrid in walk_core.cuh).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <utility>
#include <vector>

#include "tet_mesh.hpp"
#include "walk_core.cuh"

namespace ptb {

// Roughly one grid cell per `tets_per_cell` tets, cubic cells, at most 1024 per axis.  The target is at most 2^24
// cells, but rounding each axis up can exceed it: a cube at the cap gets 257^3 = 16 974 593 cells, a 1000 x 1000 x
// 15.63 slab 1024 x 1024 x 17 = 17 825 792 (the binning tests run both).
// cell_tet is left null; the caller fills the table by localising the seed points.
inline SeedGrid choose_seed_grid(const HostMesh &m, double tets_per_cell = 4.0) {
  SeedGrid g{};
  const double lx = m.bbox_hi[0] - m.bbox_lo[0], ly = m.bbox_hi[1] - m.bbox_lo[1],
               lz = m.bbox_hi[2] - m.bbox_lo[2];
  const double vol = std::max(lx * ly * lz, 1e-300);
  double cells = std::min(std::max(double(m.ntets) / tets_per_cell, 1.0), double(1 << 24));
  double h = std::cbrt(vol / cells);
  auto dim = [&](double l) { return int32_t(std::min(std::max(std::ceil(l / h), 1.0), 1024.0)); };
  g.nx = dim(lx); g.ny = dim(ly); g.nz = dim(lz);
  // grow h if the 1024 clamp cut an axis short, so the grid still covers the box
  h = std::max({h, lx / g.nx, ly / g.ny, lz / g.nz});
  g.h = h;
  g.inv_h = 1.0 / h;
  g.x0 = m.bbox_lo[0]; g.y0 = m.bbox_lo[1]; g.z0 = m.bbox_lo[2];
  g.far2 = 4.0 * h * h;  // seed when the target is more than two cells away
  g.cell_tet = nullptr;
  return g;
}

// Rank of every grid cell along the Morton (Z-order) curve through the cells that exist: the
// binning pass sorts particles by this rank, so a run of consecutive particles covers a compact
// 3-D block of the mesh instead of a one-cell-thick slab (smaller L2 working set per window).
inline std::vector<int32_t> morton_cell_ranks(const SeedGrid &g) {
  auto spread = [](uint64_t v) {  // 21 bits -> every third bit
    v &= 0x1fffff;
    v = (v | v << 32) & 0x1f00000000ffffull;
    v = (v | v << 16) & 0x1f0000ff0000ffull;
    v = (v | v << 8) & 0x100f00f00f00f00full;
    v = (v | v << 4) & 0x10c30c30c30c30c3ull;
    v = (v | v << 2) & 0x1249249249249249ull;
    return v;
  };
  const int64_t n = int64_t(g.nx) * g.ny * g.nz;
  std::vector<std::pair<uint64_t, int32_t>> key(static_cast<size_t>(n));
  for (int cz = 0; cz < g.nz; ++cz)
    for (int cy = 0; cy < g.ny; ++cy)
      for (int cx = 0; cx < g.nx; ++cx) {
        const int32_t c = (cz * g.ny + cy) * g.nx + cx;
        key[c] = {spread(cx) | spread(cy) << 1 | spread(cz) << 2, c};
      }
  std::sort(key.begin(), key.end());
  std::vector<int32_t> rank(static_cast<size_t>(n));
  for (int64_t r = 0; r < n; ++r) rank[key[r].second] = int32_t(r);
  return rank;
}

// Candidate tets of every grid cell for point location on a non-convex hull (locate_point in walk_core.cuh): CSR
// lists, off[c] .. off[c + 1] of `tets` hold the internal ids of the tets whose bounding box, widened by `pad`,
// overlaps cell c (closed intervals).  A tet that contains a point of the cell is therefore in the cell's list.
inline void cell_candidates(const HostMesh &m, const SeedGrid &g, double pad, std::vector<int64_t> *off,
                            std::vector<int32_t> *tets) {
  const int64_t ncell = int64_t(g.nx) * g.ny * g.nz;
  const int n[3] = {g.nx, g.ny, g.nz};
  const double lo[3] = {g.x0, g.y0, g.z0};
  auto range = [&](int64_t e, int lo_c[3], int hi_c[3]) {
    for (int d = 0; d < 3; ++d) {
      double a = m.coords[3 * size_t(m.t2v[4 * e]) + d], b = a;
      for (int q = 1; q < 4; ++q) {
        const double v = m.coords[3 * size_t(m.t2v[4 * e + q]) + d];
        a = std::min(a, v);
        b = std::max(b, v);
      }
      // cell k covers [lo + k h, lo + (k + 1) h]
      const double fa = std::floor((a - pad - lo[d]) * g.inv_h) - 1.0, fb = std::floor((b + pad - lo[d]) * g.inv_h) + 1.0;
      lo_c[d] = int(std::min(std::max(fa, 0.0), double(n[d] - 1)));
      hi_c[d] = int(std::min(std::max(fb, 0.0), double(n[d] - 1)));
      // trim the one-cell margin the floor above leaves for rounding, keeping every cell that overlaps
      while (lo_c[d] < hi_c[d] && lo[d] + (lo_c[d] + 1) * g.h < a - pad) ++lo_c[d];
      while (hi_c[d] > lo_c[d] && lo[d] + hi_c[d] * g.h > b + pad) --hi_c[d];
    }
  };
  off->assign(size_t(ncell) + 1, 0);
  for (int64_t e = 0; e < m.ntets; ++e) {
    int a[3], b[3];
    range(e, a, b);
    for (int z = a[2]; z <= b[2]; ++z)
      for (int y = a[1]; y <= b[1]; ++y)
        for (int x = a[0]; x <= b[0]; ++x) ++(*off)[size_t((int64_t(z) * g.ny + y) * g.nx + x) + 1];
  }
  for (int64_t c = 0; c < ncell; ++c) (*off)[size_t(c) + 1] += (*off)[size_t(c)];
  tets->resize(size_t((*off)[size_t(ncell)]));
  std::vector<int64_t> cur(off->begin(), off->end() - 1);
  for (int64_t e = 0; e < m.ntets; ++e) {
    int a[3], b[3];
    range(e, a, b);
    for (int z = a[2]; z <= b[2]; ++z)
      for (int y = a[1]; y <= b[1]; ++y)
        for (int x = a[0]; x <= b[0]; ++x) (*tets)[size_t(cur[size_t((int64_t(z) * g.ny + y) * g.nx + x)]++)] = int32_t(e);
  }
}

}  // namespace ptb
