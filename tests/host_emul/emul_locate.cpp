// TEST-ONLY host build of the point-location step (walk_core.cuh, locate_point).
//
// The seed grid is built as Engine::build_seed_grid() builds it (every seed point localised from the centroid of
// element 0 by the walk, a cell keeps the tet where its point was reached) and the candidate lists by the engine's own
// cell_candidates() (seed_grid.hpp).  Compiled by g++ so that point location can be checked against a brute-force
// reference on a machine without a GPU; never linked into libpumitally.so.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "seed_grid.hpp"
#include "tet_mesh.hpp"
#include "walk_core.cuh"

using namespace ptb;

namespace {
struct LocateEmul {
  HostMesh mesh;
  std::vector<TetRecord> recs;
  SeedGrid grid{};
  std::vector<int32_t> cell_tet;
  std::vector<int64_t> cand_off;
  std::vector<int32_t> cand;
  double extent = 0.0;

  void build() {
    recs = mesh.records;
    grid = choose_seed_grid(mesh);
    const int nc = grid.nx * grid.ny * grid.nz;
    std::vector<double> xyz(3 * size_t(nc)), flux(size_t(mesh.ntets), 0.0);
    std::vector<ParticleState> ts(nc, ParticleState{mesh.centroid0[0], mesh.centroid0[1], mesh.centroid0[2], mesh.start_elem, 0});
    for (int i = 0; i < nc; ++i)
      seed_point(grid, i % grid.nx, (i / grid.nx) % grid.ny, i / (grid.nx * grid.ny), xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    DeviceStats st{};
    WalkParams P{};
    P.tets = recs.data();
    P.flux = flux.data();
    P.state = ts.data();
    P.origin = xyz.data();
    P.begin = 0; P.end = nc;
    P.max_iters = int32_t(mesh.ntets + 16);
    P.stats = &st;
    P.cx = mesh.center[0]; P.cy = mesh.center[1]; P.cz = mesh.center[2];
    for (int i = 0; i < nc; ++i) {
      Counters c;
      Ray r;
      begin_particle(P, i, r, c, true);
      while (r.stage != kStageDone) {
        ExitScan sc;
        double raw[16];
        std::memcpy(raw, recs[r.e].d, sizeof(raw));
        scan_record(raw, r.e, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz, sc);
        advance(P, i, r, exit_parameter(sc), sc.nbr, sc.back, c, true);
      }
    }
    cell_tet.resize(nc);
    for (int i = 0; i < nc; ++i)
      cell_tet[i] = (ts[i].x == xyz[3 * i] && ts[i].y == xyz[3 * i + 1] && ts[i].z == xyz[3 * i + 2]) ? ts[i].elem : -1;
    grid.cell_tet = cell_tet.data();
    extent = std::max({mesh.bbox_hi[0] - mesh.bbox_lo[0], mesh.bbox_hi[1] - mesh.bbox_lo[1], mesh.bbox_hi[2] - mesh.bbox_lo[2]});
    // built on every mesh here so that its completeness can be checked; the walk uses it on non-convex hulls only,
    // as the engine does
    cell_candidates(mesh, grid, kLocateBand * extent, &cand_off, &cand);
  }

  LocateParams params() const {
    LocateParams p{};
    p.tets = recs.data();
    p.grid = grid;
    p.max_iters = int32_t(mesh.ntets + 16);
    p.cx = mesh.center[0]; p.cy = mesh.center[1]; p.cz = mesh.center[2];
    p.sx = mesh.centroid0[0]; p.sy = mesh.centroid0[1]; p.sz = mesh.centroid0[2];
    p.start_elem = mesh.start_elem;
    p.convex = mesh.hull_convex ? 1 : 0;
    p.cand_off = mesh.hull_convex ? nullptr : cand_off.data();
    p.cand = mesh.hull_convex ? nullptr : cand.data();
    p.slack = kLocateSlack * extent;
    return p;
  }
};
}  // namespace

extern "C" {
void *ptb_locate_create(const double *coords, int64_t nverts, const int32_t *t2v, int64_t ntets) {
  auto *e = new LocateEmul;
  std::string err;
  if (!e->mesh.from_arrays(coords, nverts, t2v, ntets, &err)) { delete e; return nullptr; }
  e->build();
  return e;
}
void ptb_locate_destroy(void *h) { delete static_cast<LocateEmul *>(h); }
int ptb_locate_hull_convex(void *h) { return static_cast<LocateEmul *>(h)->mesh.hull_convex ? 1 : 0; }
// element (caller's numbering) of each point, -1 outside
void ptb_locate_points(void *h, const double *xyz, int64_t n, int32_t *out) {
  auto *e = static_cast<LocateEmul *>(h);
  const LocateParams P = e->params();
  auto fetch = [&](int32_t t, double (&r)[16]) { std::memcpy(r, e->recs[t].d, sizeof(r)); };
  for (int64_t i = 0; i < n; ++i) {
    const int32_t t = locate_point(P, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], fetch);
    out[i] = t >= 0 ? e->mesh.orig_of_internal[t] : -1;
  }
}
// grid: dims[3] = nx, ny, nz; geom[5] = x0, y0, z0, h, inv_h; returns the number of candidate entries
int64_t ptb_locate_grid(void *h, int32_t *dims, double *geom) {
  auto *e = static_cast<LocateEmul *>(h);
  dims[0] = e->grid.nx; dims[1] = e->grid.ny; dims[2] = e->grid.nz;
  geom[0] = e->grid.x0; geom[1] = e->grid.y0; geom[2] = e->grid.z0; geom[3] = e->grid.h; geom[4] = e->grid.inv_h;
  return int64_t(e->cand.size());
}
// the candidate lists, tets in the caller's numbering
void ptb_locate_candidates(void *h, int64_t *off, int32_t *tets) {
  auto *e = static_cast<LocateEmul *>(h);
  std::memcpy(off, e->cand_off.data(), e->cand_off.size() * sizeof(int64_t));
  for (size_t k = 0; k < e->cand.size(); ++k) tets[k] = e->mesh.orig_of_internal[e->cand[k]];
}
}
