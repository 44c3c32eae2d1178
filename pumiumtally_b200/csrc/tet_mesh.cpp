// Host-side mesh preparation: generators, raw-file reader, face adjacency,
// volumes and the packed 128-byte tet records the walk kernels consume.
#include "tet_mesh.hpp"

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <utility>
#include <sys/stat.h>

namespace ptb {

namespace {

inline void sort3(int32_t &a, int32_t &b, int32_t &c) {
  if (a > b) std::swap(a, b);
  if (b > c) std::swap(b, c);
  if (a > b) std::swap(a, b);
}

inline uint64_t dbits(double x) {
  uint64_t u;
  std::memcpy(&u, &x, 8);
  return u;
}
inline double bdouble(uint64_t u) {
  double x;
  std::memcpy(&x, &u, 8);
  return x;
}

struct FaceKey {
  int32_t a, b, c;
  int32_t slot;  // 4*tet + face
  bool operator<(const FaceKey &o) const {
    if (a != o.a) return a < o.a;
    if (b != o.b) return b < o.b;
    return c < o.c;
  }
  bool same(const FaceKey &o) const { return a == o.a && b == o.b && c == o.c; }
};

}  // namespace

// Hex corner numbering and the six tets around the 0-6 diagonal; local element
// k takes entry (k+1)%6 of the cyclic list so that element 0 is {y>=x>=z}, the
// ordering the reference's known-answer test pins for Omega_h::build_box
// (test/test_pumi_tally_impl_methods.cpp:34-35, 83).
void build_kuhn_box(int nx, int ny, int nz, double lx, double ly, double lz,
                    std::vector<double> *coords, std::vector<int32_t> *t2v) {
  static const int corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0},
                                   {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
  static const int cyc[6][4] = {{0, 1, 2, 6}, {0, 2, 3, 6}, {0, 3, 7, 6},
                                {0, 7, 4, 6}, {0, 4, 5, 6}, {0, 5, 1, 6}};
  const int64_t nvx = nx + 1, nvy = ny + 1, nvz = nz + 1;
  coords->resize(3 * nvx * nvy * nvz);
  for (int64_t k = 0; k < nvz; ++k)
    for (int64_t j = 0; j < nvy; ++j)
      for (int64_t i = 0; i < nvx; ++i) {
        int64_t v = (k * nvy + j) * nvx + i;
        (*coords)[3 * v + 0] = (i == nx) ? lx : double(i) * (lx / nx);
        (*coords)[3 * v + 1] = (j == ny) ? ly : double(j) * (ly / ny);
        (*coords)[3 * v + 2] = (k == nz) ? lz : double(k) * (lz / nz);
      }
  t2v->resize(size_t(24) * nx * ny * nz);
  size_t w = 0;
  for (int64_t k = 0; k < nz; ++k)
    for (int64_t j = 0; j < ny; ++j)
      for (int64_t i = 0; i < nx; ++i) {
        int32_t c[8];
        for (int q = 0; q < 8; ++q)
          c[q] = int32_t(((k + corner[q][2]) * nvy + (j + corner[q][1])) * nvx + (i + corner[q][0]));
        for (int t = 0; t < 6; ++t) {
          const int *tt = cyc[(t + 1) % 6];
          for (int q = 0; q < 4; ++q) (*t2v)[w++] = c[tt[q]];
        }
      }
}

bool read_raw_mesh(const std::string &path, std::vector<double> *coords,
                   std::vector<int32_t> *t2v, std::string *err) {
  std::ifstream f(path, std::ios::binary);
  if (!f) { *err = "cannot open " + path; return false; }
  char magic[8];
  f.read(magic, 8);
  if (!f || std::memcmp(magic, "PUMITB2\0", 8) != 0) { *err = "not a raw mesh file: " + path; return false; }
  int64_t n[2];
  f.read(reinterpret_cast<char *>(n), 16);
  if (!f || n[0] <= 0 || n[1] <= 0 || n[0] > 2000000000LL || n[1] > 2000000000LL) { *err = "bad raw mesh header"; return false; }
  {  // the counts must fit the file before anything is allocated
    const std::streampos here = f.tellg();
    f.seekg(0, std::ios::end);
    const int64_t remaining = int64_t(f.tellg() - here);
    f.seekg(here);
    if (remaining < 24 * n[0] + 16 * n[1]) { *err = "truncated raw mesh file"; return false; }
  }
  coords->resize(size_t(3) * n[0]);
  t2v->resize(size_t(4) * n[1]);
  f.read(reinterpret_cast<char *>(coords->data()), std::streamsize(coords->size() * 8));
  f.read(reinterpret_cast<char *>(t2v->data()), std::streamsize(t2v->size() * 4));
  if (!f) { *err = "truncated raw mesh file"; return false; }
  return true;
}

bool HostMesh::load(const std::string &spec, std::string *err) {
  try {
    return load_unguarded(spec, err);
  } catch (const std::exception &ex) {  // e.g. an absurd element count in a damaged file
    *err = std::string("cannot load mesh ") + spec + ": " + ex.what();
    return false;
  }
}

bool HostMesh::load_unguarded(const std::string &spec, std::string *err) {
  coords.clear();
  t2v.clear();
  if (spec.empty()) {
    // reference wording: PumiTallyImpl.cpp:558-561
    *err = "Omega_h mesh for PumiPIC is not given. Provide --ohMesh = <osh file>";
    return false;
  }
  if (spec.rfind("box:", 0) == 0) {
    double v[6] = {0, 0, 0, -1, -1, -1};
    int n = 0;
    std::stringstream ss(spec.substr(4));
    std::string tok;
    while (n < 6 && std::getline(ss, tok, ',')) v[n++] = std::atof(tok.c_str());
    if (n != 3 && n != 6) { *err = "box spec is box:nx,ny,nz[,lx,ly,lz]"; return false; }
    for (int k = 0; k < 3; ++k)
      if (!(v[k] >= 1.0 && v[k] <= 1e6)) { *err = "box spec needs 1 <= nx,ny,nz <= 1e6"; return false; }
    for (int k = 3; k < n; ++k)
      if (!(v[k] > 0.0 && v[k] < 1e150)) { *err = "box spec needs positive, finite lx,ly,lz"; return false; }
    int nx = int(v[0]), ny = int(v[1]), nz = int(v[2]);
    if (int64_t(nx) * ny * nz * 6 > int64_t(2000000000)) { *err = "box too large for int32 element ids"; return false; }
    double lx = n == 6 ? v[3] : nx, ly = n == 6 ? v[4] : ny, lz = n == 6 ? v[5] : nz;
    build_kuhn_box(nx, ny, nz, lx, ly, lz, &coords, &t2v);
  } else {
    struct stat st;
    if (stat(spec.c_str(), &st) != 0) { *err = "mesh not found: " + spec; return false; }
    const bool is_msh = spec.size() > 4 && spec.compare(spec.size() - 4, 4, ".msh") == 0;
    const bool is_osh = spec.size() > 4 && spec.compare(spec.size() - 4, 4, ".osh") == 0;
    bool ok = (S_ISDIR(st.st_mode) || is_osh) ? read_osh_mesh(spec, &coords, &t2v, err)
              : is_msh            ? read_gmsh_mesh(spec, &coords, &t2v, err)
                                  : read_raw_mesh(spec, &coords, &t2v, err);
    if (!ok) return false;
  }
  nverts = int64_t(coords.size() / 3);
  ntets = int64_t(t2v.size() / 4);
  return finalize(err);
}

bool HostMesh::from_arrays(const double *c, int64_t nv, const int32_t *t, int64_t nt,
                           std::string *err) {
  if (!c || !t || nv < 4 || nt < 1) { *err = "empty mesh"; return false; }
  coords.assign(c, c + 3 * nv);
  t2v.assign(t, t + 4 * nt);
  nverts = nv;
  ntets = nt;
  return finalize(err);
}

bool HostMesh::finalize(std::string *err) {
  if (ntets >= int64_t(0x3fffffff)) { *err = "too many tets: element ids are 30-bit"; return false; }
  for (size_t i = 0; i < t2v.size(); ++i)
    if (t2v[i] < 0 || t2v[i] >= nverts) { *err = "tet2vert index out of range"; return false; }
  for (size_t i = 0; i < coords.size(); ++i)
    if (!(std::fabs(coords[i]) < 1e150)) { *err = "mesh coordinates must be finite (and below 1e150)"; return false; }

  for (int d = 0; d < 3; ++d) { bbox_lo[d] = coords[d]; bbox_hi[d] = coords[d]; }
  for (int64_t v = 0; v < nverts; ++v)
    for (int d = 0; d < 3; ++d) {
      bbox_lo[d] = std::min(bbox_lo[d], coords[3 * v + d]);
      bbox_hi[d] = std::max(bbox_hi[d], coords[3 * v + d]);
    }
  for (int d = 0; d < 3; ++d) {
    double s = 0;
    for (int i = 0; i < 4; ++i) s += coords[3 * size_t(t2v[i]) + d];
    centroid0[d] = s / 4.0;
  }

  // ---- internal element order: z-major background-grid cell of the centroid ----------------
  {
    const double lx = bbox_hi[0] - bbox_lo[0], ly = bbox_hi[1] - bbox_lo[1], lz = bbox_hi[2] - bbox_lo[2];
    const double cells = std::min(std::max(double(ntets) / 4.0, 1.0), double(1 << 24));
    const double h = std::cbrt(std::max(lx * ly * lz, 1e-300) / cells);
    auto dim = [&](double l) { return int64_t(std::min(std::max(std::ceil(l / h), 1.0), 1024.0)); };
    const int64_t gx = dim(lx), gy = dim(ly), gz = dim(lz);
    std::vector<std::pair<int64_t, int32_t>> key(static_cast<size_t>(ntets));
    // Z-curve through the cells by default (a window of consecutive tets is a compact 3-D block: the binned
    // kernels process particles in the same order, engine.hpp `morton_`); PUMITALLY_TET_ORDER=zmajor restores
    // the slab order for experiments
    const char *order_env = std::getenv("PUMITALLY_TET_ORDER");
    const bool morton_order = !(order_env && std::string(order_env) == "zmajor");
#pragma omp parallel for schedule(static)
    for (int64_t e = 0; e < ntets; ++e) {
      double c[3] = {0, 0, 0};
      for (int i = 0; i < 4; ++i)
        for (int d = 0; d < 3; ++d) c[d] += 0.25 * coords[3 * size_t(t2v[4 * e + i]) + d];
      auto cell = [&](double x, double lo, int64_t n) {
        const double q = (x - lo) / h;  // clamped as a double: the cast of a huge or non-finite quotient is undefined
        return q > 0.0 ? (q < double(n - 1) ? int64_t(q) : n - 1) : int64_t(0);
      };
      const int64_t cx = cell(c[0], bbox_lo[0], gx), cy = cell(c[1], bbox_lo[1], gy), cz = cell(c[2], bbox_lo[2], gz);
      int64_t k = (cz * gy + cy) * gx + cx;
      if (morton_order) {
        auto spread = [](uint64_t v) {
          v &= 0x1fffff;
          v = (v | v << 32) & 0x1f00000000ffffull;
          v = (v | v << 16) & 0x1f0000ff0000ffull;
          v = (v | v << 8) & 0x100f00f00f00f00full;
          v = (v | v << 4) & 0x10c30c30c30c30c3ull;
          v = (v | v << 2) & 0x1249249249249249ull;
          return v;
        };
        k = int64_t(spread(uint64_t(cx)) | spread(uint64_t(cy)) << 1 | spread(uint64_t(cz)) << 2);
      }
      key[e] = {k, int32_t(e)};
    }
    std::sort(key.begin(), key.end());  // ties keep the caller's relative order (second = id)
    orig_of_internal.resize(ntets);
    internal_of_orig.resize(ntets);
    std::vector<int32_t> t2v_new(t2v.size());
    for (int64_t i = 0; i < ntets; ++i) {
      const int32_t o = key[i].second;
      orig_of_internal[i] = o;
      internal_of_orig[o] = int32_t(i);
      for (int q = 0; q < 4; ++q) t2v_new[4 * i + q] = t2v[4 * size_t(o) + q];
    }
    t2v.swap(t2v_new);
    start_elem = internal_of_orig[0];
  }

  // ---- face adjacency: sort the 4E (sorted vertex triple, slot) keys --------
  const size_t nf = size_t(4) * ntets;
  t2t.assign(nf, -1);
  {
    std::vector<FaceKey> keys(nf);
#pragma omp parallel for schedule(static)
    for (int64_t e = 0; e < ntets; ++e)
      for (int f = 0; f < 4; ++f) {
        int32_t v[3];
        int k = 0;
        for (int i = 0; i < 4; ++i)
          if (i != f) v[k++] = t2v[4 * e + i];
        sort3(v[0], v[1], v[2]);
        keys[4 * e + f] = FaceKey{v[0], v[1], v[2], int32_t(4 * e + f)};
      }
    std::sort(keys.begin(), keys.end());
    for (size_t i = 0; i < nf;) {
      size_t j = i + 1;
      while (j < nf && keys[i].same(keys[j])) ++j;
      if (j - i == 2) {
        t2t[keys[i].slot] = keys[i + 1].slot / 4;
        t2t[keys[i + 1].slot] = keys[i].slot / 4;
      } else if (j - i > 2) {
        *err = "non-manifold mesh: a face is shared by more than two tets";
        return false;
      }
      i = j;
    }
  }

  // ---- is the hull convex? (tet_mesh.hpp) --------------------------------------
  {
    struct HullEdge { int32_t a, b, opp; int64_t face; };  // edge (a<b) of a hull face, its third vertex, the face
    std::vector<HullEdge> edges;
    std::vector<std::array<int32_t, 3>> hull_faces;
    for (int64_t e = 0; e < ntets; ++e)
      for (int f = 0; f < 4; ++f)
        if (t2t[4 * e + f] < 0) {
          int32_t v[3];
          int k = 0;
          for (int i = 0; i < 4; ++i)
            if (i != f) v[k++] = t2v[4 * e + i];
          const int64_t id = int64_t(hull_faces.size());
          hull_faces.push_back({v[0], v[1], v[2]});
          for (int q = 0; q < 3; ++q) {
            const int32_t a = v[q], b = v[(q + 1) % 3], o = v[(q + 2) % 3];
            edges.push_back(HullEdge{std::min(a, b), std::max(a, b), o, id});
          }
        }
    std::sort(edges.begin(), edges.end(), [](const HullEdge &x, const HullEdge &y) {
      return x.a != y.a ? x.a < y.a : (x.b != y.b ? x.b < y.b : x.face < y.face);
    });
    // outward normal of a hull face = away from the tet's fourth vertex; found again from the face id
    std::vector<double> normal(3 * hull_faces.size());
    {
      size_t id = 0;
      for (int64_t e = 0; e < ntets; ++e)
        for (int f = 0; f < 4; ++f)
          if (t2t[4 * e + f] < 0) {
            const auto &hf = hull_faces[id];
            const double *A = &coords[3 * size_t(hf[0])], *B = &coords[3 * size_t(hf[1])], *C = &coords[3 * size_t(hf[2])];
            const double *P = &coords[3 * size_t(t2v[4 * e + f])];
            double ab[3], ac[3], n[3];
            for (int d = 0; d < 3; ++d) { ab[d] = B[d] - A[d]; ac[d] = C[d] - A[d]; }
            n[0] = ab[1] * ac[2] - ab[2] * ac[1]; n[1] = ab[2] * ac[0] - ab[0] * ac[2]; n[2] = ab[0] * ac[1] - ab[1] * ac[0];
            const double len = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
            const double side = n[0] * (P[0] - A[0]) + n[1] * (P[1] - A[1]) + n[2] * (P[2] - A[2]);
            for (int d = 0; d < 3; ++d) normal[3 * id + d] = (side > 0 ? -n[d] : n[d]) / (len > 0 ? len : 1.0);
            ++id;
          }
    }
    bool convex = true;
    double diag = 0.0;
    for (int d = 0; d < 3; ++d) diag += (bbox_hi[d] - bbox_lo[d]) * (bbox_hi[d] - bbox_lo[d]);
    const double tol = 1e-9 * std::sqrt(diag);
    for (size_t i = 0; i < edges.size() && convex;) {
      size_t j = i + 1;
      while (j < edges.size() && edges[j].a == edges[i].a && edges[j].b == edges[i].b) ++j;
      if (j - i != 2) {
        convex = false;  // an edge where more than two hull faces meet: hull components touching
      } else {
        // the third vertex of each face must not lie outside the other face's plane
        const double *A = &coords[3 * size_t(edges[i].a)];
        for (int s2 = 0; s2 < 2; ++s2) {
          const HullEdge &mine = edges[i + s2], &other = edges[i + 1 - s2];
          const double *O = &coords[3 * size_t(other.opp)];
          const double *n = &normal[3 * size_t(mine.face)];
          if (n[0] * (O[0] - A[0]) + n[1] * (O[1] - A[1]) + n[2] * (O[2] - A[2]) > tol) convex = false;
        }
      }
      i = j;
    }
    // one component: a second closed surface (a void) is concave all over, so it fails the test above
    hull_convex = convex;
  }

  // ---- mesh-centred coordinates (tet_mesh.hpp) ---------------------------------
  for (int d = 0; d < 3; ++d) center[d] = 0.5 * bbox_lo[d] + 0.5 * bbox_hi[d];
  ccoords.resize(coords.size());
#pragma omp parallel for schedule(static)
  for (int64_t v = 0; v < nverts; ++v)
    for (int d = 0; d < 3; ++d) ccoords[3 * v + d] = coords[3 * v + d] - center[d];

  // ---- volumes + packed records ----------------------------------------------
  volume.resize(ntets);
  records.resize(ntets);
  bool degenerate = false;
#pragma omp parallel for schedule(static) reduction(|| : degenerate)
  for (int64_t e = 0; e < ntets; ++e) {
    const double *V[4];
    for (int i = 0; i < 4; ++i) V[i] = &ccoords[3 * size_t(t2v[4 * e + i])];
    {
      double a[3], b[3], c[3];
      for (int d = 0; d < 3; ++d) { a[d] = V[1][d] - V[0][d]; b[d] = V[2][d] - V[0][d]; c[d] = V[3][d] - V[0][d]; }
      double det = a[0] * (b[1] * c[2] - b[2] * c[1]) - a[1] * (b[0] * c[2] - b[2] * c[0]) +
                   a[2] * (b[0] * c[1] - b[1] * c[0]);
      volume[e] = std::fabs(det) / 6.0;
      if (!(volume[e] > 0.0)) degenerate = true;
    }
    TetRecord &r = records[e];
    for (int f = 0; f < 4; ++f) {
      int32_t v[3];
      int k = 0;
      for (int i = 0; i < 4; ++i)
        if (i != f) v[k++] = t2v[4 * e + i];
      sort3(v[0], v[1], v[2]);
      const double *A = &ccoords[3 * size_t(v[0])], *B = &ccoords[3 * size_t(v[1])],
                   *C = &ccoords[3 * size_t(v[2])];
      double ab[3], ac[3], n[3];
      for (int d = 0; d < 3; ++d) { ab[d] = B[d] - A[d]; ac[d] = C[d] - A[d]; }
      n[0] = ab[1] * ac[2] - ab[2] * ac[1];
      n[1] = ab[2] * ac[0] - ab[0] * ac[2];
      n[2] = ab[0] * ac[1] - ab[1] * ac[0];
      double len = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
      if (!(len > 0.0)) { degenerate = true; len = 1.0; }
      double p[4];
      p[0] = n[0] / len; p[1] = n[1] / len; p[2] = n[2] / len;
      p[3] = p[0] * A[0] + p[1] * A[1] + p[2] * A[2];
      // canonical truncation: identical for both tets sharing the face
      for (int q = 0; q < 4; ++q) p[q] = bdouble(dbits(p[q]) & ~uint64_t(0xff));
      // orient outward: the opposite vertex must satisfy n.x < c
      const double *P = V[f];
      double side = p[0] * P[0] + p[1] * P[1] + p[2] * P[2] - p[3];
      if (side > 0.0)
        for (int q = 0; q < 4; ++q) p[q] = -p[q];
      else if (side == 0.0)
        degenerate = true;
      // payload = this tet XOR neighbour (hull: neighbour = -1): the same 32 bits on both
      // sides of the face, so the two records hold bit-identical planes up to the sign bit
      // and the kernel can use the doubles as they are, payload included
      // bits 0..29: this tet XOR neighbour (hull = all ones); bits 30..31: f XOR the neighbour's
      // local index of this face.  Both are symmetric, so both records carry the same 32 bits.
      const int32_t nb = t2t[4 * e + f];
      int back = f;
      if (nb >= 0)
        for (int q = 0; q < 4; ++q)
          if (t2t[4 * size_t(nb) + q] == int32_t(e)) back = q;
      const uint32_t idmask = 0x3fffffffu;
      uint32_t pay = ((uint32_t(e) ^ (nb < 0 ? idmask : uint32_t(nb))) & idmask) | (uint32_t(f ^ back) << 30);
      for (int q = 0; q < 4; ++q)
        r.d[4 * f + q] = bdouble(dbits(p[q]) | uint64_t((pay >> (8 * q)) & 0xffu));
      if (nb < 0) {
        // Hull face: truncation and payload move the stored plane by ~1e-13 either way.  Make it err
        // outwards only: raise the offset on the 44-bit grid (the payload byte stays) until the three face
        // vertices satisfy n.x <= c, with the normal exactly as stored and a margin for the rounding of n.x.  A point exactly on the
        // hull is then inside (a destination there is reached, a track along the hull surface is walked),
        // and what leaves the mesh is clipped at most ~1e-13 further out.  Interior faces keep the
        // symmetric truncation: both tets must see the identical plane.
        const double nx = r.d[4 * f], ny = r.d[4 * f + 1], nz = r.d[4 * f + 2];
        const double need = std::max({nx * A[0] + ny * A[1] + nz * A[2], nx * B[0] + ny * B[1] + nz * B[2],
                                      nx * C[0] + ny * C[1] + nz * C[2]});
        // margin for the rounding of n.o in the kernels (fused multiply-adds there, none here; the
        // numerator and the denominator of the same crossing round differently): a few ulps of the largest
        // value n.o can take for a ray origin anywhere in the mesh
        // (centred coordinates: n.o is at most |n|.half-extent; the translation x - center is itself
        // correctly rounded, i.e. off by at most half an ulp of a number of that size, and exact far
        // from the origin)
        const double mag = std::fabs(nx) * 0.5 * (bbox_hi[0] - bbox_lo[0]) + std::fabs(ny) * 0.5 * (bbox_hi[1] - bbox_lo[1]) +
                           std::fabs(nz) * 0.5 * (bbox_hi[2] - bbox_lo[2]);
        const double target = need + 34.0 * 2.220446049250313e-16 * mag;
        double c = r.d[4 * f + 3];
        if (!(c >= target)) {
          const uint64_t low = dbits(c) & 0xffu;  // the payload byte stays
          if (target > 0.0) {                     // round the magnitude up on the 44-bit grid
            c = bdouble((((dbits(target) >> 8) + 1) << 8) | low);
          } else {                                // negative (or zero): round the magnitude down
            const uint64_t m = dbits(std::fabs(target)) >> 8;
            c = m > 1 ? -bdouble(((m - 1) << 8) | low) : bdouble(low);
          }
        }
        r.d[4 * f + 3] = c;
      }
    }
  }
  if (degenerate) { *err = "mesh contains a degenerate (zero-volume) tet"; return false; }
  // The plane offsets keep 44 mantissa bits of mesh-centred numbers: a crossing point is located to
  // ~6e-14 of the mesh extent.  What remains far from the origin is the granularity of the caller's own
  // coordinates (ulp of the absolute position against the size of a tet): worth a warning only when
  // it reaches 1e-9 of a tet edge.
  {
    double far = 0.0, vol = 0.0;
    for (int d = 0; d < 3; ++d) far = std::max({far, std::fabs(bbox_lo[d]), std::fabs(bbox_hi[d])});
    for (int64_t e = 0; e < ntets; ++e) vol += volume[e];
    const double edge = std::cbrt(6.0 * vol / double(ntets));
    if (far * 2.220446049250313e-16 > 1e-9 * edge)
      fprintf(stderr, "[pumitally] WARNING: mesh coordinates reach %.3g, %.1e mean tet edges from the origin: double "
                      "precision positions there resolve only %.1e of a tet edge; translate the mesh (and the "
                      "particle coordinates) towards the origin\n", far, far / edge, far * 2.220446049250313e-16 / edge);
  }
  return true;
}

// ---- compact layout -----------------------------------------------------------------------
bool HostMesh::build_compact(std::string *err) {
  if (nverts > int64_t(kVertMask)) { *err = "too many vertices for the compact layout (28-bit ids)"; return false; }
  // vertices in order of first use by the (spatially ordered) internal tets
  std::vector<int32_t> vnew(static_cast<size_t>(nverts), -1);
  int32_t next = 0;
  for (size_t i = 0; i < t2v.size(); ++i)
    if (vnew[t2v[i]] < 0) vnew[t2v[i]] = next++;
  for (int64_t v = 0; v < nverts; ++v)
    if (vnew[v] < 0) vnew[v] = next++;
  cverts.assign(static_cast<size_t>(nverts), VertexRec{0, 0, 0, 0});
  for (int64_t v = 0; v < nverts; ++v)
    cverts[vnew[v]] = VertexRec{ccoords[3 * v], ccoords[3 * v + 1], ccoords[3 * v + 2], 0.0};

  // slot s of tet e = local vertex (s ^ flip) for s >= 2: swapping the last two makes det > 0
  std::vector<uint8_t> flip(static_cast<size_t>(ntets));
#pragma omp parallel for schedule(static)
  for (int64_t e = 0; e < ntets; ++e) {
    const double *V[4];
    for (int i = 0; i < 4; ++i) V[i] = &ccoords[3 * size_t(t2v[4 * e + i])];
    double a[3], b[3], c[3];
    for (int d = 0; d < 3; ++d) { a[d] = V[1][d] - V[0][d]; b[d] = V[2][d] - V[0][d]; c[d] = V[3][d] - V[0][d]; }
    const double det = a[0] * (b[1] * c[2] - b[2] * c[1]) - a[1] * (b[0] * c[2] - b[2] * c[0]) +
                       a[2] * (b[0] * c[1] - b[1] * c[0]);
    flip[e] = det < 0.0;
  }
  auto local_of_slot = [&](int64_t e, int s) { return (flip[e] && s >= 2) ? (s ^ 1) : s; };  // involution

  starts.resize(static_cast<size_t>(ntets));
  bool bad = false;
#pragma omp parallel for schedule(static) reduction(|| : bad)
  for (int64_t e = 0; e < ntets; ++e) {
    TetStart &S = starts[e];
    for (int s = 0; s < 4; ++s) {
      const int32_t v = t2v[4 * e + local_of_slot(e, s)];
      for (int d = 0; d < 3; ++d) S.v[3 * s + d] = ccoords[3 * size_t(v) + d];
    }
    for (int k = 0; k < 4; ++k) {
      const int32_t nb = t2t[4 * e + local_of_slot(e, k)];
      if (nb < 0) { S.links.nbr[k] = 0x3fffffffu; S.links.opp[k] = 0; continue; }
      int back = -1;
      for (int q = 0; q < 4; ++q)
        if (t2t[4 * size_t(nb) + q] == int32_t(e)) back = q;
      if (back < 0) { bad = true; continue; }
      uint32_t map[3] = {0, 0, 0};
      int j = 0;
      for (int s = 0; s < 4; ++s) {
        if (s == k) continue;
        const int32_t vid = t2v[4 * e + local_of_slot(e, s)];
        int where = -1;
        for (int q = 0; q < 4; ++q)
          if (t2v[4 * size_t(nb) + q] == vid) where = q;
        if (where < 0 || where == back) bad = true;
        map[j++] = uint32_t(local_of_slot(nb, where < 0 ? 0 : where));
      }
      S.links.nbr[k] = uint32_t(nb) | (map[0] << 30);
      S.links.opp[k] = uint32_t(vnew[t2v[4 * size_t(nb) + back]]) | ((map[1] | (map[2] << 2)) << 28);
    }
  }
  if (bad) { *err = "inconsistent face adjacency while building the compact layout"; return false; }
  return true;
}

void linear_moments(const double v[12], const double C[3], const double *rec, int S, int k, double m1[3], double g[3]) {
  double c[3], d[4][3];
  for (int a = 0; a < 3; ++a) c[a] = 0.25 * (v[a] + v[3 + a] + v[6 + a] + v[9 + a]);
  for (int i = 0; i < 4; ++i)
    for (int a = 0; a < 3; ++a) d[i][a] = v[3 * i + a] - c[a];
  const double m0 = rec[k];
  for (int a = 0; a < 3; ++a) m1[a] = rec[(1 + a) * S + k] - (c[a] - C[a]) * m0;
  // V from the edge vectors (the d_i differ from them by the same translation)
  const double e1[3] = {d[1][0] - d[0][0], d[1][1] - d[0][1], d[1][2] - d[0][2]};
  const double e2[3] = {d[2][0] - d[0][0], d[2][1] - d[0][1], d[2][2] - d[0][2]};
  const double e3[3] = {d[3][0] - d[0][0], d[3][1] - d[0][1], d[3][2] - d[0][2]};
  const double vol = std::fabs(e1[0] * (e2[1] * e3[2] - e2[2] * e3[1]) - e1[1] * (e2[0] * e3[2] - e2[2] * e3[0]) +
                               e1[2] * (e2[0] * e3[1] - e2[1] * e3[0])) / 6.0;
  double M[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int i = 0; i < 4; ++i)
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) M[a][b] += d[i][a] * d[i][b];
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) M[a][b] *= vol / 20.0;
  // symmetric 3x3 solve by the adjugate
  const double A00 = M[1][1] * M[2][2] - M[1][2] * M[2][1], A01 = M[0][2] * M[2][1] - M[0][1] * M[2][2],
               A02 = M[0][1] * M[1][2] - M[0][2] * M[1][1], A11 = M[0][0] * M[2][2] - M[0][2] * M[2][0],
               A12 = M[0][2] * M[1][0] - M[0][0] * M[1][2], A22 = M[0][0] * M[1][1] - M[0][1] * M[1][0];
  const double det = M[0][0] * A00 + M[0][1] * (M[1][2] * M[2][0] - M[1][0] * M[2][2]) + M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
  if (!(std::fabs(det) > 0.0) || !std::isfinite(det)) {
    g[0] = g[1] = g[2] = 0.0;
    return;
  }
  const double inv = 1.0 / det;
  g[0] = (A00 * m1[0] + A01 * m1[1] + A02 * m1[2]) * inv;
  g[1] = (A01 * m1[0] + A11 * m1[1] + A12 * m1[2]) * inv;
  g[2] = (A02 * m1[0] + A12 * m1[1] + A22 * m1[2]) * inv;
}

}  // namespace ptb
