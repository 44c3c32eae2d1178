// Host-side tet mesh container and the packed device record format.
//
// Replaces what the reference obtains from Omega_h (mesh read
// PumiTallyImpl.cpp:553-568, coords / tet->vert adjacency
// PumiTallyImpl.cpp:384-385, 495-496) and from pumi-pic (face adjacency used by
// the external tracer).  Nothing here is on the per-step hot path.
#pragma once
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

namespace ptb {

// One tet = one 128-byte, 128-byte-aligned record = exactly one L2 line and
// one cp.async.bulk transfer:
//
//   d[4f+0..2] = outward normal of the face opposite local vertex f
//   d[4f+3]    = plane offset c  (n.x == c on the face, n.x < c inside)
//
// Both tets that share a face carry the *same* plane up to an exact sign flip
// (it is built once from the three face vertices in ascending global id), so
// the ray parameter of a crossing is bit-identical seen from either side and
// the walk is watertight.  The low 8 bits of each of the 16 mantissas carry a
// payload instead of geometry: the four low bytes of face f's four doubles
// spell  (this tet id) XOR (id of the neighbour across face f, -1 = hull).
// The XOR is the same number in both records, so the planes stay bit-identical
// on both sides *with* the payload in place (a 2^-44 relative perturbation) and
// the kernel needs no masking; it recovers the neighbour as payload XOR own id.
struct alignas(128) TetRecord {
  double d[16];
};
static_assert(sizeof(TetRecord) == 128, "TetRecord must be one 128-byte line");

// Compact (vertex-indexed) layout read by the edge-function walk; see walk_compact.cuh.
// Per tet, indexed by local face k = face opposite local vertex ("slot") k.  Slots are ordered
// so that the tet is positively oriented: det(v1-v0, v2-v0, v3-v0) > 0.
//   nbr[k]  bits 0..29  neighbour across face k (all ones = hull)
//           bits 30..31 map[0]
//   opp[k]  bits 0..27  vertex of that neighbour opposite the shared face
//           bits 28..31 map[1] | map[2] << 2
// map[j] = the neighbour's slot of this tet's j-th slot other than k (ascending).
struct alignas(32) TetLinks {
  uint32_t nbr[4];
  uint32_t opp[4];
};
static_assert(sizeof(TetLinks) == 32, "TetLinks must be one sector");

struct alignas(32) VertexRec {
  double x, y, z, pad;
};

// First tet of a ray: the four vertices in slot order + the links, one 128-byte line.
struct alignas(128) TetStart {
  double v[12];
  TetLinks links;
};
static_assert(sizeof(TetStart) == 128, "TetStart must be one 128-byte line");

constexpr uint32_t kVertMask = 0x0fffffffu;  // vertex ids are 28-bit in the compact layout

struct HostMesh {
  int64_t nverts = 0;
  int64_t ntets = 0;
  std::vector<double> coords;    // [3*nverts]
  std::vector<int32_t> t2v;      // [4*ntets]
  std::vector<int32_t> t2t;      // [4*ntets], neighbour across face opposite vertex f, -1 hull
  std::vector<double> volume;    // [ntets]
  std::vector<TetRecord> records;  // [ntets]
  std::vector<TetStart> starts;    // [ntets]  compact layout (build_compact())
  std::vector<VertexRec> cverts;   // [nverts] vertices in order of first use by the internal tet order
  double centroid0[3] = {0, 0, 0};  // centroid of (the caller's) element 0 (PumiTallyImpl.cpp:500-509)

  // INTERNAL ELEMENT ORDER.  finalize() renumbers the tets along a Z-order (Morton) curve through the
  // cells of a background grid, by the cell that holds their centroid, so that tets that are close in
  // space are close in memory whatever numbering the mesh file came with (the spatially binned walk
  // processes particles along the same curve).  t2v, t2t, volume and records are stored in this
  // internal order; everything that leaves the library (flux, element ids, adjacency, VTK) is
  // translated back to the caller's numbering with these two maps.
  std::vector<int32_t> orig_of_internal, internal_of_orig;
  int32_t start_elem = 0;  // internal id of the caller's element 0 (where particles are parked)

  template <typename T>
  std::vector<T> to_original(const T *internal, int ncomp = 1) const {
    std::vector<T> out(size_t(ntets) * ncomp);
    for (int64_t i = 0; i < ntets; ++i)
      for (int c = 0; c < ncomp; ++c) out[size_t(orig_of_internal[i]) * ncomp + c] = internal[size_t(i) * ncomp + c];
    return out;
  }
  std::vector<int32_t> adjacency_original() const {
    std::vector<int32_t> out(size_t(4) * ntets);
    for (int64_t i = 0; i < ntets; ++i)
      for (int f = 0; f < 4; ++f) {
        const int32_t nb = t2t[4 * i + f];
        out[size_t(4) * orig_of_internal[i] + f] = nb < 0 ? -1 : orig_of_internal[nb];
      }
    return out;
  }
  double bbox_lo[3] = {0, 0, 0}, bbox_hi[3] = {0, 0, 0};
  // MESH-CENTRED COORDINATES.  Face planes (and the compact layout's vertices) are stored relative to
  // `center`, the middle of the bounding box, and the kernels translate every ray origin once
  // (x - center) before walking.  The 44-bit plane offsets then locate a crossing to ~6e-14 of the
  // mesh EXTENT instead of the largest absolute coordinate, so the tally keeps its digits however far
  // from the origin the mesh sits (only the granularity of the caller's own doubles remains).
  // Is the hull one closed, everywhere locally convex surface?  (Every hull edge is shared by two hull
  // faces whose dihedral angle, seen from inside, is <= 180 degrees, and there is one hull component.)
  // Only then does "walk straight from A to B inside the mesh" reach every B in the mesh, which is what
  // the seed-grid shortcut of the relocation walk relies on to be equivalent to the reference.
  bool hull_convex = true;
  double center[3] = {0, 0, 0};
  std::vector<double> ccoords;  // [3*nverts] coords - center, as the kernels compute it (fl(x - c))

  // "box:nx,ny,nz[,lx,ly,lz]" | raw mesh file | Gmsh .msh (2.2 / 4.1, ASCII or binary) | Omega_h .osh directory.
  bool load(const std::string &spec, std::string *err);
  bool load_unguarded(const std::string &spec, std::string *err);
  bool from_arrays(const double *coords, int64_t nverts, const int32_t *tet2vert, int64_t ntets,
                   std::string *err);
  // adjacency + volumes + packed records; called by load()/from_arrays().
  bool finalize(std::string *err);
  // compact layout (starts[].links is the TetLinks table); needs finalize() first.
  bool build_compact(std::string *err);
};

// Linear flux moments of one element from the walk's raw record (walk_core.cuh, moment_tally).  v: the element's
// four vertices (12 doubles, the caller's coordinates); C: the centre the walk accumulated about (HostMesh::center);
// rec: the element's record, S slots per moment ([m0][Rx][Ry][Rz]); k: the score.  Returns m1 = R - (c - C) m0, the
// first moment about the centroid c, and g = M^-1 m1 with M = (V/20) sum_i (v_i - c)(v_i - c)^T, the gradient of the
// flux's L2 projection onto linear functions on the element.  fp64; a degenerate element (M singular) gets g = 0.
void linear_moments(const double v[12], const double C[3], const double *rec, int S, int k, double m1[3], double g[3]);

// Generators / readers (tet_mesh.cpp, osh_reader.cpp)
void build_kuhn_box(int nx, int ny, int nz, double lx, double ly, double lz,
                    std::vector<double> *coords, std::vector<int32_t> *t2v);
bool read_raw_mesh(const std::string &path, std::vector<double> *coords,
                   std::vector<int32_t> *t2v, std::string *err);
bool read_gmsh_mesh(const std::string &path, std::vector<double> *coords,
                    std::vector<int32_t> *t2v, std::string *err);
bool read_osh_mesh(const std::string &dir, std::vector<double> *coords,
                   std::vector<int32_t> *t2v, std::string *err);

}  // namespace ptb
