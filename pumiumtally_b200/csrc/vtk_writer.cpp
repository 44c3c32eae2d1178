#include "vtk_writer.hpp"

#include <cerrno>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <utility>
#include <sys/stat.h>

namespace ptb {
namespace {

bool make_dir(const std::string &p, std::string *err) {
  if (mkdir(p.c_str(), 0777) == 0 || errno == EEXIST) return true;
  *err = "cannot create directory " + p + ": " + std::strerror(errno);
  return false;
}

struct Block {
  const void *data;
  uint64_t bytes;
};

}  // namespace

bool vtk_cell_flipped(const HostMesh &m, const int32_t *v) {
  const double *a = m.coords.data() + 3 * size_t(v[0]), *b = m.coords.data() + 3 * size_t(v[1]);
  const double *c = m.coords.data() + 3 * size_t(v[2]), *d = m.coords.data() + 3 * size_t(v[3]);
  const double ab[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, ac[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]},
               ad[3] = {d[0] - a[0], d[1] - a[1], d[2] - a[2]};
  const double det = ab[0] * (ac[1] * ad[2] - ac[2] * ad[1]) - ab[1] * (ac[0] * ad[2] - ac[2] * ad[0]) +
                     ab[2] * (ac[0] * ad[1] - ac[1] * ad[0]);
  return det < 0.0;
}

bool write_vtk_dataset(const std::string &path, const HostMesh &m, const std::vector<double> &flux,
                       const std::vector<double> &volume, int rank, int nranks, std::string *err,
                       const std::vector<std::pair<std::string, const double *>> &extra,
                       const std::vector<int> &extra_ncomp) {
  auto ncomp = [&](size_t i) { return i < extra_ncomp.size() ? uint64_t(extra_ncomp[i]) : uint64_t(1); };
  if (!make_dir(path, err) || !make_dir(path + "/pieces", err)) return false;
  const uint64_t V = uint64_t(m.nverts), Etot = uint64_t(m.ntets);
  // One piece per rank.  After the batch-end exchange every rank holds the same global tally, so
  // rank r writes the r-th contiguous slice of the elements (caller's numbering) and the pieces
  // tile the mesh; with one rank the piece is the whole mesh, as in the reference.
  const uint64_t e0 = Etot * uint64_t(rank) / uint64_t(nranks), e1 = Etot * uint64_t(rank + 1) / uint64_t(nranks);
  const uint64_t E = e1 - e0;
  std::vector<int32_t> offsets(E);
  for (uint64_t e = 0; e < E; ++e) offsets[e] = int32_t(4 * (e + 1));
  std::vector<uint8_t> types(E, 10);  // VTK_TETRA
  // connectivity in the caller's element order (the cell data arrays already are), every tet
  // positively oriented as VTK expects: det(v1-v0, v2-v0, v3-v0) > 0
  std::vector<int32_t> conn = m.to_original(m.t2v.data(), 4);
  for (uint64_t e = e0; e < e1; ++e) {
    int32_t *v = conn.data() + 4 * e;
    if (vtk_cell_flipped(m, v)) std::swap(v[2], v[3]);
  }
  std::vector<Block> blocks = {{m.coords.data(), V * 24}, {conn.data() + 4 * e0, E * 16},
                               {offsets.data(), E * 4},   {types.data(), E},
                               {flux.data() + e0, E * 8}, {volume.data() + e0, E * 8}};
  for (size_t i = 0; i < extra.size(); ++i)  // whole-mesh arrays, caller's element order
    blocks.push_back({extra[i].second + e0 * ncomp(i), E * 8 * ncomp(i)});
  std::vector<uint64_t> off(blocks.size());
  uint64_t acc = 0;
  for (size_t i = 0; i < blocks.size(); ++i) { off[i] = acc; acc += 8 + blocks[i].bytes; }

  const std::string piece = path + "/pieces/piece_" + std::to_string(rank) + ".vtu";
  std::ofstream f(piece, std::ios::binary);
  if (!f) { *err = "cannot open " + piece; return false; }
  f << "<?xml version=\"1.0\"?>\n"
    << "<VTKFile type=\"UnstructuredGrid\" version=\"1.0\" byte_order=\"LittleEndian\" header_type=\"UInt64\">\n"
    << "<UnstructuredGrid>\n"
    << "<Piece NumberOfPoints=\"" << V << "\" NumberOfCells=\"" << E << "\">\n"
    << "<Points>\n<DataArray type=\"Float64\" Name=\"coordinates\" NumberOfComponents=\"3\" format=\"appended\" offset=\"" << off[0] << "\"/>\n</Points>\n"
    << "<Cells>\n"
    << "<DataArray type=\"Int32\" Name=\"connectivity\" format=\"appended\" offset=\"" << off[1] << "\"/>\n"
    << "<DataArray type=\"Int32\" Name=\"offsets\" format=\"appended\" offset=\"" << off[2] << "\"/>\n"
    << "<DataArray type=\"UInt8\" Name=\"types\" format=\"appended\" offset=\"" << off[3] << "\"/>\n"
    << "</Cells>\n"
    << "<CellData>\n"
    << "<DataArray type=\"Float64\" Name=\"flux\" NumberOfComponents=\"1\" format=\"appended\" offset=\"" << off[4] << "\"/>\n"
    << "<DataArray type=\"Float64\" Name=\"volume\" NumberOfComponents=\"1\" format=\"appended\" offset=\"" << off[5] << "\"/>\n";
  for (size_t i = 0; i < extra.size(); ++i)
    f << "<DataArray type=\"Float64\" Name=\"" << extra[i].first << "\" NumberOfComponents=\"" << ncomp(i)
      << "\" format=\"appended\" offset=\"" << off[6 + i] << "\"/>\n";
  f << "</CellData>\n"
    << "</Piece>\n</UnstructuredGrid>\n<AppendedData encoding=\"raw\">\n_";
  for (size_t i = 0; i < blocks.size(); ++i) {
    f.write(reinterpret_cast<const char *>(&blocks[i].bytes), 8);
    f.write(reinterpret_cast<const char *>(blocks[i].data), std::streamsize(blocks[i].bytes));
  }
  f << "\n</AppendedData>\n</VTKFile>\n";
  if (!f) { *err = "write failed: " + piece; return false; }
  f.close();

  if (rank == 0) {
    std::ofstream p(path + "/pieces.pvtu");
    if (!p) { *err = "cannot open " + path + "/pieces.pvtu"; return false; }
    p << "<?xml version=\"1.0\"?>\n"
      << "<VTKFile type=\"PUnstructuredGrid\" version=\"1.0\" byte_order=\"LittleEndian\" header_type=\"UInt64\">\n"
      << "<PUnstructuredGrid GhostLevel=\"0\">\n"
      << "<PPoints>\n<PDataArray type=\"Float64\" Name=\"coordinates\" NumberOfComponents=\"3\"/>\n</PPoints>\n"
      << "<PCellData>\n"
      << "<PDataArray type=\"Float64\" Name=\"flux\" NumberOfComponents=\"1\"/>\n"
      << "<PDataArray type=\"Float64\" Name=\"volume\" NumberOfComponents=\"1\"/>\n";
    for (size_t i = 0; i < extra.size(); ++i)
      p << "<PDataArray type=\"Float64\" Name=\"" << extra[i].first << "\" NumberOfComponents=\"" << ncomp(i) << "\"/>\n";
    p << "</PCellData>\n";
    for (int r = 0; r < nranks; ++r) p << "<Piece Source=\"pieces/piece_" << r << ".vtu\"/>\n";
    p << "</PUnstructuredGrid>\n</VTKFile>\n";
  }
  return true;
}

}  // namespace ptb
