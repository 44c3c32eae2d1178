// VTK output of the normalised tally (reference: FinalizeTallies,
// PumiTallyImpl.cpp:411-416 -> Omega_h::vtk::write_parallel(filename, mesh, 3)).
#pragma once
#include <string>
#include <utility>
#include <vector>

#include "tet_mesh.hpp"

namespace ptb {

// Writes the directory layout Omega_h's parallel writer produces --
// <path>/pieces.pvtu and <path>/pieces/piece_<rank>.vtu -- with cell data
// "flux" (raw flux / tet volume) and "volume".  Arrays are stored as raw
// appended binary (little endian, UInt64 block headers).  flux and volume are
// whole-mesh arrays in the caller's element order; rank r of nranks writes the
// r-th contiguous slice of the elements as its piece, rank 0 also the .pvtu.
// `extra`: further named Float64 cell arrays of the same shape (the per-bin fluxes of a filtered tally).
// `extra_ncomp[i]`: components per element of extra[i], interleaved (3 for the flux gradients); 1 where the vector
// is shorter.
// The writer stores every tet positively oriented, as VTK expects: a tet whose caller's vertices v[0..3] are
// negatively oriented is written with v[2] and v[3] swapped.
bool vtk_cell_flipped(const HostMesh &mesh, const int32_t *v);

bool write_vtk_dataset(const std::string &path, const HostMesh &mesh,
                       const std::vector<double> &flux, const std::vector<double> &volume,
                       int rank, int nranks, std::string *err,
                       const std::vector<std::pair<std::string, const double *>> &extra = {},
                       const std::vector<int> &extra_ncomp = {});

}  // namespace ptb
