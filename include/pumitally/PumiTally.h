// pumitally::PumiTally -- drop-in facade of the H100 track-length tally engine.
//
// This header declares the same class, in the same namespace, with the same
// member functions, argument types, const-ness and data layout (one
// std::unique_ptr<PumiTallyImpl>) as the reference's public header
// (reference: src/pumitally/PumiTally.h:34-107), so a translation unit compiled
// against either header links against either library: the Itanium-mangled
// symbols are identical (checked by tests/test_abi_symbols.py).
//
// Everything behind the pointer is new: CUDA kernels for sm_90a reached through
// the extern "C" layer in include/pumitally_c.h.
#ifndef PUMITALLY_PUMITALLY_H
#define PUMITALLY_PUMITALLY_H

#include <cstdint>
#include <memory>
#include <string>

namespace pumitally {

struct ParticleAtElemBoundary;  // kept so code naming the reference type still parses
struct PumiTallyImpl;           // opaque; owns the engine handle

class PumiTally {
public:
  // Loads the tet mesh and allocates state for `num_particles` particles, all
  // parked at the centroid of element 0 (reference: PumiTally.h:50-51,
  // PumiTallyImpl.cpp:31-52).
  //
  // `mesh_filename` may name
  //   * an Omega_h mesh directory  "<name>.osh"  (no trailing '/'),
  //   * a raw mesh file written by pumiumtally_b200.mesh.save_raw_mesh, or
  //   * a synthetic Kuhn box       "box:nx,ny,nz[,lx,ly,lz]".
  // argc/argv are accepted for source compatibility (the reference forwards
  // them to MPI/Kokkos); recognised options: --pumitally-device=<id>.
  PumiTally(const std::string &mesh_filename, int32_t num_particles, int &argc,
            char **&argv);

  // Localises every particle: walks from the centroid of element 0 to
  // init_particle_positions[3*i..3*i+2] with tallying off.  Call exactly once.
  // `size` is the number of doubles, i.e. 3 * num_particles (reference:
  // PumiTally.h:66-67, PumiTallyImpl.cpp:54-64; the "number of particles"
  // wording in the reference header does not match its own assert).
  void CopyInitialPosition(double *init_particle_positions,
                           std::int32_t size) const;

  // One transport step for the whole batch (reference: PumiTally.h:87-89,
  // PumiTallyImpl.cpp:66-149): particles with flying[i]==1 are first relocated
  // to particle_origin (never tallied), then fly to particle_destinations while
  // every tet they cross receives  track length * weights[i].  Tracks leaving
  // the mesh are clipped at the hull.  All pointers are host memory laid out
  // x0,y0,z0,x1,...; `size` = 3 * num_particles; flying[] is zeroed on return.
  void MoveToNextLocation(double *particle_origin,
                          double *particle_destinations, int8_t *flying,
                          double *weights, int32_t size) const;

  // Normalises the tally by tet volume and writes "fluxresult.vtk" with cell
  // data "flux" and "volume", then prints the [TIME] block (reference:
  // PumiTally.h:95, PumiTallyImpl.cpp:151-157, 382-416, 22-29).
  void WriteTallyResults() const;

  ~PumiTally();

private:
  std::unique_ptr<PumiTallyImpl> pimpl_;
};

} // namespace pumitally

#endif // PUMITALLY_PUMITALLY_H
