// TEST-ONLY C wrappers of the per-move binning launchers (bin_kernels.cu) and of the initial-weight sum
// (walk_kernels.cu) of libpumitally.so, so that tests/test_gpu_bin_kernels.py can call them on raw device pointers and
// grid geometries it chose itself (grids far larger than its meshes, keys on cell boundaries and outside the box,
// ranges that start past 0).  Not part of the library and not a C ABI of the project.
#include <cstdint>

#include "walk_kernels.hpp"

namespace {

ptb::SeedGrid make_grid(double x0, double y0, double z0, double h, double inv_h, int32_t nx, int32_t ny, int32_t nz,
                        const int32_t *cell_rank) {
  ptb::SeedGrid g{};
  g.cell_tet = nullptr;  // the binning passes never read it
  g.cell_rank = cell_rank;
  g.x0 = x0; g.y0 = y0; g.z0 = z0;
  g.h = h;
  g.inv_h = inv_h;
  g.far2 = 4.0 * h * h;
  g.nx = nx; g.ny = ny; g.nz = nz;
  return g;
}

}  // namespace

extern "C" {

int ptb_test_bin_particles(double x0, double y0, double z0, double h, double inv_h, int32_t nx, int32_t ny, int32_t nz,
                           const int32_t *cell_rank, const double *origin, const void *state, const double *mid,
                           const int8_t *flying, int32_t begin, int32_t end, int32_t *pcell, unsigned int *count,
                           unsigned int *sums, int32_t *order, unsigned int *work_count, void *stream) {
  return int(ptb::launch_bin_particles(make_grid(x0, y0, z0, h, inv_h, nx, ny, nz, cell_rank), origin,
                                       static_cast<const ptb::ParticleState *>(state), mid, flying, begin, end, pcell,
                                       count, sums, order, work_count, static_cast<cudaStream_t>(stream)));
}

int ptb_test_bin_pack_particles(double x0, double y0, double z0, double h, double inv_h, int32_t nx, int32_t ny,
                                int32_t nz, const int32_t *cell_rank, const double *origin, const double *dest,
                                const double *weights, const int8_t *flying, const void *state, int32_t begin,
                                int32_t end, int32_t *pcell, unsigned int *count, unsigned int *sums, void *rows,
                                unsigned int *work_count, int midpoint_key, void *stream) {
  return int(ptb::launch_bin_pack_particles(make_grid(x0, y0, z0, h, inv_h, nx, ny, nz, cell_rank), origin, dest,
                                            weights, flying, static_cast<const ptb::ParticleState *>(state), begin,
                                            end, pcell, count, sums, static_cast<ptb::PackedRow *>(rows), work_count,
                                            midpoint_key != 0, static_cast<cudaStream_t>(stream)));
}

int ptb_test_sum_flying_weights(const int8_t *flying, const double *weights, int32_t begin, int32_t end, double *total,
                                void *stream) {
  return int(ptb::launch_sum_flying_weights(flying, weights, begin, end, total, static_cast<cudaStream_t>(stream)));
}

}  // extern "C"
