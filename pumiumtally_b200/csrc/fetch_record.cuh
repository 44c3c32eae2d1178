// The tet-record fetch of the point-location kernels (locate_kernels.cu, ww_kernels.cu), so that every kernel that
// calls locate_point reads the records the same way.
#pragma once
#include <cstdint>

#include "tet_mesh.hpp"

namespace ptb {

// One tet record as four 32-byte sectors, two 128-bit read-only loads each.
__device__ __forceinline__ void fetch_record(const TetRecord *tets, int32_t e, double (&r)[16]) {
  const double *p = tets[e].d;
#pragma unroll
  for (int f = 0; f < 4; ++f)
    asm volatile(
        "ld.global.nc.v2.f64 {%0,%1}, [%4];\n\t"
        "ld.global.nc.v2.f64 {%2,%3}, [%4+16];"
        : "=d"(r[4 * f]), "=d"(r[4 * f + 1]), "=d"(r[4 * f + 2]), "=d"(r[4 * f + 3])
        : "l"(p + 4 * f));
}

}  // namespace ptb
