"""H100-native unstructured-mesh track-length tally engine.

The product is ``lib/libpumitally.so`` (CUDA kernels for sm_90a + C++ host side,
C ABI in ``include/pumitally_c.h``, C++ facade ``pumitally::PumiTally``).  This
package holds its sources (``csrc/``), the in-tree build, a ctypes mirror of the
reference interface (``tally.PumiTally``) and the synthetic mesh / particle
generators used by the tests and the benchmark.
"""
from .tally import PumiTally, load_library  # noqa: F401
