"""The region-sum order (batch_stats.cuh: build_region_plan, chunk_sum, region_sums_host) compiled for the host by g++
as a TEST-ONLY build (tests/host_emul/emul_regions.cpp), against math.fsum.  The region kernel of stats_kernels.cu runs
the same chunk_sum over the same plan, and the engine sums the region volumes with region_sums_host."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT

_LIB = []
U = 2.0 ** -53  # unit roundoff of double


def regions_lib():
    if not _LIB:
        so = os.path.join(HERE, "host_emul", "libptb_regions.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        src = os.path.join(HERE, "host_emul", "emul_regions.cpp")
        deps = [src] + [os.path.join(csrc, h) for h in ("batch_stats.cuh", "walk_core.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off",
                                   "-I", csrc, src, "-o", so])
        L = C.CDLL(so)
        L.ptb_region_sums.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
        L.ptb_region_sums.restype = C.c_int32
        L.ptb_region_chunk.restype = C.c_int32
        _LIB.append(L)
    return _LIB[0]


def region_sums(region, nregions, values):
    region = np.ascontiguousarray(region, dtype=np.int32)
    values = np.ascontiguousarray(values, dtype=np.float64)
    out = np.empty(nregions)
    levels = regions_lib().ptb_region_sums(region.ctypes.data, len(region), nregions, values.ctypes.data,
                                           out.ctypes.data)
    return out, levels


def check_against_fsum(region, nregions, values):
    """Every region's sum within the bound of the order: each level adds at most kRegionChunk terms left to right, so
    the error is at most h u / (1 - h u) * sum |x| with h = levels * (kRegionChunk - 1)."""
    got, levels = region_sums(region, nregions, values)
    h = levels * (regions_lib().ptb_region_chunk() - 1)
    for g in range(nregions):
        x = values[region == g]
        want = math.fsum(x)
        bound = h * U / (1 - h * U) * math.fsum(np.abs(x))
        assert abs(got[g] - want) <= bound, (g, len(x), got[g], want, bound)
    return got, levels


def test_chunk_is_32():
    assert regions_lib().ptb_region_chunk() == 32


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_region_sizes_around_the_chunk(seed):
    """Regions of 0, 1, chunk - 1, chunk, chunk + 1 and a few thousand elements, interleaved, plus elements in none."""
    rng = np.random.default_rng(seed)
    C_ = regions_lib().ptb_region_chunk()
    sizes = [0, 1, C_ - 1, C_, C_ + 1, 2 * C_ + 1, C_ * C_, C_ * C_ + 1, 3000]
    region = np.concatenate([np.full(s, g, dtype=np.int32) for g, s in enumerate(sizes)] + [np.full(500, -1, np.int32)])
    rng.shuffle(region)
    values = rng.lognormal(0.0, 2.0, len(region)) * rng.choice([-1.0, 1.0], len(region))
    got, levels = check_against_fsum(region, len(sizes), values)
    assert got[0] == 0.0                                  # empty: 0
    assert got[1] == values[region == 1][0]               # one element: its value, bit for bit
    assert levels == 3                                    # 3000 elements: 94 chunks, then 3, then 1
    again, _ = region_sums(region, len(sizes), values)
    assert again.tobytes() == got.tobytes()               # the same bits every time


def test_one_region_holds_all_elements_but_one():
    rng = np.random.default_rng(5)
    E = 40000
    region = np.zeros(E, dtype=np.int32)
    region[rng.integers(E)] = -1
    values = rng.uniform(0.0, 1.0, E)
    got, levels = check_against_fsum(region, 1, values)
    assert levels == 4  # 39,999 -> 1250 -> 40 -> 2 -> 1


def test_every_element_its_own_region():
    """nregions == E single-element regions: one level, every sum the element's value itself (also -0.0)."""
    rng = np.random.default_rng(8)
    E = 3001
    perm = rng.permutation(E).astype(np.int32)
    values = rng.normal(0.0, 1.0, E)
    values[:5] = -0.0
    got, levels = region_sums(perm, E, values)
    assert levels == 1
    want = np.empty(E)
    want[perm] = values
    assert got.tobytes() == want.tobytes()


def test_order_is_ascending_internal_id():
    """Within a chunk the sum runs left to right in ascending element id: 1 + 1e16 - 1e16 ... is order-dependent."""
    region = np.zeros(3, dtype=np.int32)
    got, _ = region_sums(region, 1, np.array([1.0, 1e16, -1e16]))
    assert got[0] == (1.0 + 1e16) - 1e16 == 0.0
    got, _ = region_sums(region, 1, np.array([1e16, -1e16, 1.0]))
    assert got[0] == 1.0
