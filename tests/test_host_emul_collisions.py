"""The collision estimator's per-event step (walk_core.cuh, collision_event) behind point location (locate_point),
compiled for the host by g++ as a TEST-ONLY build (tests/host_emul/emul_collisions.cpp) in both rounding flavours,
against a numpy reference (tests/collisions_ref.py) on the Kuhn, renumbered Delaunay, L-shaped and carved-void meshes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from collisions_ref import assert_close, event_mix, reference_collisions
from helpers import HERE, ROOT
from locate_ref import MESHES

_LIBS = {}


def collide_lib(fma):
    if fma not in _LIBS:
        so = os.path.join(HERE, "host_emul", "libptb_collide_fma.so" if fma else "libptb_collide.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_collisions.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
                os.path.join(csrc, "osh_reader.cpp"), os.path.join(csrc, "gmsh_reader.cpp")]
        deps = srcs + [os.path.join(HERE, "host_emul", "emul_locate.cpp")] + \
            [os.path.join(csrc, h) for h in ("walk_core.cuh", "tet_mesh.hpp", "seed_grid.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp",
                                   *(["-mfma", "-ffp-contract=fast"] if fma else ["-ffp-contract=off"]),
                                   "-I", csrc, "-I", os.path.join(ROOT, "include"), *srcs, "-o", so, "-lz"])
        L = C.CDLL(so)
        L.ptb_locate_create.restype = C.c_void_p
        L.ptb_locate_create.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        L.ptb_locate_destroy.argtypes = [C.c_void_p]
        L.ptb_collide_centre.argtypes = [C.c_void_p, C.c_void_p]
        L.ptb_collide.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                  C.c_void_p]
        _LIBS[fma] = L
    return _LIBS[fma]


def _ptr(a):
    return None if a is None else a.ctypes.data


def collide(L, h, nelem, pts, w, r, bins, times, nscores, nbins, edges, moments):
    T = 1 if edges is None else len(edges) - 1
    m0 = np.empty((T, nbins, nscores, nelem))
    R = np.empty(m0.shape + (3,))
    counts = np.zeros(3, dtype=np.uint64)
    ed = None if edges is None else np.ascontiguousarray(edges, dtype=np.float64)
    L.ptb_collide(h, _ptr(pts), len(pts), _ptr(w), _ptr(r), _ptr(bins), _ptr(times), nscores, nbins, _ptr(ed),
                  0 if edges is None else len(edges) - 1, moments, m0.ctypes.data, R.ctypes.data, counts.ctypes.data)
    return m0, R, tuple(int(c) for c in counts)


EDGES = np.array([0.0, 1.0, 2.5, 3.0, 4.0])
CASES = {  # nscores, nbins, time edges, moments, responses given, bins given
    "s1": (1, 1, None, 0, False, False),
    "s1_mo_t": (1, 1, EDGES, 1, False, True),
    "s3_b3_t": (3, 3, EDGES, 0, True, True),
    "s3_b3_mo": (3, 3, None, 1, True, True),
    "s8_b2_t_mo": (8, 2, EDGES, 1, True, True),
}


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mesh", list(MESHES))
def test_events_match_the_numpy_reference(mesh, case, fma):
    nscores, nbins, edges, moments, with_r, with_bins = CASES[case]
    c, t = MESHES[mesh]()
    L = collide_lib(fma)
    h = L.ptb_locate_create(np.ascontiguousarray(c).ctypes.data, len(c),
                            np.ascontiguousarray(t, dtype=np.int32).ctypes.data, len(t))
    assert h
    try:
        centre = np.empty(3)
        L.ptb_collide_centre(h, centre.ctypes.data)
        rng = np.random.default_rng(len(case) * 7 + len(mesh))
        pts, elem, w, r, bins, times = event_mix(mesh, c, t, rng, 1500, nscores, nbins, edges)
        if not with_r:
            r = None
        if not with_bins:
            bins = None
        m0, R, counts = collide(L, h, len(t), pts, w, r, bins, times, nscores, nbins, edges, moments)
        wm0, wR, a0, aR, wcounts = reference_collisions(elem, pts, w, r, bins, times, nbins, edges, len(t), centre)
        assert counts == wcounts
        assert wcounts[0] > 250 and wcounts[1] > 50 and wcounts[2] >= 7
        assert_close(m0, wm0, a0, f"{mesh} {case} m0")
        if moments:
            assert_close(R, wR, aR, f"{mesh} {case} R")
        else:
            assert not R.any()
    finally:
        L.ptb_locate_destroy(h)


def test_time_bin_edges_belong_to_the_bin_above():
    """Times exactly on an edge go to the bin above it; T_0 is tallied, T_n and later are not, nor anything before
    T_0."""
    c, t = MESHES["kuhn"]()
    L = collide_lib(False)
    h = L.ptb_locate_create(np.ascontiguousarray(c).ctypes.data, len(c),
                            np.ascontiguousarray(t, dtype=np.int32).ctypes.data, len(t))
    try:
        p = np.array([[0.5, 0.5, 0.5]])
        for time, want in ((0.0, 0), (1.0, 1), (2.5, 2), (np.nextafter(2.5, 0.0), 1), (4.0, None), (-1e-300, None),
                           (3.999, 3)):
            m0, _, counts = collide(L, h, len(t), p, np.ones(1), None, None, np.array([time]), 1, 1, EDGES, 0)
            got = np.nonzero(m0.sum(axis=(1, 2, 3)))[0]
            assert (list(got) == ([] if want is None else [want])), (time, got)
            assert counts == ((1, 0, 0) if want is not None else (0, 0, 0))
    finally:
        L.ptb_locate_destroy(h)
