"""The point-location step of the CUDA kernels (walk_core.cuh, locate_point), compiled for the host by g++ as a TEST-ONLY
build (tests/host_emul/emul_locate.cpp), in both rounding flavours, against a brute-force barycentric reference
(tests/locate_ref.py) on convex (Kuhn, renumbered Delaunay) and non-convex (L-shaped, carved void) meshes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT
from locate_ref import (MESHES, _inside_shape, assert_contains, band_points, barycentric, generic_points,
                        non_finite_points, outside_points, special_points)

_LIBS = {}


def locate_lib(fma):
    if fma not in _LIBS:
        so = os.path.join(HERE, "host_emul", "libptb_locate_fma.so" if fma else "libptb_locate.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_locate.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
                os.path.join(csrc, "osh_reader.cpp"), os.path.join(csrc, "gmsh_reader.cpp")]
        deps = srcs + [os.path.join(csrc, h) for h in ("walk_core.cuh", "tet_mesh.hpp", "seed_grid.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp",
                                   *(["-mfma", "-ffp-contract=fast"] if fma else ["-ffp-contract=off"]),
                                   "-I", csrc, "-I", os.path.join(ROOT, "include"), *srcs, "-o", so, "-lz"])
        L = C.CDLL(so)
        L.ptb_locate_create.restype = C.c_void_p
        L.ptb_locate_create.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        L.ptb_locate_destroy.argtypes = [C.c_void_p]
        L.ptb_locate_hull_convex.argtypes = [C.c_void_p]
        L.ptb_locate_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.ptb_locate_grid.restype = C.c_int64
        L.ptb_locate_grid.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ptb_locate_candidates.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _LIBS[fma] = L
    return _LIBS[fma]


class LocateEmul:
    def __init__(self, coords, t2v, fma):
        self._L = locate_lib(fma)
        c = np.ascontiguousarray(coords, dtype=np.float64)
        t = np.ascontiguousarray(t2v, dtype=np.int32)
        self._h = self._L.ptb_locate_create(c.ctypes.data, len(c), t.ctypes.data, len(t))
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.ptb_locate_destroy(self._h)

    @property
    def hull_convex(self):
        return bool(self._L.ptb_locate_hull_convex(self._h))

    def locate(self, pts):
        p = np.ascontiguousarray(pts, dtype=np.float64).reshape(-1, 3)
        out = np.empty(len(p), dtype=np.int32)
        self._L.ptb_locate_points(self._h, p.ctypes.data, len(p), out.ctypes.data)
        return out

    def candidates(self):
        dims = np.zeros(3, dtype=np.int32)
        geom = np.zeros(5)
        m = self._L.ptb_locate_grid(self._h, dims.ctypes.data, geom.ctypes.data)
        off = np.empty(int(dims.prod()) + 1, dtype=np.int64)
        tets = np.empty(max(m, 1), dtype=np.int32)
        self._L.ptb_locate_candidates(self._h, off.ctypes.data, tets.ctypes.data)
        return dims, geom, off, tets[:m]


FMA = pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
MESH = pytest.mark.parametrize("mesh", list(MESHES))


@FMA
@MESH
def test_generic_points_get_their_unique_tet(mesh, fma):
    c, t = MESHES[mesh]()
    eng = LocateEmul(c, t, fma)
    assert eng.hull_convex == (mesh in ("kuhn", "delaunay"))
    pts, want = generic_points(mesh, c, t, 3000, np.random.default_rng(7))
    assert len(pts) > 1000
    np.testing.assert_array_equal(eng.locate(pts), want)


@FMA
@MESH
def test_vertices_edge_midpoints_and_face_centres_get_an_element_that_contains_them(mesh, fma):
    c, t = MESHES[mesh]()
    eng = LocateEmul(c, t, fma)
    pts = special_points(c, t)
    pts = pts[_inside_shape(mesh, pts, 1e-9)]  # notch and void faces are hull: either answer (test below)
    assert len(pts) > 100
    assert_contains(c, t, pts, eng.locate(pts), mesh)


@FMA
@MESH
def test_points_outside_the_mesh_and_non_finite_points_get_minus_one(mesh, fma):
    c, t = MESHES[mesh]()
    eng = LocateEmul(c, t, fma)
    pts = np.concatenate([outside_points(mesh, c, np.random.default_rng(3)), non_finite_points()])
    got = eng.locate(pts)
    assert (got == -1).all(), pts[got != -1][:5]


@FMA
@MESH
def test_points_in_the_hull_band_get_a_hull_element_or_minus_one(mesh, fma):
    c, t = MESHES[mesh]()
    eng = LocateEmul(c, t, fma)
    pts = band_points(mesh, c, np.random.default_rng(11))
    got = eng.locate(pts)
    hit = got >= 0
    if hit.any():
        lam = barycentric(c, t, pts[hit], got[hit])
        assert (lam >= -1e-8).all()
    assert hit.any()  # most band points are inside the hull planes


@MESH
def test_candidate_lists_are_complete(mesh):
    """Every tet holding a point of a cell is in that cell's list: sampled at the vertices, edge and face points and
    random interior points of every tet, each point's cell found as locate_point finds it."""
    c, t = MESHES[mesh]()
    eng = LocateEmul(c, t, False)
    (nx, ny, nz), (x0, y0, z0, h, inv_h), off, tets = eng.candidates()
    rng = np.random.default_rng(5)
    v = np.asarray(c)[np.asarray(t)]  # [E, 4, 3]
    lam = np.concatenate([np.eye(4), np.full((1, 4), 0.25), rng.dirichlet(np.ones(4), size=24),
                          np.array([[0.5, 0.5, 0, 0], [0, 0.5, 0.5, 0], [1 / 3, 1 / 3, 1 / 3, 0]])])
    pts = np.einsum("sk,ekd->esd", lam, v)  # [E, S, 3]
    f = (pts - np.array([x0, y0, z0])) * inv_h
    dims = np.array([nx, ny, nz])
    ok = (f >= 0).all(2) & (f < dims).all(2)
    cell = (np.floor(f[..., 2]) * ny + np.floor(f[..., 1])) * nx + np.floor(f[..., 0])
    missing = 0
    for e in range(len(t)):
        for cc in np.unique(cell[e][ok[e]]).astype(np.int64):
            missing += e not in set(tets[off[cc]:off[cc + 1]].tolist())
    assert missing == 0
    assert off[-1] == len(tets) and (np.diff(off) >= 0).all()
