"""The moment tally step of the CUDA kernels (walk_core.cuh, moment_tally), compiled for the host by g++ as a
TEST-ONLY build (tests/host_emul/emul_moments.cpp), in both rounding flavours.  The records are centred and solved by
linear_moments() (tet_mesh.cpp), the engine's own function.  Checked against an exact clip-and-sum reference, against
the analytic gradient of a linear flux, and against the same step without moments."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT
from moments_ref import (assert_m0_close, assert_moments_close, reference_moments, tet_geometry,
                         tet_quadrature_moments)
from pumiumtally_b200.mesh import delaunay_box, kuhn_box
from pumiumtally_b200.workload import SyntheticWorkload
from test_host_emul_scores import responses
from time_bins_ref import time_workload

_LIBS = {}


def moments_lib(fma):
    if fma not in _LIBS:
        so = os.path.join(HERE, "host_emul", "libptb_moments_fma.so" if fma else "libptb_moments.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_moments.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
                os.path.join(csrc, "osh_reader.cpp"), os.path.join(csrc, "gmsh_reader.cpp")]
        deps = srcs + [os.path.join(csrc, h) for h in ("walk_core.cuh", "tet_mesh.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp",
                                   *(["-mfma", "-ffp-contract=fast"] if fma else ["-ffp-contract=off"]),
                                   "-I", csrc, "-I", os.path.join(ROOT, "include"), *srcs, "-o", so, "-lz"])
        L = C.CDLL(so)
        L.ptb_moments_create.restype = C.c_void_p
        L.ptb_moments_create.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                         C.c_int, C.c_int]
        L.ptb_moments_destroy.argtypes = [C.c_void_p]
        L.ptb_moments_localize.argtypes = [C.c_void_p, C.c_void_p]
        L.ptb_moments_move.argtypes = [C.c_void_p] * 8
        L.ptb_moments_get.argtypes = [C.c_void_p] * 7
        L.ptb_linear_moments.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _LIBS[fma] = L
    return _LIBS[fma]


class MomentEmul:
    """edges None: the scored step (responses None: every response 1, moments only); moments 0 or 1."""

    def __init__(self, coords, t2v, n, nscores, edges, moments, fma):
        self._L = moments_lib(fma)
        coords = np.ascontiguousarray(coords, dtype=np.float64)
        t2v = np.ascontiguousarray(t2v, dtype=np.int32)
        self.edges = None if edges is None else np.ascontiguousarray(edges, dtype=np.float64)
        self.n, self.nscores, self.ne = n, nscores, len(t2v)
        self.nt = 1 if edges is None else len(edges) - 1
        self._h = self._L.ptb_moments_create(coords.ctypes.data, len(coords), t2v.ctypes.data, len(t2v), n, nscores,
                                             None if edges is None else self.edges.ctypes.data,
                                             0 if edges is None else len(self.edges), moments)
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.ptb_moments_destroy(self._h)

    def CopyInitialPosition(self, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float64)
        self._L.ptb_moments_localize(self._h, xyz.ctypes.data)

    def move(self, o, d, f, w, r=None, times=None, speeds=None):
        o, d, w = (np.ascontiguousarray(a, dtype=np.float64) for a in (o, d, w))
        arrs = [None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in (r, times, speeds)]
        self._L.ptb_moments_move(self._h, o.ctypes.data, d.ctypes.data, f.ctypes.data, w.ctypes.data,
                                 *(None if a is None else a.ctypes.data for a in arrs))

    def get(self):
        m0 = np.empty((self.nt, self.nscores, self.ne))
        m1 = np.zeros((self.nt, self.nscores, self.ne, 3))
        g = np.zeros((self.nt, self.nscores, self.ne, 3))
        elem = np.empty(self.n, dtype=np.int32)
        pos = np.empty((self.n, 3))
        st = np.zeros(4, dtype=np.uint64)
        self._L.ptb_moments_get(self._h, m0.ctypes.data, m1.ctypes.data, g.ctypes.data, elem.ctypes.data,
                                pos.ctypes.data, st.ctypes.data)
        return m0, m1, g, elem, pos, dict(segments=int(st[0]), tracks=int(st[1]), relocations=int(st[2]),
                                          lost=int(st[3]))


MESHES = {"kuhn": lambda: (kuhn_box(6, 5, 4), (6.0, 5.0, 4.0)), "delaunay": lambda: (delaunay_box(600), (1.0, 1.0, 1.0))}
EDGES = np.linspace(0.0, 4.0, 9)


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("timed", [False, True], ids=["untimed", "timed"])
@pytest.mark.parametrize("nscores", [1, 3])
@pytest.mark.parametrize("mesh", ["kuhn", "delaunay"])
def test_moments_match_the_exact_reference(mesh, nscores, timed, fma):
    (c, t), box = MESHES[mesh]()
    n = 3000
    wl = SyntheticWorkload(box=box, num_particles=n, mean_length=0.5 * min(box), seed=23)
    rng = np.random.default_rng(nscores + 11)
    edges = EDGES if timed else None
    eng = MomentEmul(c, t, n, nscores, edges, 1, fma)
    _, diam, _, _ = tet_geometry(c, t)
    init = wl.initial_positions()
    eng.CopyInitialPosition(init.reshape(-1).copy())
    nt = len(EDGES) - 1 if timed else 1
    want0, want1 = np.zeros((nt, nscores, len(t))), np.zeros((nt, nscores, len(t), 3))
    absum, absw = np.zeros((nt, nscores, len(t))), np.zeros((nt, nscores, len(t)))
    # where a piece starts or ends is known to rounding only: the reference and the walk compute a crossing at a
    # grazing angle from different planes, and cut a flight at a time edge at distance (T - t) * v against ray
    # parameter (T - t0) / tpp
    cut = 1e-12 * max(box)
    for step in range(3):
        o, d, f, w = wl.next_step()
        r = responses(rng, n, nscores) if nscores > 1 else None
        times, speeds = time_workload(rng, o, d, min(box), EDGES) if timed else (None, None)
        f1 = f.copy()
        eng.move(o.reshape(-1), d.reshape(-1), f1, w, r, times, speeds)
        assert not f1.any()
        m0, m1, g, elem, pos, st = eng.get()
        # the flight starts at the origin and ends where the walk stopped (a hull clip ends it)
        rr = np.ones((n, 1)) if r is None else r
        a0, a1, ab, aw = reference_moments(c, t, o, pos, f == 1, w, rr, edges, times, speeds)
        want0, want1, absum, absw = want0 + a0, want1 + a1, absum + ab, absw + aw
        assert_m0_close(m0, want0, absum, f"{mesh} step {step}", cut=cut, abs_w=absw)
        assert_moments_close(m1, want1, absum, diam, f"{mesh} step {step}", cut=cut, abs_w=absw)
    assert np.abs(want1).max() > 0 and st["lost"] == 0


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
def test_gradient_of_a_linearly_falling_flux(fma):
    """Parallel tracks along +x from x = 0+, lengths uniform on [0, Lx): the flux is exactly phi0 * (1 - x / Lx)."""
    c, t = kuhn_box(6, 5, 4)
    lx, ly, lz = 6.0, 5.0, 4.0
    n = 400_000
    rng = np.random.default_rng(2024)
    o = np.column_stack([np.full(n, 1e-7), rng.uniform(0, ly, n), rng.uniform(0, lz, n)])
    d = o.copy()
    d[:, 0] += rng.uniform(0.0, lx - 2e-7, n)
    w = np.ones(n)
    eng = MomentEmul(c, t, n, 1, None, 1, fma)
    eng.CopyInitialPosition(o.reshape(-1).copy())
    eng.move(o.reshape(-1), d.reshape(-1), np.ones(n, dtype=np.int8), w)
    m0, m1, g, *_ = eng.get()
    _, _, vol = tet_quadrature_moments(c, t, np.zeros(3), 0.0, np.zeros(3))
    phi0 = n / (ly * lz)
    gm = (g[0, 0] * vol[:, None]).sum(axis=0) / vol.sum()
    np.testing.assert_allclose(gm[0], -phi0 / lx, rtol=0.05)
    assert abs(gm[1]) < 0.05 * phi0 / lx and abs(gm[2]) < 0.05 * phi0 / lx
    np.testing.assert_allclose(m0[0, 0].sum(), (d[:, 0] - o[:, 0]).sum(), rtol=1e-12)


def test_solve_returns_the_gradient_of_a_linear_field():
    """M_e^-1 applied to the exact moments of a linear field is that field's gradient, with the record accumulated
    about the mesh centre as the kernels accumulate it.  (On well-shaped tets; a sliver's M_e is ill-conditioned and
    its solve loses digits accordingly.)"""
    (c, t), _ = MESHES["kuhn"]()
    L = moments_lib(False)
    grad = np.array([0.7, -1.3, 2.1])
    centre = 0.5 * (np.asarray(c).min(axis=0) + np.asarray(c).max(axis=0))
    m0, R, _ = tet_quadrature_moments(c, t, centre, 4.0, grad)
    v = np.ascontiguousarray(np.asarray(c, dtype=np.float64)[np.asarray(t)].reshape(len(t), 12))
    m1, g = np.empty(3), np.empty(3)
    for e in range(len(t)):
        rec = np.ascontiguousarray([m0[e], R[e, 0], R[e, 1], R[e, 2]])
        L.ptb_linear_moments(v[e].ctypes.data, centre.ctypes.data, rec.ctypes.data, 1, 0, m1.ctypes.data, g.ctypes.data)
        np.testing.assert_allclose(g, grad, rtol=1e-12, atol=1e-12 * np.abs(grad).max())


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("timed", [False, True], ids=["scored", "timed"])
def test_moments_change_nothing_else(timed, fma):
    (c, t), box = MESHES["delaunay"]()
    n, nscores = 2500, 3
    wl = SyntheticWorkload(box=box, num_particles=n, mean_length=0.5, seed=8)
    rng = np.random.default_rng(5)
    edges = EDGES / 4 if timed else None
    on = MomentEmul(c, t, n, nscores, edges, 1, fma)
    off = MomentEmul(c, t, n, nscores, edges, 0, fma)
    init = wl.initial_positions()
    for e in (on, off):
        e.CopyInitialPosition(init.reshape(-1).copy())
    for _ in range(2):
        o, d, f, w = wl.next_step()
        r = responses(rng, n, nscores)
        times, speeds = time_workload(rng, o, d, 1.0, edges) if timed else (None, None)
        for e in (on, off):
            e.move(o.reshape(-1), d.reshape(-1), f.copy(), w, r, times, speeds)
    m0, _, _, elem, pos, st = on.get()
    w0, _, _, welem, wpos, wst = off.get()
    if fma:  # g++ may contract the step's product into the host build's += on one side only
        np.testing.assert_allclose(m0, w0, rtol=1e-13, atol=1e-15 * np.abs(w0).max())
    else:  # the same operands, reduced in the same order
        np.testing.assert_array_equal(m0, w0)
    np.testing.assert_array_equal(elem, welem)
    np.testing.assert_array_equal(pos, wpos)
    assert st == wst
