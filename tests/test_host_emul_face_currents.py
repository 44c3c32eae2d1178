"""The face-current crossing step of the CUDA kernels (walk_core.cuh, CU in advance and start_tally_to), compiled for
the host by g++ as a TEST-ONLY build (tests/host_emul/emul_face_currents.cpp), in both rounding flavours.  Checked bit
for bit against the exact clip-and-walk reference (tests/face_currents_ref.py): the interior slot (next, back), the hull
slot (e, back), nothing for a relocation, the end of a flight, a face the iteration limit stopped the walk at or a bad
track, and the time bin of each crossing.  Weights are dyadic (k / 8), so every sum is exact in any order."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from face_currents_ref import face_walk, reference_currents, unit_planes
from helpers import HERE, ROOT, l_shaped_mesh
from pumiumtally_b200.mesh import delaunay_box, kuhn_box

EDGES = np.linspace(0.0, 4.0, 9)
MESHES = {
    "box": lambda: kuhn_box(5, 4, 3, 2.5, 1.0, 0.75),
    "kuhn": lambda: kuhn_box(6, 5, 4),
    "delaunay": lambda: delaunay_box(600),
    "l_shaped": lambda: l_shaped_mesh(6, 6, 3),
}
_LIBS = {}


def currents_lib(fma):
    if fma not in _LIBS:
        so = os.path.join(HERE, "host_emul", "libptb_currents_fma.so" if fma else "libptb_currents.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_face_currents.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
                os.path.join(csrc, "osh_reader.cpp"), os.path.join(csrc, "gmsh_reader.cpp")]
        deps = srcs + [os.path.join(csrc, h) for h in ("walk_core.cuh", "tet_mesh.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp",
                                   *(["-mfma", "-ffp-contract=fast"] if fma else ["-ffp-contract=off"]),
                                   "-I", csrc, "-I", os.path.join(ROOT, "include"), *srcs, "-o", so, "-lz"])
        L = C.CDLL(so)
        L.ptb_currents_create.restype = C.c_void_p
        L.ptb_currents_create.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                          C.c_int, C.c_int, C.c_int]
        L.ptb_currents_destroy.argtypes = [C.c_void_p]
        L.ptb_currents_localize.argtypes = [C.c_void_p, C.c_void_p]
        L.ptb_currents_move.argtypes = [C.c_void_p] * 8
        L.ptb_currents_get.argtypes = [C.c_void_p] * 7
        _LIBS[fma] = L
    return _LIBS[fma]


class CurrentEmul:
    def __init__(self, coords, t2v, n, nscores=1, edges=None, moments=0, max_iters=0, fma=False):
        self._L = currents_lib(fma)
        coords = np.ascontiguousarray(coords, dtype=np.float64)
        t2v = np.ascontiguousarray(t2v, dtype=np.int32)
        self.edges = None if edges is None else np.ascontiguousarray(edges, dtype=np.float64)
        self.n, self.ne = n, len(t2v)
        self.nt = 1 if edges is None else len(edges) - 1
        self._h = self._L.ptb_currents_create(coords.ctypes.data, len(coords), t2v.ctypes.data, len(t2v), n, nscores,
                                              None if edges is None else self.edges.ctypes.data,
                                              0 if edges is None else len(self.edges), moments, max_iters)
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.ptb_currents_destroy(self._h)

    def localize(self, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float64)
        self._L.ptb_currents_localize(self._h, xyz.ctypes.data)

    def move(self, o, d, f, w, r=None, times=None, speeds=None):
        o, d, w = (np.ascontiguousarray(a, dtype=np.float64) for a in (o, d, w))
        f = np.ascontiguousarray(f, dtype=np.int8)
        arrs = [None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in (r, times, speeds)]
        self._L.ptb_currents_move(self._h, o.ctypes.data, d.ctypes.data, f.ctypes.data, w.ctypes.data,
                                  *(None if a is None else a.ctypes.data for a in arrs))

    def get(self):
        out = np.empty((self.nt, self.ne, 4))
        inn = np.empty((self.nt, self.ne, 4))
        adj = np.empty((self.ne, 4), dtype=np.int32)
        elem = np.empty(self.n, dtype=np.int32)
        pos = np.empty((self.n, 3))
        stats = np.zeros(4, dtype=np.uint64)
        self._L.ptb_currents_get(self._h, out.ctypes.data, inn.ctypes.data, adj.ctypes.data, elem.ctypes.data,
                                 pos.ctypes.data, stats.ctypes.data)
        return out, inn, adj.astype(np.int64), elem, pos, stats


def _interior_points(rng, coords, t2v, n):
    lam = 0.02 + 0.92 * rng.dirichlet(np.ones(4), n)
    lam /= lam.sum(axis=1, keepdims=True)
    tets = rng.integers(0, len(t2v), n)
    return np.ascontiguousarray(np.einsum("iq,iqk->ik", lam, coords[t2v[tets]])), tets


def _check(mesh, fma, nscores=1, timed=False, moments=0, max_iters=0, relocate=False, steps=2, n=3000, seed=0):
    """Moves of the host build against the reference.  relocate: each flight starts with a relocation (tally off) from
    the particle's last position, weighted like the flight (convex meshes); otherwise a weight-0 positioning move puts
    every particle at its origin first.  A few flights have a non-finite weight or destination (bad tracks)."""
    coords, t2v = MESHES[mesh]()
    rng = np.random.default_rng(seed)
    edges = EDGES if timed else None
    emul = CurrentEmul(coords, t2v, n, nscores, edges, moments, max_iters, fma)
    _, _, adj, _, _, _ = emul.get()
    planes = unit_planes(coords, t2v)
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    scale = (hi - lo).max()
    init, _ = _interior_points(rng, coords, t2v, n)
    emul.localize(init)
    want_out = np.zeros((emul.nt, 1, len(t2v), 4))
    want_in = np.zeros_like(want_out)
    for step in range(steps):
        o, tets = _interior_points(rng, coords, t2v, n)
        w = rng.integers(1, 17, n) / 8.0
        r = rng.uniform(0.0, 2.0, (n, nscores)) if nscores > 1 else None
        if relocate:
            start, ok = tets, np.ones(n, dtype=bool)
        else:
            emul.move(o, o, np.ones(n, np.int8), np.zeros(n), r, np.zeros(n) if timed else None,
                      np.ones(n) if timed else None)
            _, _, _, elem, pos, _ = emul.get()
            start, ok = elem.astype(np.int64), (pos == o).all(axis=1)
        u = rng.normal(size=(n, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        d = o + u * rng.exponential(0.5 * scale, n)[:, None]
        times = rng.uniform(EDGES[0] - 1.0, EDGES[-1] + 0.5, n)
        speeds = rng.uniform(0.3, 3.0, n)
        tpp = np.linalg.norm(d - o, axis=1) / speeds
        fly = ok & (rng.random(n) < 0.9)
        bad_w, bad_d = fly & (rng.random(n) < 0.02), fly & (rng.random(n) < 0.02)
        good = fly & ~bad_w & ~bad_d
        cr = face_walk(planes, adj, start, o, d, good, times, tpp, edges, max_iters or None)
        fly &= ~cr[4]
        good &= ~cr[4]
        cr = face_walk(planes, adj, start, o, d, good, times, tpp, edges, max_iters or None)
        assert not cr[4][good].any()
        a, b = reference_currents(adj, cr, w, None, emul.nt, 1)
        want_out += a
        want_in += b
        w_in, d_in = w.copy(), d.copy()
        w_in[bad_w] = np.nan
        d_in[bad_d] = np.inf
        emul.move(o, d_in, fly.astype(np.int8), w_in, r, times if timed else None, speeds if timed else None)
    out, inn, _, _, _, stats = emul.get()
    label = f"{mesh} fma={fma} nscores={nscores} timed={timed} moments={moments} max_iters={max_iters}"
    np.testing.assert_array_equal(out, want_out[:, 0], err_msg=label + " outgoing")
    np.testing.assert_array_equal(inn, want_in[:, 0], err_msg=label + " incoming")
    assert want_out.sum() > 0, "no crossing tested"
    # (three crossings seldom reach the hull of the Delaunay ball)
    assert max_iters or (want_out[:, 0] * (adj < 0)).sum() > 0, "no hull crossing tested"
    return stats


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("mesh", sorted(MESHES))
def test_crossings_match_the_exact_reference(mesh, fma):
    _check(mesh, fma, seed=1)


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("moments", [0, 1])
@pytest.mark.parametrize("mesh", ["kuhn", "delaunay", "l_shaped"])
def test_time_bin_of_each_crossing(mesh, moments, fma):
    _check(mesh, fma, nscores=1, timed=True, moments=moments, seed=2)


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("mesh", ["box", "delaunay"])
def test_currents_are_weight_not_response(mesh, fma):
    _check(mesh, fma, nscores=3, seed=3)


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("mesh", ["box", "kuhn", "delaunay"])
def test_relocation_adds_nothing(mesh, fma):
    stats = _check(mesh, fma, relocate=True, seed=4)
    assert stats[2] > 0  # relocations crossed faces, tally off


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("mesh", ["kuhn", "delaunay"])
def test_nothing_at_the_iteration_limit(mesh, fma):
    stats = _check(mesh, fma, max_iters=3, seed=5)
    assert stats[3] > 0  # walks the limit stopped
