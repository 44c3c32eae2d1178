"""The timed tally step of the CUDA kernels (walk_core.cuh, scored walk with a time filter), compiled for the host
by g++ as a TEST-ONLY build (tests/host_emul/emul_time.cpp) and checked against the oracle: time bin j of score k
must be the brute-force tally of the flights' pieces that lie in bin j, with weights w * r[:, k], in both rounding
flavours."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT, assert_flux_close, assert_positions_close
from oracle.oracle import OraclePumiTally
from pumiumtally_b200.mesh import delaunay_box, kuhn_box
from pumiumtally_b200.workload import SyntheticWorkload
from test_host_emul_scores import ScoredEmul, responses
from time_bins_ref import edge_crossings, reference_time_tally, time_workload

_LIBS = {}


def timed_lib(fma):
    if fma not in _LIBS:
        so = os.path.join(HERE, "host_emul", "libptb_timed_fma.so" if fma else "libptb_timed.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_time.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
                os.path.join(csrc, "osh_reader.cpp"), os.path.join(csrc, "gmsh_reader.cpp")]
        deps = srcs + [os.path.join(csrc, h) for h in ("walk_core.cuh", "tet_mesh.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp",
                                   *(["-mfma", "-ffp-contract=fast"] if fma else ["-ffp-contract=off"]),
                                   "-I", csrc, "-I", os.path.join(ROOT, "include"), *srcs, "-o", so, "-lz"])
        L = C.CDLL(so)
        L.ptb_timed_create.restype = C.c_void_p
        L.ptb_timed_create.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                       C.c_int]
        L.ptb_timed_destroy.argtypes = [C.c_void_p]
        L.ptb_timed_localize.argtypes = [C.c_void_p, C.c_void_p]
        L.ptb_timed_move.argtypes = [C.c_void_p] * 8
        L.ptb_timed_get.argtypes = [C.c_void_p] * 5
        _LIBS[fma] = L
    return _LIBS[fma]


class TimedEmul:
    def __init__(self, coords, t2v, n, nscores, edges, fma):
        self._L = timed_lib(fma)
        coords = np.ascontiguousarray(coords, dtype=np.float64)
        t2v = np.ascontiguousarray(t2v, dtype=np.int32)
        self.edges = np.ascontiguousarray(edges, dtype=np.float64)
        self.n, self.nscores, self.ne, self.nt = n, nscores, len(t2v), len(edges) - 1
        self._h = self._L.ptb_timed_create(coords.ctypes.data, len(coords), t2v.ctypes.data, len(t2v), n, nscores,
                                           self.edges.ctypes.data, len(self.edges))
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.ptb_timed_destroy(self._h)

    def CopyInitialPosition(self, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float64)
        self._L.ptb_timed_localize(self._h, xyz.ctypes.data)

    def move(self, o, d, f, w, r, times, speeds):
        o, d, w, times, speeds = (np.ascontiguousarray(a, dtype=np.float64) for a in (o, d, w, times, speeds))
        r = None if r is None else np.ascontiguousarray(r, dtype=np.float64)
        self._L.ptb_timed_move(self._h, o.ctypes.data, d.ctypes.data, f.ctypes.data, w.ctypes.data,
                               None if r is None else r.ctypes.data, times.ctypes.data, speeds.ctypes.data)

    def get(self):
        flux = np.empty((self.nt, self.nscores, self.ne))
        elem = np.empty(self.n, dtype=np.int32)
        pos = np.empty((self.n, 3))
        st = np.zeros(4, dtype=np.uint64)
        self._L.ptb_timed_get(self._h, flux.ctypes.data, elem.ctypes.data, pos.ctypes.data, st.ctypes.data)
        return flux, elem, pos, dict(segments=int(st[0]), tracks=int(st[1]), relocations=int(st[2]), lost=int(st[3]))


MESHES = {"kuhn": lambda: (kuhn_box(6, 5, 4), (6.0, 5.0, 4.0)), "delaunay": lambda: (delaunay_box(600), (1.0, 1.0, 1.0))}
EDGES = np.linspace(0.0, 4.0, 9)


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("nscores", [1, 3])
@pytest.mark.parametrize("mesh", ["kuhn", "delaunay"])
def test_timed_step_matches_the_cut_flights(mesh, nscores, fma):
    (c, t), box = MESHES[mesh]()
    n = 3000
    wl = SyntheticWorkload(box=box, num_particles=n, mean_length=0.5 * min(box), seed=17)
    rng = np.random.default_rng(nscores + 5)
    eng = TimedEmul(c, t, n, nscores, EDGES, fma)
    orc = OraclePumiTally(c, t, n)
    init = wl.initial_positions()
    for e in (eng, orc):
        e.CopyInitialPosition(init.reshape(-1).copy())
    want = np.zeros((len(EDGES) - 1, nscores, len(t)))
    crossings = []
    for step in range(3):
        o, d, f, w = wl.next_step()
        r = responses(rng, n, nscores) if nscores > 1 else None
        times, speeds = time_workload(rng, o, d, min(box), EDGES)
        f1 = f.copy()
        eng.move(o.reshape(-1), d.reshape(-1), f1, w, r, times, speeds)
        assert not f1.any()
        orc.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w)
        alive = f == 1
        # the flight starts at the origin and ends where the plain move stopped (a hull clip ends it)
        want += reference_time_tally(c, t, o, orc.positions, times, speeds, EDGES, alive, w,
                                     np.ones((n, 1)) if r is None else r)
        crossings.append(edge_crossings(o, d, times, speeds, EDGES, alive)[alive])
        flux, elem, pos, st = eng.get()
        for j in range(len(EDGES) - 1):
            for k in range(nscores):
                assert_flux_close(flux[j, k], want[j, k], f"{mesh} time {j} score {k} step {step}")
        np.testing.assert_array_equal(elem, orc.elem_ids)
        assert_positions_close(pos, orc.positions, f"{mesh} step {step}")
    cr = np.concatenate(crossings)
    assert (cr >= 1).mean() > 0.4 and (cr >= 2).mean() > 0.05, "the inputs must cross edges, some several"
    assert st["segments"] == orc.n_segments and st["tracks"] == orc.n_tracks and st["lost"] == 0


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
def test_exact_hits_on_edges(fma):
    """A track starting exactly on an edge belongs to the bin above it; a flight ending exactly on an edge adds
    nothing to the bin above that edge."""
    c, t = kuhn_box(6, 5, 4)
    n = 4
    edges = np.array([0.0, 1.0, 2.0, 3.0, 4.0])
    eng = TimedEmul(c, t, n, 1, edges, fma)
    orc = OraclePumiTally(c, t, n)
    # straight flights of length exactly 1 along x, through generic y, z
    o = np.array([[1.25, 2.375, 1.3125], [3.25, 1.625, 2.5625], [0.5, 3.875, 0.6875], [2.0, 0.8125, 3.1875]])
    d = o + np.array([1.0, 0.0, 0.0])
    for e in (eng, orc):
        e.CopyInitialPosition(o.reshape(-1).copy())
    w = np.array([1.0, 0.5, 2.0, 1.5])
    # (0) starts on edge 1, ends on edge 3: bins 1 and 2 only;  (1) starts on edge 2, ends inside bin 2
    # (2) starts on the last edge: nothing;  (3) starts inside bin 0, ends on edge 1: bin 0 only
    times = np.array([1.0, 2.0, 4.0, 0.5])
    speeds = np.array([0.5, 4.0, 1.0, 2.0])
    f = np.ones(n, dtype=np.int8)
    eng.move(o.reshape(-1), d.reshape(-1), f.copy(), w, None, times, speeds)
    flux, elem, pos, st = eng.get()
    want = reference_time_tally(c, t, o, d, times, speeds, edges, f == 1, w, np.ones((n, 1)))
    for j in range(4):
        assert_flux_close(flux[j, 0], want[j, 0], f"time {j}")
    per_particle = []
    for i in range(n):
        one = TimedEmul(c, t, n, 1, edges, fma)
        one.CopyInitialPosition(o.reshape(-1).copy())
        fi = np.zeros(n, dtype=np.int8)
        fi[i] = 1
        one.move(o.reshape(-1), d.reshape(-1), fi, w, None, times, speeds)
        per_particle.append(one.get()[0][:, 0].sum(axis=1))
    per_particle = np.array(per_particle)  # [particle, time bin]
    assert per_particle[0, 0] == 0.0 and per_particle[0, 3] == 0.0
    np.testing.assert_allclose(per_particle[0, 1:3], [0.5, 0.5], rtol=1e-12)
    assert per_particle[1, :2].sum() == 0.0 and per_particle[1, 3] == 0.0
    np.testing.assert_allclose(per_particle[1, 2], 0.5, rtol=1e-12)
    assert not per_particle[2].any()
    assert per_particle[3, 1:].sum() == 0.0
    np.testing.assert_allclose(per_particle[3, 0], 1.5, rtol=1e-12)
    orc.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w)
    np.testing.assert_array_equal(elem, orc.elem_ids)
    assert st["lost"] == 0


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("edges", [[-100.0, 100.0], [-100.0, 0.5, 1.0, 2.0, 100.0]], ids=["one_bin", "four_bins"])
def test_enclosing_edges_conserve_the_untimed_tally(edges, fma):
    (c, t), box = MESHES["delaunay"]()
    n, nscores = 2500, 3
    edges = np.array(edges)
    wl = SyntheticWorkload(box=box, num_particles=n, mean_length=0.5, seed=4)
    rng = np.random.default_rng(9)
    eng = TimedEmul(c, t, n, nscores, edges, fma)
    ref = ScoredEmul(c, t, n, nscores, fma)
    init = wl.initial_positions()
    for e in (eng, ref):
        e.CopyInitialPosition(init.reshape(-1).copy())
    for _ in range(2):
        o, d, f, w = wl.next_step()
        r = responses(rng, n, nscores)
        times, speeds = time_workload(rng, o, d, 1.0, np.array([0.0, 0.5, 1.0, 2.0]))
        eng.move(o.reshape(-1), d.reshape(-1), f.copy(), w, r, times, speeds)
        ref.move(o.reshape(-1), d.reshape(-1), f.copy(), w, r)
    flux, elem, pos, st = eng.get()
    want, welem, wpos, wst = ref.get()
    if len(edges) == 2:  # one bin holding every flight: the scored step's reductions, operand for operand
        np.testing.assert_array_equal(flux[0], want)
    for k in range(nscores):
        assert_flux_close(flux[:, k].sum(axis=0), want[k], f"score {k}")
    np.testing.assert_array_equal(elem, welem)
    np.testing.assert_array_equal(pos, wpos)
    assert st == wst


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
def test_non_finite_or_non_positive_times_and_speeds_are_lost_flights(fma):
    c, t = kuhn_box(5, 5, 5)
    n, nscores = 2000, 2
    edges = np.linspace(0.0, 3.0, 7)
    wl = SyntheticWorkload(box=(5.0, 5.0, 5.0), num_particles=n, seed=5)
    rng = np.random.default_rng(3)
    eng = TimedEmul(c, t, n, nscores, edges, fma)
    orc = OraclePumiTally(c, t, n)
    init = wl.initial_positions()
    for e in (eng, orc):
        e.CopyInitialPosition(init.reshape(-1).copy())
    o, d, f, w = wl.next_step()
    f[:] = 1
    o[:] = init  # no relocation: a lost flight leaves the particle where it is
    r = responses(rng, n, nscores)
    times, speeds = time_workload(rng, o, d, 5.0, edges)
    bad = np.arange(0, 80)
    times[bad[:10]] = np.nan
    times[bad[10:20]] = np.inf
    times[bad[20:30]] = -np.inf
    speeds[bad[30:40]] = 0.0
    speeds[bad[40:50]] = -1.0
    speeds[bad[50:60]] = np.inf
    speeds[bad[60:70]] = np.nan
    speeds[bad[70:80]] = -0.0
    eng.move(o.reshape(-1), d.reshape(-1), f.copy(), w, r, times, speeds)
    f_ref = f.copy()
    f_ref[bad] = 0
    orc.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f_ref.copy(), w)
    alive = f_ref == 1
    want = reference_time_tally(c, t, o, orc.positions, np.nan_to_num(times), np.nan_to_num(speeds, posinf=1.0),
                                edges, alive, w, r)
    flux, elem, pos, st = eng.get()
    assert np.isfinite(flux).all() and np.isfinite(pos).all()
    for j in range(len(edges) - 1):
        for k in range(nscores):
            assert_flux_close(flux[j, k], want[j, k], f"time {j} score {k}")
    np.testing.assert_array_equal(elem, orc.elem_ids)
    np.testing.assert_array_equal(pos[bad], init[bad])
    assert st["lost"] == len(bad)
