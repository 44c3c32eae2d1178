"""The scored tally step of the CUDA kernels (walk_core.cuh instantiated for several scores), compiled for
the host by g++ as a TEST-ONLY build (tests/host_emul/emul_scores.cpp) and checked against the oracle: score
k of a scored move must be the oracle's tally with weights w * r[:, k], in both rounding flavours."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT, assert_flux_close, assert_positions_close
from oracle.oracle import OraclePumiTally
from pumiumtally_b200.mesh import delaunay_box, kuhn_box
from pumiumtally_b200.workload import SyntheticWorkload

_LIBS = {}


def scored_lib(fma):
    if fma not in _LIBS:
        so = os.path.join(HERE, "host_emul", "libptb_scored_fma.so" if fma else "libptb_scored.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_scores.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
                os.path.join(csrc, "osh_reader.cpp"), os.path.join(csrc, "gmsh_reader.cpp")]
        deps = srcs + [os.path.join(csrc, h) for h in ("walk_core.cuh", "tet_mesh.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp",
                                   *(["-mfma", "-ffp-contract=fast"] if fma else ["-ffp-contract=off"]),
                                   "-I", csrc, "-I", os.path.join(ROOT, "include"), *srcs, "-o", so, "-lz"])
        L = C.CDLL(so)
        L.ptb_scored_create.restype = C.c_void_p
        L.ptb_scored_create.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_int]
        L.ptb_scored_destroy.argtypes = [C.c_void_p]
        L.ptb_scored_localize.argtypes = [C.c_void_p, C.c_void_p]
        L.ptb_scored_move.argtypes = [C.c_void_p] * 6
        L.ptb_scored_get.argtypes = [C.c_void_p] * 5
        _LIBS[fma] = L
    return _LIBS[fma]


class ScoredEmul:
    def __init__(self, coords, t2v, n, nscores, fma):
        self._L = scored_lib(fma)
        coords = np.ascontiguousarray(coords, dtype=np.float64)
        t2v = np.ascontiguousarray(t2v, dtype=np.int32)
        self.n, self.nscores, self.ne = n, nscores, len(t2v)
        self._h = self._L.ptb_scored_create(coords.ctypes.data, len(coords), t2v.ctypes.data, len(t2v), n, nscores)
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.ptb_scored_destroy(self._h)

    def CopyInitialPosition(self, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float64)
        self._L.ptb_scored_localize(self._h, xyz.ctypes.data)

    def move(self, o, d, f, w, r):
        o, d, w, r = (np.ascontiguousarray(a, dtype=np.float64) for a in (o, d, w, r))
        self._L.ptb_scored_move(self._h, o.ctypes.data, d.ctypes.data, f.ctypes.data, w.ctypes.data, r.ctypes.data)

    def get(self):
        flux = np.empty((self.nscores, self.ne))
        elem = np.empty(self.n, dtype=np.int32)
        pos = np.empty((self.n, 3))
        st = np.zeros(4, dtype=np.uint64)
        self._L.ptb_scored_get(self._h, flux.ctypes.data, elem.ctypes.data, pos.ctypes.data, st.ctypes.data)
        return flux, elem, pos, dict(segments=int(st[0]), tracks=int(st[1]), relocations=int(st[2]), lost=int(st[3]))


def responses(rng, n, nscores, negative=False):
    """In [0, 2] with exact zeros and ones (or in [-1, 2] with negative=True)."""
    r = rng.uniform(-1.0 if negative else 0.0, 2.0, (n, nscores))
    r[rng.random((n, nscores)) < 0.1] = 0.0
    r[rng.random((n, nscores)) < 0.1] = 1.0
    return r


MESHES = {"kuhn": lambda: (kuhn_box(6, 5, 4), (6.0, 5.0, 4.0)), "delaunay": lambda: (delaunay_box(600), (1.0, 1.0, 1.0))}


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("nscores", [1, 3, 8])
@pytest.mark.parametrize("mesh", ["kuhn", "delaunay"])
def test_scored_step_matches_the_oracle_score_by_score(mesh, nscores, fma):
    (c, t), box = MESHES[mesh]()
    n = 3000
    wl = SyntheticWorkload(box=box, num_particles=n, mean_length=0.5 * min(box), seed=11)
    rng = np.random.default_rng(nscores)
    eng = ScoredEmul(c, t, n, nscores, fma)
    orcs = [OraclePumiTally(c, t, n) for _ in range(nscores)]
    init = wl.initial_positions()
    for e in [eng] + orcs:
        e.CopyInitialPosition(init.reshape(-1).copy())
    for step in range(3):
        o, d, f, w = wl.next_step()
        r = responses(rng, n, nscores, negative=mesh == "delaunay")
        f1 = f.copy()
        eng.move(o.reshape(-1), d.reshape(-1), f1, w, r)
        assert not f1.any()
        for k, orc in enumerate(orcs):
            orc.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w * r[:, k])
        flux, elem, pos, st = eng.get()
        for k, orc in enumerate(orcs):
            assert_flux_close(flux[k], orc.flux, f"{mesh} score {k} step {step}")
        np.testing.assert_array_equal(elem, orcs[0].elem_ids)
        assert_positions_close(pos, orcs[0].positions, f"{mesh} step {step}")
    assert st["segments"] == orcs[0].n_segments and st["tracks"] == orcs[0].n_tracks and st["lost"] == 0


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
def test_non_finite_responses_are_lost_flights(fma):
    c, t = kuhn_box(5, 5, 5)
    n, nscores = 2000, 4
    wl = SyntheticWorkload(box=(5.0, 5.0, 5.0), num_particles=n, seed=5)
    rng = np.random.default_rng(3)
    eng = ScoredEmul(c, t, n, nscores, fma)
    orcs = [OraclePumiTally(c, t, n) for _ in range(nscores)]
    init = wl.initial_positions()
    for e in [eng] + orcs:
        e.CopyInitialPosition(init.reshape(-1).copy())
    o, d, f, w = wl.next_step()
    f[:] = 1
    o[:] = init  # no relocation: a lost flight leaves the particle where it is
    r = responses(rng, n, nscores)
    bad = np.arange(0, 60)
    r[bad[:20], 0] = np.nan
    r[bad[20:40], 3] = np.inf
    r[bad[40:], 1] = -np.inf
    eng.move(o.reshape(-1), d.reshape(-1), f.copy(), w, r)
    f_ref = f.copy()
    f_ref[bad] = 0
    for k, orc in enumerate(orcs):
        orc.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f_ref.copy(), w * np.nan_to_num(r[:, k]))
    flux, elem, pos, st = eng.get()
    assert np.isfinite(flux).all() and np.isfinite(pos).all()
    for k, orc in enumerate(orcs):
        assert_flux_close(flux[k], orc.flux, f"score {k}")
    np.testing.assert_array_equal(elem, orcs[0].elem_ids)
    np.testing.assert_array_equal(pos[bad], init[bad])
    assert st["lost"] == len(bad)
