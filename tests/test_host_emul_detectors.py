"""The point detectors' per-ray step (walk_core.cuh, detector_event / detector_ray) behind point location (locate_point),
compiled for the host by g++ as a TEST-ONLY build (tests/host_emul/emul_detectors.cpp) in both rounding flavours, against
a numpy reference (tests/detectors_ref.py) on the Kuhn, renumbered Delaunay, L-shaped and carved-void meshes."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from detectors_ref import ball_g, locate, reference_detectors
from helpers import HERE, ROOT
from locate_ref import MESHES, generic_points

_LIBS = {}


def detect_lib(fma):
    if fma not in _LIBS:
        so = os.path.join(HERE, "host_emul", "libptb_detect_fma.so" if fma else "libptb_detect.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_detectors.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
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
        L.ptb_detect.argtypes = [C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 6 + \
            [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
             C.c_void_p]
        L.ptb_ball_g.restype = C.c_double
        L.ptb_ball_g.argtypes = [C.c_double]
        _LIBS[fma] = L
    return _LIBS[fma]


def _ptr(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data


class Emul:
    def __init__(self, mesh, fma):
        self.c, self.t = MESHES[mesh]()
        self.L = detect_lib(fma)
        self.keep = (np.ascontiguousarray(self.c), np.ascontiguousarray(self.t, dtype=np.int32))
        self.h = self.L.ptb_locate_create(self.keep[0].ctypes.data, len(self.c), self.keep[1].ctypes.data, len(self.t))
        assert self.h

    def close(self):
        self.L.ptb_locate_destroy(self.h)

    def detect(self, pts, w, sigma, det, r0, pdf=None, r=None, bins=None, times=None, speeds=None, edges=None,
               nscores=1):
        nbins = sigma.shape[0]
        T = 1 if edges is None else len(edges) - 1
        out = np.empty((T, nbins, nscores, len(det)))
        counts = np.zeros(7, dtype=np.uint64)
        arrs = [np.ascontiguousarray(a, dtype=np.float64) if a is not None else None
                for a in (pts, w, pdf, r, None, times, speeds, edges, sigma, det, r0)]
        b = None if bins is None else np.ascontiguousarray(bins, dtype=np.int32)
        self.L.ptb_detect(self.h, _ptr(arrs[0]), len(pts), _ptr(arrs[1]), _ptr(arrs[2]), _ptr(arrs[3]), _ptr(b),
                          _ptr(arrs[5]), _ptr(arrs[6]), nscores, nbins, _ptr(arrs[7]), 0 if edges is None else T,
                          _ptr(arrs[8]), _ptr(arrs[9]), len(det), _ptr(arrs[10]), out.ctypes.data, counts.ctypes.data)
        return out, tuple(int(x) for x in counts)


def check_counts(got, want):
    assert got[:4] == want[:4] and got[5:] == want[5:], (got, want)


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("mesh", list(MESHES))
def test_random_sigma_matches_the_numpy_reference(mesh, fma):
    """Random per-element Sigma, pdfs, responses, score bins and time bins on generic rays: scores to rtol 1e-12."""
    em = Emul(mesh, fma)
    try:
        rng = np.random.default_rng(17 + len(mesh))
        pts, elem = generic_points(mesh, em.c, em.t, 120, rng)
        det, _ = generic_points(mesh, em.c, em.t, 3, rng)
        n, D, nbins, nscores = len(pts), len(det), 3, 2
        sigma = rng.uniform(0.05, 0.8, size=(nbins, len(em.t)))
        r0 = np.array([0.0, 0.3, 2.0])
        w = rng.uniform(0.5, 2.0, n)
        pdf = rng.uniform(0.0, 0.4, size=(n, D))
        r = rng.uniform(0.2, 2.0, size=(n, nscores))
        bins = rng.integers(-1, nbins + 1, n)
        edges = np.array([0.0, 0.7, 1.5, 4.0])
        times = rng.uniform(-0.2, 2.5, n)
        speeds = rng.uniform(1.0, 5.0, n)
        got, cnt = em.detect(pts, w, sigma, det, r0, pdf, r, bins, times, speeds, edges, nscores)
        want, wcnt = reference_detectors(em.c, em.t, elem, pts, w, pdf, r, bins, times, speeds, edges, nbins, nscores,
                                         sigma, det, r0)
        check_counts(cnt, wcnt)
        assert wcnt[0] > 50 and wcnt[3] > 5
        if mesh in ("l_shape", "void"):
            assert wcnt[1] > 0
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-300)
    finally:
        em.close()


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("mesh", ["kuhn", "delaunay"])
def test_homogeneous_sigma_gives_sigma_times_r(mesh, fma):
    """With one Sigma everywhere tau = Sigma R, also for rays in face planes and through vertices."""
    em = Emul(mesh, fma)
    try:
        lo, hi = em.c.min(0), em.c.max(0)
        inner = em.c[((em.c > lo + 1e-9) & (em.c < hi - 1e-9)).all(1)]
        rng = np.random.default_rng(3)
        pts = np.concatenate([inner[:60], generic_points(mesh, em.c, em.t, 40, rng)[0]])
        det = inner[[3, 7]] if mesh == "kuhn" else inner[[3, 7]] * 0.999 + 0.001 * inner[[4, 8]]
        sig = 0.37
        sigma = np.full((1, len(em.t)), sig)
        got, cnt = em.detect(pts, np.ones(len(pts)), sigma, det, np.zeros(2))
        # an event exactly on a detector with r0 == 0 is rejected, for every detector
        ok = np.all([np.sqrt(((det[d] - pts) ** 2).sum(1)) > 0 for d in range(2)], axis=0)
        for d in range(2):
            R = np.sqrt(((det[d] - pts) ** 2).sum(1))
            want = np.exp(-sig * R[ok]) / (4 * math.pi * R[ok] ** 2)
            # every event of the call adds to this one slot
            assert math.isclose(got[0, 0, 0, d], math.fsum(want), rel_tol=1e-13)
        assert cnt[1] == 0 and cnt[2] == 0
    finally:
        em.close()


def test_ball_formula_keeps_digits_near_zero():
    L = detect_lib(False)
    for x in (0.0, 1e-300, 1e-17, 1e-12, 1e-8, 1e-4, 0.5, 3.0, 50.0, 800.0):
        assert L.ptb_ball_g(x) == pytest.approx(ball_g(x), rel=1e-15, abs=0.0)
    assert L.ptb_ball_g(1e-12) == pytest.approx(1.0 - 0.5e-12, rel=1e-15)  # 1 - exp(-x) would lose it


def test_rays_across_the_notch_are_shadowed():
    em = Emul("l_shape", False)
    try:
        pts = np.array([[7.0, 3.0, 1.0], [6.5, 3.5, 0.5]])
        det = np.array([[3.0, 7.0, 1.0]])  # the line crosses x > 4, y > 4: outside the mesh
        got, cnt = em.detect(pts, np.ones(2), np.full((1, len(em.t)), 0.1), det, np.zeros(1))
        assert not got.any() and cnt[1] == 2 and cnt[0] == 0
    finally:
        em.close()


def test_outcome_ranking_and_counters():
    """Rejected (non-finite inputs, a bad pdf value at any detector, an event on a detector with r0 == 0) before
    outside, outside before skipped; every event counted once."""
    em = Emul("kuhn", False)
    try:
        nan = np.nan
        det = np.array([[1.5, 1.5, 1.5], [3.5, 2.5, 2.0]])
        pts = np.array([[1.2, 1.1, 0.9], [nan, 1.0, 1.0], [-5.0, 1.0, 1.0], [-5.0, 1.0, 1.0], [1.5, 1.5, 1.5],
                        [2.2, 1.3, 1.7], [2.2, 1.3, 1.7]])
        w = np.array([1.0, 1.0, 1.0, np.inf, 1.0, 1.0, 1.0])
        pdf = np.full((7, 2), 0.1)
        pdf[2, 0] = -1.0  # rejection takes precedence over outside
        pdf[5, 1] = nan   # rejects the whole event
        bins = np.array([0, 0, 0, 0, 0, 0, 2])  # the last event's rays are skipped
        sigma = np.full((2, len(em.t)), 0.2)
        got, cnt = em.detect(pts, w, sigma, det, np.array([0.0, 0.5]), pdf=pdf, bins=bins)
        elem = locate(em.c, em.t, np.nan_to_num(pts, nan=-1e9))
        want, wcnt = reference_detectors(em.c, em.t, elem, pts, w, pdf, None, bins, None, None, None, 2, 1, sigma, det,
                                         np.array([0.0, 0.5]))
        check_counts(cnt, wcnt)
        # rejected: events 1 (nan), 2 (negative pdf), 3 (inf weight), 4 (on detector 0, r0 == 0) and 5 (nan pdf);
        # outside: none left; skipped: event 6's rays
        assert cnt[6] == 5 and cnt[5] == 0
        assert sum(cnt[:4]) == 2 * (7 - 5) - 2
        np.testing.assert_allclose(got, want, rtol=1e-12)
    finally:
        em.close()
