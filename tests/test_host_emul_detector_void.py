"""The detector void (pumitally_set_detector_void; walk_core.cuh, detector_ray<true> / hull_entry) behind point location,
compiled for the host by g++ as a TEST-ONLY build (tests/host_emul/emul_detector_void.cpp) in both rounding flavours,
against the void reference (tests/detector_void_ref.py) on the Kuhn, Delaunay, L-shaped, carved-void and comb meshes,
against the comb's analytic optical depths and hull entries, and on rays along hull faces, edges and vertices.  Also the
checkpoint format version 4 through a host build of checkpoint.cpp."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from detector_void_ref import comb_mesh, reference_void
from detectors_ref import locate
from helpers import HERE, ROOT
from locate_ref import MESHES, extent, generic_points
from pumiumtally_b200.mesh import kuhn_box

_LIBS = {}
ALL_MESHES = dict(MESHES, comb=comb_mesh)


def void_lib(fma):
    if fma not in _LIBS:
        so = os.path.join(HERE, "host_emul", "libptb_detect_void_fma.so" if fma else "libptb_detect_void.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_detector_void.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
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
        L.ptb_locate_hull_convex.argtypes = [C.c_void_p]
        L.ptb_detect_void.argtypes = [C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 6 + \
            [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
             C.c_void_p, C.c_void_p]
        L.ptb_hull_candidates.restype = C.c_int64
        L.ptb_hull_candidates.argtypes = [C.c_void_p, C.c_void_p]
        _LIBS[fma] = L
    return _LIBS[fma]


def _ptr(a):
    return None if a is None else a.ctypes.data


class Emul:
    def __init__(self, c, t, fma=False):
        self.c, self.t = c, t
        self.L = void_lib(fma)
        self.keep = (np.ascontiguousarray(c), np.ascontiguousarray(t, dtype=np.int32))
        self.h = self.L.ptb_locate_create(self.keep[0].ctypes.data, len(c), self.keep[1].ctypes.data, len(t))
        assert self.h

    def close(self):
        self.L.ptb_locate_destroy(self.h)

    def detect(self, pts, w, sigma, det, r0, pdf=None, r=None, bins=None, times=None, speeds=None, edges=None,
               nscores=1, max_iters=0):
        nbins = sigma.shape[0]
        T = 1 if edges is None else len(edges) - 1
        out = np.empty((T, nbins, nscores, len(det)))
        counts = np.zeros(8, dtype=np.uint64)
        f = [None if a is None else np.ascontiguousarray(a, dtype=np.float64)
             for a in (pts, w, pdf, r, times, speeds, edges, sigma, det, r0)]
        b = None if bins is None else np.ascontiguousarray(bins, dtype=np.int32)
        self.L.ptb_detect_void(self.h, _ptr(f[0]), len(pts), _ptr(f[1]), _ptr(f[2]), _ptr(f[3]), _ptr(b), _ptr(f[4]),
                               _ptr(f[5]), nscores, nbins, _ptr(f[6]), 0 if edges is None else T, _ptr(f[7]),
                               _ptr(f[8]), len(det), _ptr(f[9]), max_iters, out.ctypes.data, counts.ctypes.data)
        return out, tuple(int(x) for x in counts)


def cavity_points(name, c, rng, n):
    """Points in the mesh's notch, cavity or slots (none on the Kuhn and Delaunay boxes)."""
    if name == "l_shape":  # the notch x > 4, y > 4
        return np.column_stack([rng.uniform(4.05, 7.95, n), rng.uniform(4.05, 7.95, n), rng.uniform(0.05, 1.95, n)])
    if name == "void":  # the cube [2, 3]^3
        return rng.uniform(2.05, 2.95, size=(n, 3))
    if name == "comb":  # the slots x in [2k + 1, 2k + 2], y > 1
        k = rng.integers(0, 4, n)
        return np.column_stack([2 * k + 1 + rng.uniform(0.05, 0.95, n), rng.uniform(1.05, 2.95, n),
                                rng.uniform(0.05, 1.95, n)])
    return np.zeros((0, 3))


def outside_points(c, rng, n, far=1e3):
    """Points beyond the bounding box: a shell up to one extent away, and a few up to `far` extents away."""
    lo, hi = c.min(0), c.max(0)
    L = hi - lo
    shell = rng.uniform(lo - L, hi + L, size=(8 * n, 3))
    shell = shell[((shell < lo - 1e-2 * L) | (shell > hi + 1e-2 * L)).any(1)][:n]
    u = rng.normal(size=(n // 4 + 1, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    dist = np.exp(rng.uniform(0.0, math.log(far), len(u))) * extent(c)
    return np.concatenate([shell, 0.5 * (lo + hi) + u * dist[:, None]])


def check_counts(cnt, want, n_events, D, skipped=0):
    assert cnt[:4] == want[:4] and cnt[5:7] == want[5:], (cnt, want)
    assert cnt[1] == 0 and cnt[2] == 0 and cnt[5] == 0  # never shadowed, lost or outside
    assert sum(cnt[:4]) == D * (n_events - cnt[6]) - skipped


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("mesh", list(ALL_MESHES))
def test_matches_the_void_reference(mesh, fma):
    """Detectors inside, in the notch, cavity or slots, beyond the bounding box and up to 10^3 extents away; events
    inside, in the notch, cavity or slots and beyond the bounding box; random Sigma, pdfs, responses, score bins and time
    bins: scores to rtol 1e-12."""
    c, t = ALL_MESHES[mesh]()
    em = Emul(c, t, fma)
    try:
        rng = np.random.default_rng(29 + len(mesh))
        pts = np.concatenate([generic_points(mesh, c, t, 50, rng)[0], cavity_points(mesh, c, rng, 20),
                              outside_points(c, rng, 20, far=3.0)])
        det = np.concatenate([generic_points(mesh, c, t, 1, rng)[0], cavity_points(mesh, c, rng, 1),
                              outside_points(c, rng, 1, far=1e3)[-2:]])
        n, D, nbins, nscores = len(pts), len(det), 2, 2
        elem = locate(c, t, pts)
        sigma = rng.uniform(0.05, 0.8, size=(nbins, len(t)))
        r0 = rng.uniform(0.0, 0.6, D)
        r0[0] = 0.0
        w = rng.uniform(0.5, 2.0, n)
        pdf = rng.uniform(0.0, 0.4, size=(n, D))
        r = rng.uniform(0.2, 2.0, size=(n, nscores))
        bins = rng.integers(0, nbins, n)
        got, cnt = em.detect(pts, w, sigma, det, r0, pdf, r, bins, nscores=nscores)
        want, wcnt = reference_void(c, t, elem, pts, w, pdf, r, bins, None, None, None, nbins, nscores, sigma, det, r0)
        check_counts(cnt, wcnt, n, D)
        assert wcnt[0] > 100 and cnt[7] > 0
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-300)
        # time bins crossed by the arrival times skip some rays: the identity holds less those
        edges = np.array([0.0, 1.0, 3.0, 6.0])
        times = rng.uniform(0.0, 2.0, n)
        speeds = rng.uniform(1.0, 4.0, n)
        got, cnt = em.detect(pts, w, sigma, det, r0, pdf, r, bins, times, speeds, edges, nscores)
        want, wcnt = reference_void(c, t, elem, pts, w, pdf, r, bins, times, speeds, edges, nbins, nscores, sigma, det,
                                    r0)
        assert cnt[:4] == wcnt[:4] and cnt[1] == cnt[2] == cnt[5] == 0
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-300)
    finally:
        em.close()


def test_outside_events_inside_r0_use_sigma_zero():
    c, t = l_shape = MESHES["l_shape"]()
    em = Emul(c, t)
    try:
        det = np.array([[6.0, 6.0, 1.0]])  # in the notch
        pts = np.array([[6.2, 6.1, 1.0], [5.9, 5.5, 0.7]])
        got, cnt = em.detect(pts, np.array([1.0, 2.0]), np.full((1, len(t)), 0.7), det, np.array([1.0]))
        assert got[0, 0, 0, 0] == pytest.approx(3.0 * 3.0 / (4 * math.pi), rel=1e-15)
        assert cnt[3] == 2 and cnt[5] == 0 and cnt[7] == 0
    finally:
        em.close()


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
def test_comb_rays_parallel_to_x_are_analytic(fma):
    """Rays parallel to x through the comb's slabs (x in [2k, 2k + 1], one Sigma each) across the slots: tau = sum_j
    Sigma_j t_j to 1e-13, and the hull entries are the slabs entered (every slab the ray crosses but the event's)."""
    c, t = comb_mesh()
    em = Emul(c, t, fma)
    try:
        rng = np.random.default_rng(7)
        slab_sig = rng.uniform(0.1, 1.0, 5)
        cen = c[t].mean(1)
        sigma = slab_sig[np.clip(np.floor(cen[:, 0] / 2.0).astype(int), 0, 4)][None, :]
        n = 60
        yz = np.column_stack([rng.uniform(1.05, 2.95, n), rng.uniform(0.05, 1.95, n)])
        xa = rng.uniform(-3.0, 12.0, n)
        xb = rng.uniform(-3.0, 12.0, n)
        for i in range(n):  # keep the ends off the slab faces
            for x in (xa, xb):
                if abs(x[i] - round(x[i])) < 1e-3:
                    x[i] += 0.01
        entries_want = 0
        for i in range(n):
            pts = np.array([[xa[i], *yz[i]]])
            det = np.array([[xb[i], *yz[i]]])
            lo, hi = min(xa[i], xb[i]), max(xa[i], xb[i])
            tau, ent = 0.0, 0
            for k in range(5):
                ln = max(0.0, min(hi, 2.0 * k + 1.0) - max(lo, 2.0 * k))
                tau += slab_sig[k] * ln
                ent += ln > 0.0 and not (2.0 * k <= xa[i] <= 2.0 * k + 1.0)
            R = hi - lo
            got, cnt = em.detect(pts, np.ones(1), sigma, det, np.zeros(1))
            assert got[0, 0, 0, 0] == pytest.approx(math.exp(-tau) / (4 * math.pi * R * R), rel=1e-13), i
            assert cnt[0] == 1 and cnt[7] == ent, (i, cnt, ent)
            entries_want += ent
        assert entries_want > 2 * n
    finally:
        em.close()


@pytest.mark.parametrize("fma", [False, True], ids=["plain", "fma"])
def test_rays_along_hull_faces_edges_and_vertices(fma):
    """Axis-aligned rays from outside a Kuhn box to beyond it, along hull faces, hull edges and through hull vertices
    (and along interior face planes): with one Sigma, tau = Sigma times the box's length along the axis; none lost."""
    Lx, Ly, Lz = 6.0, 5.0, 4.0
    c, t = kuhn_box(6, 5, 4)
    em = Emul(c, t, fma)
    try:
        sig = 0.37
        sigma = np.full((1, len(t)), sig)
        rays = []
        for y, z in [(0.0, 0.5), (0.0, 0.0), (Ly, Lz), (0.0, 2.0), (2.0, 3.0), (1.0, 0.0), (Ly, 1.7), (2.5, Lz)]:
            rays.append(((-2.0, y, z), (Lx + 3.0, y, z), Lx))
        for x, z in [(0.0, 0.5), (Lx, Lz), (3.0, 0.0), (2.0, 2.0)]:
            rays.append(((x, -1.5, z), (x, Ly + 0.5, z), Ly))
        for x, y in [(0.0, 0.0), (Lx, 2.0), (1.0, 1.0), (3.3, Ly)]:
            rays.append(((x, y, 7.0), (x, y, -0.25), Lz))
        lost = 0
        for a, b, inside in rays:
            R = float(np.linalg.norm(np.subtract(b, a)))
            got, cnt = em.detect(np.array([a]), np.ones(1), sigma, np.array([b]), np.zeros(1))
            assert got[0, 0, 0, 0] == pytest.approx(math.exp(-sig * inside) / (4 * math.pi * R * R), rel=1e-12), (a, b)
            assert cnt[7] == 1, (a, b, cnt)  # a convex hull: entered once, never again
            lost += cnt[2]
        assert lost == 0
    finally:
        em.close()


def test_hull_lists_hold_only_hull_tets():
    for name in ("kuhn", "comb"):
        c, t = ALL_MESHES[name]()
        em = Emul(c, t)
        try:
            nhull = C.c_int64()
            entries = em.L.ptb_hull_candidates(em.h, C.byref(nhull))
            faces = np.sort(t[:, [[1, 2, 3], [0, 2, 3], [0, 1, 3], [0, 1, 2]]], axis=2).reshape(-1, 3)
            _, inv, cnt = np.unique(faces, axis=0, return_inverse=True, return_counts=True)
            hull = (cnt[inv.ravel()] == 1).reshape(-1, 4).any(1)
            assert nhull.value == hull.sum() < len(t)
            assert entries >= nhull.value
        finally:
            em.close()


# ---- checkpoint format version 4 ------------------------------------------------------------------------------------
_CK = []


def ckpt_lib():
    if not _CK:
        so = os.path.join(HERE, "host_emul", "libptb_ckpt_void.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_checkpoint_detector_void.cpp"), os.path.join(csrc, "checkpoint.cpp")]
        deps = srcs + [os.path.join(csrc, "checkpoint.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-I", csrc, *srcs, "-o", so,
                                   "-lz"])
        L = C.CDLL(so)
        L.ptb_ckpt_void_write.restype = C.c_int64
        L.ptb_ckpt_void_write.argtypes = [C.c_int32, C.c_void_p, C.c_int64]
        L.ptb_ckpt_void_read.restype = C.c_int32
        L.ptb_ckpt_void_read.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_char_p, C.c_int64]
        _CK.append(L)
    return _CK[0]


def _write(on):
    buf = np.zeros(1 << 16, dtype=np.uint8)
    n = ckpt_lib().ptb_ckpt_void_write(on, buf.ctypes.data, buf.size)
    assert n > 0
    return buf[:n].copy()


def _read(data, on):
    ver = np.zeros(1, dtype=np.uint32)
    counts = np.zeros(8, dtype=np.uint64)
    nw = np.zeros(1, dtype=np.int32)
    err = C.create_string_buffer(256)
    rc = ckpt_lib().ptb_ckpt_void_read(data.ctypes.data, data.size, on, ver.ctypes.data, counts.ctypes.data,
                                       nw.ctypes.data, err, 256)
    return rc, int(ver[0]), counts[:nw[0]].tolist(), err.value.decode()


def test_checkpoint_version_4_round_trips_with_eight_counters():
    on, off = _write(1), _write(0)
    assert _read(on, 1) == (0, 4, [1, 2, 3, 4, 5, 6, 7, 8], "")
    assert _read(off, 0) == (0, 3, [1, 2, 3, 4, 5, 6, 7], "")
    assert on.size == off.size + 8  # the eighth counter, nothing else


def test_checkpoint_across_the_void_setting_is_refused():
    for data, engine in ((_write(1), 0), (_write(0), 1)):
        rc, _, _, err = _read(data, engine)
        assert rc == 1 and "detector void" in err


def test_checkpoint_version_4_corruption_is_detected():
    data = _write(1)
    data[40] ^= 1
    rc, _, _, err = _read(data, 1)
    assert rc == 2 and "version 4" in err
