"""The cosine-binned face-current crossing step of the CUDA kernels (walk_core.cuh, MU in advance and start_tally_to),
compiled for the host by g++ without contraction as a TEST-ONLY build (tests/host_emul/emul_current_cosines.cpp).

The cosine of every crossing is restated here from the stored record normals, with the operations walk_core.cuh pins:
bden = nx * ux + ny * uy + nz * uz (the exit scan's sum), len = sqrt(ux * ux + uy * uy + uz * uz), inv = 1.0 / len,
mu = min(bden * inv, 1.0), each rounded once.  The crossings themselves come from the exact clip-and-walk reference
(face_currents_ref.face_walk).  Weights are dyadic (k / 8), so every sum is exact in any order and the comparisons are
bit for bit, per time bin and cosine bin.

Also: every MU kernel of walk_kernels.cu, compiled for sm_90a with -Xptxas -v, is reported, has at most 16 B more spill
stores and loads than its CU twin, and no stack frame beyond the twin's, except the packed timed moment kernel, whose
frame is 8 B larger (pinned)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from current_cosines_ref import cosine_bins
from face_currents_ref import face_walk, reference_currents, unit_planes
from helpers import HERE, ROOT, l_shaped_mesh
from pumiumtally_b200.mesh import delaunay_box, kuhn_box

TIME_EDGES = np.linspace(0.0, 4.0, 9)
MESHES = {
    "kuhn": lambda: kuhn_box(6, 5, 4),
    "delaunay": lambda: delaunay_box(600),
    "l_shaped": lambda: l_shaped_mesh(6, 6, 3),
}
_LIB = []


def cosines_lib():
    if not _LIB:
        so = os.path.join(HERE, "host_emul", "libptb_cosines.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_current_cosines.cpp"), os.path.join(csrc, "tet_mesh.cpp"),
                os.path.join(csrc, "osh_reader.cpp"), os.path.join(csrc, "gmsh_reader.cpp")]
        deps = srcs + [os.path.join(csrc, h) for h in ("walk_core.cuh", "tet_mesh.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp",
                                   "-ffp-contract=off", "-I", csrc, "-I", os.path.join(ROOT, "include"), *srcs,
                                   "-o", so, "-lz"])
        L = C.CDLL(so)
        L.ptb_cosines_create.restype = C.c_void_p
        L.ptb_cosines_create.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_int, C.c_int]
        L.ptb_cosines_destroy.argtypes = [C.c_void_p]
        L.ptb_cosines_localize.argtypes = [C.c_void_p, C.c_void_p]
        L.ptb_cosines_move.argtypes = [C.c_void_p] * 7
        L.ptb_cosines_get.argtypes = [C.c_void_p] * 5
        L.ptb_cosines_records.argtypes = [C.c_void_p] * 2
        L.ptb_cosines_adjacency.argtypes = [C.c_void_p] * 2
        _LIB.append(L)
    return _LIB[0]


class CosineEmul:
    def __init__(self, coords, t2v, n, mu_edges, edges=None, moments=0):
        self._L = cosines_lib()
        coords = np.ascontiguousarray(coords, dtype=np.float64)
        t2v = np.ascontiguousarray(t2v, dtype=np.int32)
        self.edges = None if edges is None else np.ascontiguousarray(edges, dtype=np.float64)
        self.mu_edges = np.ascontiguousarray(mu_edges, dtype=np.float64)
        self.n, self.ne = n, len(t2v)
        self.nt = 1 if edges is None else len(edges) - 1
        self.nmu = len(self.mu_edges) - 1
        self._h = self._L.ptb_cosines_create(coords.ctypes.data, len(coords), t2v.ctypes.data, len(t2v), n,
                                             None if edges is None else self.edges.ctypes.data,
                                             0 if edges is None else len(self.edges), self.mu_edges.ctypes.data,
                                             len(self.mu_edges), moments)
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.ptb_cosines_destroy(self._h)

    def localize(self, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float64)
        self._L.ptb_cosines_localize(self._h, xyz.ctypes.data)

    def move(self, o, d, f, w, times=None, speeds=None):
        o, d, w = (np.ascontiguousarray(a, dtype=np.float64) for a in (o, d, w))
        f = np.ascontiguousarray(f, dtype=np.int8)
        arrs = [None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in (times, speeds)]
        self._L.ptb_cosines_move(self._h, o.ctypes.data, d.ctypes.data, f.ctypes.data, w.ctypes.data,
                                 *(None if a is None else a.ctypes.data for a in arrs))

    def get(self):
        out = np.empty((self.nt, self.nmu, self.ne, 4))
        inn = np.empty_like(out)
        elem = np.empty(self.n, dtype=np.int32)
        pos = np.empty((self.n, 3))
        self._L.ptb_cosines_get(self._h, out.ctypes.data, inn.ctypes.data, elem.ctypes.data, pos.ctypes.data)
        return out, inn, elem, pos

    def adjacency(self):
        a = np.empty((self.ne, 4), dtype=np.int32)
        self._L.ptb_cosines_adjacency(self._h, a.ctypes.data)
        return a.astype(np.int64)

    def records(self):
        r = np.empty((self.ne, 4, 4))
        self._L.ptb_cosines_records(self._h, r.ctypes.data)
        return r


def pinned_cosines(recs, o, d, ids, e, f):
    """The cosine of each crossing (flight ids, element e left through local face f), restated with the pinned
    operations on the stored normals."""
    n = recs[e, f, :3]
    u = d[ids] - o[ids]
    ux, uy, uz = u[:, 0], u[:, 1], u[:, 2]
    bden = n[:, 0] * ux + n[:, 1] * uy + n[:, 2] * uz
    inv = 1.0 / np.sqrt(ux * ux + uy * uy + uz * uz)
    return np.minimum(bden * inv, 1.0)


def _interior_points(rng, coords, t2v, n):
    lam = 0.02 + 0.92 * rng.dirichlet(np.ones(4), n)
    lam /= lam.sum(axis=1, keepdims=True)
    tets = rng.integers(0, len(t2v), n)
    return np.ascontiguousarray(np.einsum("iq,iqk->ik", lam, coords[t2v[tets]]))


def _check(mesh, mu_edges, timed=False, moments=0, axis=False, steps=2, n=3000, seed=0, on_edge=False):
    """Moves of the host build against the exact crossings binned by the restated cosine.  axis: the flights run along
    the coordinate axes (normal incidence on a Kuhn mesh's axis-aligned faces).  on_edge: the cosine edges are replaced,
    between the moves, by cosines the first move's crossings actually have (crossings exactly on an edge)."""
    coords, t2v = MESHES[mesh]()
    rng = np.random.default_rng(seed)
    edges = TIME_EDGES if timed else None
    planes = unit_planes(coords, t2v)
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    scale = (hi - lo).max()
    mu_edges = np.asarray(mu_edges, dtype=np.float64)
    if on_edge:  # a probe run of the same flights finds real cosines; the edges become some of them
        probe_emul = CosineEmul(coords, t2v, n, [0.0, 1.0], edges, moments)
        probe_emul.localize(_interior_points(rng, coords, t2v, n))
        probe = _flights(rng, coords, t2v, planes, lo, scale, n, axis, timed, probe_emul)
        mu = pinned_cosines(probe_emul.records(), probe["o"], probe["d"], *probe["cr"][:3])
        mu_edges = np.unique(np.concatenate([[0.0], rng.choice(mu[mu < 1.0], 6, replace=False), [1.0]]))
        rng = np.random.default_rng(seed)
    emul = CosineEmul(coords, t2v, n, mu_edges, edges, moments)
    recs = emul.records()
    emul.localize(_interior_points(rng, coords, t2v, n))
    want_out = np.zeros((emul.nt, 1, emul.nmu, len(t2v), 4))
    want_in = np.zeros_like(want_out)
    seen = np.zeros(emul.nmu + 1, dtype=np.int64)
    mus = []
    for step in range(steps):
        fl = _flights(rng, coords, t2v, planes, lo, scale, n, axis, timed, emul)
        ids, e, f, j = fl["cr"][:4]
        mu = pinned_cosines(recs, fl["o"], fl["d"], ids, e, f)
        mus.append(mu)
        k = cosine_bins(mu, mu_edges)
        seen += np.bincount(k + 1, minlength=emul.nmu + 1)
        for c in range(emul.nmu):
            m = k == c
            a, b = reference_currents(fl["adj"], (ids[m], e[m], f[m], j[m]), fl["w"], None, emul.nt, 1)
            want_out[:, :, c] += a
            want_in[:, :, c] += b
        emul.move(fl["o"], fl["d"], fl["fly"].astype(np.int8), fl["w"], fl["times"] if timed else None,
                  fl["speeds"] if timed else None)
    out, inn, _, _ = emul.get()
    label = f"{mesh} edges={mu_edges} timed={timed} moments={moments} axis={axis}"
    np.testing.assert_array_equal(out, want_out[:, 0], err_msg=label + " outgoing")
    np.testing.assert_array_equal(inn, want_in[:, 0], err_msg=label + " incoming")
    assert seen[1:].sum() > 0, "no binned crossing tested"
    return np.concatenate(mus), mu_edges, seen


def _flights(rng, coords, t2v, planes, lo, scale, n, axis, timed, emul):
    """One move's flights from fresh interior origins, positioned first by a weight-0 move; the flights the reference
    cannot decide are left on the ground."""
    adj = emul.adjacency()
    o = _interior_points(rng, coords, t2v, n)
    emul.move(o, o, np.ones(n, np.int8), np.zeros(n), np.zeros(n) if timed else None, np.ones(n) if timed else None)
    _, _, elem, pos = emul.get()
    start, ok = elem.astype(np.int64), (pos == o).all(axis=1)
    if axis:
        u = np.zeros((n, 3))
        u[np.arange(n), rng.integers(0, 3, n)] = rng.choice([-1.0, 1.0], n)
    else:
        u = rng.normal(size=(n, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
    d = o + u * rng.exponential(0.5 * scale, n)[:, None]
    times = rng.uniform(TIME_EDGES[0] - 1.0, TIME_EDGES[-1] + 0.5, n)
    speeds = rng.uniform(0.3, 3.0, n)
    tpp = np.linalg.norm(d - o, axis=1) / speeds
    w = rng.integers(1, 17, n) / 8.0
    fly = ok & (rng.random(n) < 0.9)
    te = TIME_EDGES if timed else None
    cr = face_walk(planes, adj, start, o, d, fly, times, tpp, te)
    fly &= ~cr[4]
    cr = face_walk(planes, adj, start, o, d, fly, times, tpp, te)
    assert not cr[4][fly].any()
    return dict(o=o, d=d, w=w, fly=fly, times=times, speeds=speeds, cr=cr, adj=adj)


@pytest.mark.parametrize("mesh", sorted(MESHES))
def test_cosine_bin_of_every_crossing(mesh):
    mu, _, seen = _check(mesh, np.linspace(0.0, 1.0, 9), seed=1)
    assert (seen[1:] > 0).all()  # every bin met


@pytest.mark.parametrize("mesh", ["kuhn", "delaunay"])
def test_crossings_exactly_on_an_edge(mesh):
    mu, mu_edges, _ = _check(mesh, np.linspace(0.0, 1.0, 5), seed=2, on_edge=True)
    assert np.isin(mu, mu_edges[1:-1]).sum() > 0, "no crossing exactly on an edge"


def test_normal_incidence_lands_in_the_last_bin():
    """Axis-parallel flights on a Kuhn box cross its axis-aligned faces at mu = 1 (after the clamp)."""
    mu, mu_edges, seen = _check("kuhn", [0.0, 0.5, 0.9, 1.0], axis=True, seed=3)
    assert (mu == 1.0).sum() > 0
    assert seen[0] == 0  # nothing outside [0, 1]


@pytest.mark.parametrize("mesh", ["kuhn", "l_shaped"])
def test_edges_that_do_not_cover_the_range(mesh):
    mu, mu_edges, seen = _check(mesh, [0.2, 0.45, 0.7, 0.9], seed=4)
    assert seen[0] > 0  # crossings outside the edges add nothing


@pytest.mark.parametrize("moments", [0, 1])
@pytest.mark.parametrize("mesh", sorted(MESHES))
def test_time_bin_and_cosine_bin_of_each_crossing(mesh, moments):
    _check(mesh, [0.0, 0.25, 0.5, 0.75, 1.0], timed=True, moments=moments, seed=5)


def test_cosine_bin_rule():
    e = np.array([0.0, 0.25, 0.5, 1.0])
    mu = np.array([0.0, 0.1, 0.25, 0.49, 0.5, 0.99, 1.0, -0.1, 1.5])
    np.testing.assert_array_equal(cosine_bins(mu, e), [0, 0, 1, 1, 2, 2, 2, -1, -1])
    np.testing.assert_array_equal(cosine_bins(np.array([0.1, 0.2, 0.9, 0.95]), np.array([0.2, 0.9])), [-1, 0, 0, -1])


# ---- the MU kernels' resource use against their CU twins -------------------------------------------------------------
PTXAS = re.compile(r"Compiling entry function '([^']+)'.*?\n(?:.*\n)*?.*?Function properties for \1\n\s*(\d+) bytes "
                   r"stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers")


def _twin(name):
    if "walk_persist_current_mu_kernel" in name:
        return name.replace("30walk_persist_current_mu_kernel", "27walk_persist_current_kernel")
    return re.sub(r"(\d+)(walk_ldg_\w*current)_mu_kernel", lambda m: f"{int(m.group(1)) - 3}{m.group(2)}_kernel", name)


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"),
                    reason="nvcc not available")
def test_mu_kernels_resources(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-I", csrc, "-I", os.path.join(ROOT, "include"), "-c", os.path.join(csrc, "walk_kernels.cu"),
                          "-o", str(tmp_path / "w.o")], capture_output=True, text=True, check=True)
    k = {m[0]: tuple(map(int, m[1:])) for m in PTXAS.findall(res.stderr)}
    mu = sorted(n for n in k if "_mu_kernel" in n)
    # 4 thread-per-particle kernels and 3 persistent variants (8, 16, 24) x timed x moments
    assert len(mu) == 16, mu
    for name in mu:
        twin = _twin(name)
        assert twin in k, name
        (fr, st, ld, _), (tfr, tst, tld, _) = k[name], k[twin]
        assert st <= tst + 16 and ld <= tld + 16, (name, k[name], k[twin])
        if "walk_persist" in name and "Li2ELi8ELb1ELb1E" in name:
            # The one exception to "no stack frame beyond the twin's": the packed (24) timed moment kernel holds 24 B
            # of frame against its twin's 16 B.  Pinned to that, so that any growth fails here.
            assert (fr, tfr) == (24, 16), (name, k[name], k[twin])
        else:
            assert fr <= tfr, (name, k[name], k[twin])
