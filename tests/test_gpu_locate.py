"""Point queries (pumitally_locate_points, pumitally_evaluate_points): which element contains each point, and every
normalised result there.  Located elements are checked against a brute-force barycentric reference and the oracle's
localisation; evaluated values against a numpy recomputation from the engine's own accessors.  A query must change
nothing."""
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT
from locate_ref import (MESHES, _inside_shape, assert_contains, band_points, barycentric, generic_points,
                        non_finite_points, outside_points, special_points)
from oracle.oracle import OraclePumiTally
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_moments import _configure, _move
from test_gpu_scores import assert_same_particles, responses
from time_bins_ref import time_workload

pytestmark = pytest.mark.gpu

EDGES = np.linspace(0.0, 4.0, 5)


def _locate(eng, pts, path):
    import torch

    if path == "host":
        return eng.locate(pts)
    t = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float64)).cuda()
    out = eng.locate_device(t)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mesh", list(MESHES))
def test_locate_every_kind_of_point(mesh, path):
    c, t = MESHES[mesh]()
    eng = PumiTally.from_arrays(c, t, 16)
    eng.set_option("chunk", 1024)  # several chunks, the last one partial
    rng = np.random.default_rng(1)
    pts, want = generic_points(mesh, c, t, 2999, rng)  # not a multiple of the block
    np.testing.assert_array_equal(_locate(eng, pts, path), want)
    sp = special_points(c, t)
    sp = sp[_inside_shape(mesh, sp, 1e-9)]
    assert_contains(c, t, sp, _locate(eng, sp, path), mesh)
    out = np.concatenate([outside_points(mesh, c, rng), non_finite_points()])
    assert (_locate(eng, out, path) == -1).all()
    band = band_points(mesh, c, rng)
    got = _locate(eng, band, path)
    if (got >= 0).any():
        assert (barycentric(c, t, band[got >= 0], got[got >= 0]) >= -1e-8).all()
    assert eng.get_option("locate_candidates") > 0 if mesh in ("l_shape", "void") else eng.get_option("locate_candidates") == 0
    # before any particle was placed: nothing changed
    assert eng.stats()["moves"] == 0 and (eng.flux == 0).all()


@pytest.mark.parametrize("mesh", ["kuhn", "delaunay"])
def test_locate_equals_the_oracle_localisation_on_convex_meshes(mesh):
    c, t = MESHES[mesh]()
    pts, _ = generic_points(mesh, c, t, 2000, np.random.default_rng(4))
    orc = OraclePumiTally(c, t, len(pts))
    orc.CopyInitialPosition(pts.reshape(-1).copy())
    eng = PumiTally.from_arrays(c, t, 16)
    np.testing.assert_array_equal(eng.locate(pts), orc.elem_ids)


def test_config_c2_ten_million_points():
    """Full-size c2 (998,250 tets): 10 M uniform points in a box 10 % larger than the mesh; every returned tet contains
    its point and every -1 lies outside the mesh's box.  The host call (chunked) agrees with the device call."""
    import torch

    cfg = CONFIGS["c2"]
    cells = np.array(cfg["cells"], dtype=np.float64)
    coords, t2v = kuhn_box(*cfg["cells"])
    eng = PumiTally.from_arrays(coords, t2v, 16)
    n = 10_000_000
    g = torch.Generator(device="cuda").manual_seed(9)
    pts = (torch.rand((n, 3), dtype=torch.float64, device="cuda", generator=g) * torch.tensor(1.1 * cells, device="cuda")
           - torch.tensor(0.05 * cells, device="cuda")).contiguous()
    elem = eng.locate_device(pts)
    torch.cuda.synchronize()
    elem, p = elem.cpu().numpy(), pts.cpu().numpy()
    outside = ((p < 0) | (p > cells)).any(1)
    assert (elem[outside] == -1).all()
    assert (elem[elem < 0] == -1).all() and outside[elem < 0].all()
    assert (elem >= 0).sum() > 0.7 * n
    for a in range(0, n, 1 << 20):
        e, q = elem[a:a + (1 << 20)], p[a:a + (1 << 20)]
        lam = barycentric(coords, t2v, q[e >= 0], e[e >= 0])
        assert (lam >= -1e-9).all()
    sub = slice(0, 3_000_000)
    np.testing.assert_array_equal(eng.locate(p[sub]), elem[sub])


def test_queries_change_nothing():
    """Stats, positions, elements, flux, moments and the auto-tuner's state are bit-identical before and after queries
    interleaved with moves, and the particles equal those of an unqueried twin."""
    import torch

    c, t = kuhn_box(8, 7, 6)
    n = 4000
    wls = [SyntheticWorkload(box=(8.0, 7.0, 6.0), num_particles=n, mean_length=1.0, seed=3) for _ in range(2)]
    a, b = PumiTally.from_arrays(c, t, n), PumiTally.from_arrays(c, t, n)
    a.set_moments(1)
    b.set_moments(1)
    rng = np.random.default_rng(2)
    q = rng.uniform(-1, 9, size=(5000, 3))

    def snapshot():
        return (a.stats(), [a.get_option(k) for k in ("variant", "launches", "autotune")]), a.elem_ids, a.positions, \
            a.flux, a.flux_moments()

    def same(x, y, label):
        assert x[0] == y[0], label
        for u, v in zip(x[1:], y[1:]):
            np.testing.assert_array_equal(u, v, err_msg=label)

    before = a.stats()
    a.locate(q)  # before CopyInitialPosition
    assert a.stats() == before
    for e, wl in zip((a, b), wls):
        e.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    qd = torch.from_numpy(q).cuda()
    for step in range(3):
        for e, wl in zip((a, b), wls):
            o, d, f, w = wl.next_step()
            e.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
        s0 = snapshot()
        a.locate(q)
        a.evaluate(q)
        a.locate_device(qd)
        torch.cuda.synchronize()
        same(s0, snapshot(), f"step {step}")
        assert_same_particles(a, b, f"step {step}")


def _want(eng, c, t, pts, moments):
    nf, _ = eng.normalized_flux_time()
    elem = eng.locate(pts)
    inside = elem >= 0
    want = np.full(nf.shape[:3] + (len(pts),), np.nan)
    want[..., inside] = nf[..., elem[inside]]
    if moments:
        g = eng.flux_gradient()
        cen = np.asarray(c)[np.asarray(t)].mean(axis=1)
        dx = pts[inside] - cen[elem[inside]]
        want[..., inside] += (g[..., elem[inside], :] * dx).sum(-1)
    return want, elem


@pytest.mark.parametrize("moments", [0, 1])
@pytest.mark.parametrize("layout", ["plain", "bins", "scores_time"])
def test_evaluate_equals_the_recomputation(layout, moments):
    c, t = kuhn_box(6, 5, 4)
    n = 6000
    wl = SyntheticWorkload(box=(6.0, 5.0, 4.0), num_particles=n, mean_length=1.0, seed=5)
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_option("chunk", 1024)
    nscores, edges, nbins = (3, EDGES, 2) if layout == "scores_time" else (1, None, 2 if layout == "bins" else 1)
    _configure(eng, nscores, edges, moments=moments, nbins=nbins)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    rng = np.random.default_rng(8)
    for _ in range(2):
        o, d, f, w = wl.next_step()
        bins = rng.integers(0, nbins, n).astype(np.int32)
        r = responses(rng, n, nscores)
        if edges is not None:
            times, speeds = time_workload(rng, o, d, 6.0, edges)
            _move(eng, "timed", o, d, f, w, r, times, speeds, bins)
        elif nbins > 1:
            _move(eng, "binned", o, d, f, w, bins=bins)
        else:
            _move(eng, "plain", o, d, f, w)
    pts = np.concatenate([rng.uniform(-0.5, 6.5, size=(4000, 3)), non_finite_points()])
    want, welem = _want(eng, c, t, pts, moments)
    got, elem = eng.evaluate(pts)
    np.testing.assert_array_equal(elem, welem)
    assert np.isnan(got[..., elem < 0]).all()
    np.testing.assert_allclose(got[..., elem >= 0], want[..., elem >= 0], rtol=1e-12, atol=1e-12 * np.abs(want[..., elem >= 0]).max())
    first, _ = eng.evaluate(pts, first_only=True)
    np.testing.assert_array_equal(first, got[0, 0, 0])
    if moments:  # at the centroid the reconstruction is the element's value
        nf, _ = eng.normalized_flux_time()
        cen = np.asarray(c)[np.asarray(t)].mean(axis=1)
        at_c, e2 = eng.evaluate(cen)
        np.testing.assert_array_equal(e2, np.arange(len(t)))
        np.testing.assert_allclose(at_c, nf, rtol=1e-12, atol=1e-14 * np.abs(nf).max())


def test_evaluate_normalisation_cache_and_refusals():
    import ctypes as C

    c, t = kuhn_box(5, 5, 5)
    n = 3000
    wl = SyntheticWorkload(box=(5.0, 5.0, 5.0), num_particles=n, mean_length=1.0, seed=6)
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_moments(1)
    pts = np.random.default_rng(1).uniform(0.01, 4.99, size=(777, 3))
    eng.set_source_normalization(3)
    with pytest.raises(RuntimeError):  # no source weight seen yet: fails as get_normalized_flux does
        eng.evaluate(pts)
    with pytest.raises(RuntimeError):
        eng.normalized_flux()
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())

    def move():
        o, d, f, w = wl.next_step()
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())

    def check(label):
        want, _ = _want(eng, c, t, pts, 1)
        got, _ = eng.evaluate(pts)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max(), err_msg=label)
        return got

    move()
    v3 = check("mode 3")
    move()  # a move invalidates the table
    v3b = check("after a move")
    assert not np.array_equal(v3, v3b)
    eng.set_source_normalization(2, 7.5)  # so does a normalisation change
    v2 = check("mode 2")
    eng.set_source_normalization(0)
    v0 = check("mode 0")
    np.testing.assert_allclose(v2, v0 / 7.5, rtol=1e-12)
    eng.reset_tally()  # and a reset
    got, _ = eng.evaluate(pts)
    assert (got == 0).all()
    # n: npts or everything, nothing else
    L = eng._L
    out = np.empty(2 * len(pts))
    p = np.ascontiguousarray(pts)
    dp = C.POINTER(C.c_double)
    assert L.pumitally_evaluate_points(eng._h, p.ctypes.data_as(dp), len(pts), out.ctypes.data_as(dp), 2 * len(pts), None) != 0
    assert L.pumitally_evaluate_points(eng._h, p.ctypes.data_as(dp), len(pts), out.ctypes.data_as(dp), len(pts), None) == 0


def test_cxx_program_with_point_queries(tmp_path):
    """A C++ caller of PumiTallyExtras.h: LocatePoints and EvaluatePoints next to the reference class."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "locate_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "locate_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "LOCATE_OK" in out, out
