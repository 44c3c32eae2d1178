"""Cosine bins of the face currents (pumitally_set_current_cosine_bins): every crossing of the face currents also goes
to the bin of the cosine between its flight and the face normal that points the way it travels.  Weights are dyadic
(k / 8), so every sum is exact in any order; crossings within 1e-9 of a cosine edge are not flown, so the comparisons
with the exact reference are bit for bit."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from current_cosines_ref import cosine_walk, reference_cosine_currents
from face_currents_ref import unit_planes
from helpers import ROOT, box_case, l_shaped_mesh
from pumiumtally_b200.mesh import delaunay_box, kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_face_currents import EDGES, KINDS, _configure, _interior_points, _move
from test_gpu_scores import _bins, engine

pytestmark = pytest.mark.gpu

MU_EDGES = np.array([0.0, 0.15, 0.4, 0.55, 0.8, 0.95, 1.0])
MESHES = {
    "kuhn": lambda: box_case((5, 6, 4), 1)[:2],
    "l_shaped": lambda: l_shaped_mesh(6, 6, 3),
    "delaunay": lambda: delaunay_box(600),
}


def _regions(coords, t2v, nreg=5):
    c = coords[t2v].mean(axis=1)
    return (np.floor((c[:, 0] - c[:, 0].min()) / (np.ptp(c[:, 0]) + 1e-12) * nreg)).astype(np.int32).clip(0, nreg - 1)


def _run(coords, t2v, n, kind, variant, device, mu_edges=MU_EDGES, steps=2, seed=0, regions=True):
    """Moves with cosine bins against the exact reference and against a twin engine without cosine bins."""
    rng = np.random.default_rng(seed)
    eng = engine(coords, t2v, n, variant)
    eng.set_current_cosine_bins(mu_edges)
    _configure(eng, kind)
    other = engine(coords, t2v, n, variant)
    _configure(other, kind)
    reg = _regions(coords, t2v)
    if regions:
        for e in (eng, other):
            e.set_regions(reg, 5)
            e.set_region_currents(True)
    adj = eng.adjacency
    planes = unit_planes(coords, t2v)
    ntime, nbins, C = (len(EDGES) - 1 if kind == "timed" else 1), eng.score_bins, len(mu_edges) - 1
    want_out = np.zeros((ntime, nbins, C, len(t2v), 4))
    want_in = np.zeros_like(want_out)
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    init = _interior_points(rng, coords, t2v, n)
    for e in (eng, other):
        e.CopyInitialPosition(init.reshape(-1).copy())
    for step in range(steps):
        o = _interior_points(rng, coords, t2v, n)
        w = rng.integers(1, 17, n) / 8.0
        r = np.ascontiguousarray(rng.uniform(0.0, 2.0, (n, eng.scores)))
        bins = _bins(n, nbins, step) if nbins > 1 else None
        ones = np.ones(n, dtype=np.int8)
        for e in (eng, other):
            _move(e, kind, o, o, ones, np.zeros(n), (bins, r, np.zeros(n), np.ones(n)), device)
        ok = (eng.positions == o).all(axis=1)
        start = eng.elem_ids.astype(np.int64)
        u = rng.normal(size=(n, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        d = o + u * rng.exponential(0.6 * (hi - lo).max(), n)[:, None]
        times = rng.uniform(EDGES[0] - 1.0, EDGES[-1] + 0.5, n)
        speeds = rng.uniform(0.3, 3.0, n)
        tpp = np.linalg.norm(d - o, axis=1) / speeds
        te = EDGES if kind == "timed" else None
        fly = ok & (rng.random(n) < 0.9)
        cr = cosine_walk(planes, adj, start, o, d, fly, mu_edges, times, tpp, te)
        fly &= ~cr[5]
        cr = cosine_walk(planes, adj, start, o, d, fly, mu_edges, times, tpp, te)
        assert not cr[5][fly].any()
        for e in (eng, other):
            _move(e, kind, o, d, fly.astype(np.int8), w, (bins, r, times, speeds), device)
        a, b = reference_cosine_currents(adj, cr, w, bins, ntime, nbins, mu_edges)
        want_out += a
        want_in += b
    got_out, got_in = eng.face_current_results(0), eng.face_current_results(1)
    np.testing.assert_array_equal(got_out, want_out, err_msg=f"{kind} v{variant} outgoing")
    np.testing.assert_array_equal(got_in, want_in, err_msg=f"{kind} v{variant} incoming")
    hull = adj < 0
    np.testing.assert_array_equal(eng.leakage(0), (want_out * hull).sum(axis=(3, 4)))
    if regions:
        _check_region_currents(eng, adj, reg, want_out)
    np.testing.assert_array_equal(eng.elem_ids, other.elem_ids)
    np.testing.assert_array_equal(eng.positions, other.positions)
    fa, fb = eng.flux_time, other.flux_time
    np.testing.assert_allclose(fa, fb, rtol=1e-12, atol=1e-14 * np.abs(fb).max())
    return eng, other


def _check_region_currents(eng, adj, reg, want_out):
    """Partials: the outgoing currents of the faces between two regions, and of the hull faces into -2; nets: the
    difference of the two partials of a pair, in every cosine bin."""
    frm, to = eng.region_current_pairs()
    P = len(frm)
    E = len(adj)
    e, f = np.nonzero(np.ones((E, 4), dtype=bool))
    nb = adj[e, f]
    src = reg[e]
    dst = np.where(nb >= 0, reg[np.maximum(nb, 0)], -2)
    keep = src != dst
    pair = {(int(a), int(b)): p for p, (a, b) in enumerate(zip(frm, to))}
    idx = np.array([pair[(int(a), int(b))] for a, b in zip(src[keep], dst[keep])])
    T, B, C = want_out.shape[:3]
    want = np.zeros((T, B, C, P))
    vals = want_out[:, :, :, e[keep], f[keep]]
    for q in range(len(idx)):
        want[..., idx[q]] += vals[..., q]
    np.testing.assert_array_equal(eng.region_current_results(0), want)
    rev = np.array([pair.get((int(b), int(a)), -1) for a, b in zip(frm, to)])
    net = want - np.where(rev >= 0, want[..., np.maximum(rev, 0)], 0.0)
    np.testing.assert_array_equal(eng.region_current_results(1), net)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("variant", [0, 8, 16, 24])
def test_cosines_match_the_exact_reference(variant, kind):
    coords, t2v = MESHES["kuhn"]()
    _run(coords, t2v, 5000, kind, variant, device=False, seed=10 + variant + 7 * KINDS.index(kind))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("variant", [0, 8, 16, 24])
def test_device_moves_match_the_exact_reference(variant, kind):
    coords, t2v = MESHES["kuhn"]()
    _run(coords, t2v, 4000, kind, variant, device=True, seed=100 + variant + 7 * KINDS.index(kind))


@pytest.mark.parametrize("kind", ["plain", "timed", "moment"])
@pytest.mark.parametrize("mesh", ["l_shaped", "delaunay"])
@pytest.mark.parametrize("variant", [8, 16, 24])
def test_other_meshes(mesh, variant, kind):
    coords, t2v = MESHES[mesh]()
    _run(coords, t2v, 4000, kind, variant, device=False, seed=300 + variant + 7 * KINDS.index(kind))


def test_edges_that_do_not_cover_the_range():
    coords, t2v = MESHES["kuhn"]()
    _run(coords, t2v, 5000, "binned", 8, device=False, mu_edges=np.array([0.2, 0.5, 0.7]), seed=5)


@pytest.mark.parametrize("C", [1, 4, 64])
def test_sum_over_cosine_bins_is_the_result_without_them(C):
    """Full-size c2 with unit weights: every current sum is an exact integer, whatever the order of the reductions."""
    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    wl = SyntheticWorkload(cfg["cells"], cfg["particles"], mean_length=cfg["mean_length"], mu_min=cfg["mu_min"])
    reg = _regions(coords, t2v, 8)
    engs = []
    for cos in (True, False):
        e = engine(coords, t2v, wl.n)
        e.set_face_currents(True)
        if cos:
            e.set_current_cosine_bins(np.linspace(0.0, 1.0, C + 1))
        e.set_regions(reg, 8)
        e.set_region_currents(True)
        e.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
        engs.append(e)
    w = np.ones(wl.n)
    for _ in range(2):
        o, d, f, _ = wl.next_step()
        for e in engs:
            e.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
    a, b = engs
    assert a.current_cosine_bins == C
    for dr in (0, 1):
        np.testing.assert_array_equal(a.face_current_results(dr).sum(axis=2), b.face_current_results(dr))
    np.testing.assert_array_equal(a.leakage(0).sum(axis=2), b.leakage(0))
    for which in (0, 1):
        np.testing.assert_array_equal(a.region_current_results(which).sum(axis=2), b.region_current_results(which))
    fa, fb = a.flux_time, b.flux_time
    np.testing.assert_allclose(fa, fb, rtol=1e-12, atol=1e-14 * np.abs(fb).max())


def test_isotropic_flux_gives_b2_minus_a2():
    """Homogeneous unit box, origins uniform, directions isotropic, flights of fixed length L: on the faces of elements
    whose centroid lies farther than L plus the cell diameter from the hull the angular flux is isotropic, so the share
    of crossings with cosine in [a, b) is b^2 - a^2.  Every bin of 8 within 5 sigma of the multinomial.  L is a quarter
    of the cell edge, shorter than the spacing of any family of parallel faces, so no flight crosses two faces of the
    same normal (whose cosines would be equal and the crossings not independent)."""
    nc = 24
    coords, t2v = kuhn_box(nc, nc, nc, 1.0, 1.0, 1.0)  # [0, 1]^3, cell edge 1 / nc
    n = 4_000_000
    L = 0.25 / nc
    eng = engine(coords, t2v, n)
    eng.set_face_currents(True)
    edges = np.linspace(0.0, 1.0, 9)
    eng.set_current_cosine_bins(edges)
    rng = np.random.default_rng(3)
    o = rng.uniform(0.0, 1.0, (n, 3))
    eng.CopyInitialPosition(o.reshape(-1).copy())
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    eng.MoveToNextLocation(o.reshape(-1).copy(), (o + L * u).reshape(-1).copy(), np.ones(n, np.int8), np.ones(n))
    out = eng.face_current_results(0)[0, 0]  # [C, E, 4]
    cent = coords[t2v].mean(axis=1)
    margin = L + np.sqrt(3.0) / nc
    inner = ((cent > margin) & (cent < 1.0 - margin)).all(axis=1)
    assert inner.sum() > 40_000, inner.sum()  # the interior cells, not a corner
    counts = out[:, inner].sum(axis=(1, 2))
    N = counts.sum()
    p = edges[1:] ** 2 - edges[:-1] ** 2
    sigma = np.sqrt(N * p * (1 - p))
    assert N > 1e5
    assert (np.abs(counts - N * p) < 5 * sigma).all(), (counts / N, p)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_batch_statistics(mode):
    coords, t2v, _ = box_case((5, 5, 4), 1)
    n = 3000
    eng = engine(coords, t2v, n, 8)
    eng.set_score_bins(2)
    eng.set_face_currents(True)
    eng.set_current_cosine_bins([0.0, 0.3, 0.7, 1.0])
    reg = _regions(coords, t2v)
    eng.set_regions(reg, 5)
    eng.set_region_currents(True)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(mode, 3.0 if mode == 2 else 1.0)
    rng = np.random.default_rng(mode)
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
    vals = {0: [], 1: [], "leak": [], "rp": [], "rn": []}
    for b in range(8):
        o = eng.positions
        d = o + rng.normal(size=(n, 3)) * rng.uniform(0.2, 3.0, (n, 1))
        w = rng.integers(1, 17, n) / 8.0
        eng.MoveToNextLocationBinned(o.reshape(-1).copy(), d.reshape(-1).copy(), np.ones(n, np.int8), w,
                                     _bins(n, 2, b))
        vals[0].append(eng.face_current_results(0))
        vals[1].append(eng.face_current_results(1))
        vals["leak"].append(eng.leakage(0))
        vals["rp"].append(eng.region_current_results(0))
        vals["rn"].append(eng.region_current_results(1))
        eng.end_batch()
    for key, got in ((0, lambda k: eng.face_current_results(0, k)), (1, lambda k: eng.face_current_results(1, k)),
                     ("leak", eng.leakage), ("rp", lambda k: eng.region_current_results(0, k)),
                     ("rn", lambda k: eng.region_current_results(1, k))):
        x = np.stack(vals[key])
        mean, se = x.mean(axis=0), x.std(axis=0, ddof=1) / np.sqrt(len(x))
        scale = np.abs(x).max() + 1e-300
        np.testing.assert_allclose(got(1), mean, rtol=1e-13, atol=1e-14 * scale)
        np.testing.assert_allclose(got(2), se, rtol=1e-9, atol=1e-12 * scale)
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = np.where(mean != 0, se / np.abs(mean), 0.0)
        # a net whose mean cancels to rounding noise has an ill-conditioned relative error: not compared
        ok = np.abs(mean) > 1e-9 * scale
        np.testing.assert_allclose(got(3)[ok], rel[ok], rtol=1e-8, atol=1e-12)


def test_checkpoints(tmp_path, capfd):
    coords, t2v, _ = box_case((5, 5, 4), 1)
    n = 3000
    rng = np.random.default_rng(9)
    init = _interior_points(rng, coords, t2v, n)

    def make(mu_edges):
        e = engine(coords, t2v, n, 8)
        e.set_face_currents(True)
        if mu_edges is not None:
            e.set_current_cosine_bins(mu_edges)
        e.set_batch_statistics(True)
        e.CopyInitialPosition(init.reshape(-1).copy())
        return e

    def fly(e, seed):
        r = np.random.default_rng(seed)
        o = e.positions
        e.MoveToNextLocation(o.reshape(-1).copy(), (o + r.normal(size=(n, 3))).reshape(-1).copy(),
                             np.ones(n, np.int8), r.integers(1, 17, n) / 8.0)

    E1 = [0.0, 0.5, 1.0]
    eng = make(E1)
    plain = make(None)
    for b in range(3):
        for e in (eng, plain):
            fly(e, b)
            if b < 2:
                e.end_batch()
    p = str(tmp_path / "a.ckpt")
    eng.save_checkpoint(p)
    assert open(p, "rb").read(12)[8] == 2  # the cosine edges need format version 2
    loaded = make(E1)
    loaded.load_checkpoint(p)
    for k in range(4):
        for dr in (0, 1):
            np.testing.assert_array_equal(loaded.face_current_results(dr, k), eng.face_current_results(dr, k))
        np.testing.assert_array_equal(loaded.leakage(k), eng.leakage(k))
    p2 = str(tmp_path / "b.ckpt")
    loaded.save_checkpoint(p2)
    assert open(p, "rb").read() == open(p2, "rb").read()
    eng.end_batch()
    p3 = str(tmp_path / "c.ckpt")
    eng.save_checkpoint(p3)
    merged = make(E1)
    merged.merge_checkpoint(p3)
    np.testing.assert_array_equal(merged.face_current_results(0, 1), eng.face_current_results(0, 1))
    np.testing.assert_array_equal(merged.leakage(2), eng.leakage(2))
    # without cosine bins the file keeps version 1 (its bytes: test_a_file_without_bins_keeps_the_previous_bytes)
    pp = str(tmp_path / "plain.ckpt")
    plain.save_checkpoint(pp)
    assert open(pp, "rb").read(12)[8] == 1
    # other edges, bins against none and none against bins: refused, the message names the cosine bins
    before = merged.face_current_results(0, 1)
    for target, path in ((make([0.0, 0.25, 1.0]), p3), (make([0.0, 0.5 + 2**-40, 1.0]), p3), (make(None), p3),
                         (merged, pp)):
        capfd.readouterr()
        with pytest.raises(RuntimeError):
            target.load_checkpoint(path)
        assert "cosine" in capfd.readouterr().err
        with pytest.raises(RuntimeError):
            target.merge_checkpoint(path)
        assert "cosine" in capfd.readouterr().err
    np.testing.assert_array_equal(merged.face_current_results(0, 1), before)


FIXTURE = os.path.join(ROOT, "tests", "golden", "face_currents_v1.ckpt")


def write_fixture_checkpoint(cls, path, bins_set_and_removed=False):
    """The state of tests/golden/face_currents_v1.ckpt: one particle (every sum has a single order, so the bits do not
    depend on the order of the reductions) flying three moves through a 3x3x2 Kuhn box with face currents and batch
    statistics, the last one out through the hull, two batches folded and the third open.  The fixture was written by
    this function with the build before cosine bins existed (cls its PumiTally)."""
    coords, t2v = kuhn_box(3, 3, 2)
    e = cls.from_arrays(coords, t2v, 1)
    e.set_option("variant", 8)
    e.set_face_currents(True)
    if bins_set_and_removed:
        e.set_current_cosine_bins([0.0, 0.5, 1.0])
        e.set_current_cosine_bins(None)
    e.set_batch_statistics(True)
    e.CopyInitialPosition(np.array([0.3, 0.4, 0.5]))
    for b, (d, w) in enumerate((((2.6, 1.2, 1.7), 0.75), ((0.4, 2.7, 0.3), 1.25), ((5.0, 1.5, 1.0), 0.5))):
        e.MoveToNextLocation(e.positions.reshape(-1).copy(), np.array(d), np.ones(1, np.int8), np.array([w]))
        if b < 2:
            e.end_batch()
    e.save_checkpoint(path)


@pytest.mark.parametrize("removed", [False, True], ids=["never_set", "set_and_removed"])
def test_a_file_without_bins_keeps_the_previous_bytes(tmp_path, removed):
    """Saved without cosine bins (never set, or set and removed), a checkpoint is byte for byte the file the build
    before cosine bins wrote for the same state, and loads back."""
    p = str(tmp_path / "x.ckpt")
    write_fixture_checkpoint(PumiTally, p, removed)
    got, want = open(p, "rb").read(), open(FIXTURE, "rb").read()
    assert got == want
    coords, t2v = kuhn_box(3, 3, 2)
    e = PumiTally.from_arrays(coords, t2v, 1)
    e.set_face_currents(True)
    e.set_batch_statistics(True)
    e.load_checkpoint(FIXTURE)
    assert e.face_current_results(0, 1).sum() > 0 and e.leakage(0)[0, 0] > 0


def test_refusals_change_nothing():
    coords, t2v, _ = box_case((4, 4, 4), 1)
    n = 2000
    eng = engine(coords, t2v, n, 8)
    eng.set_face_currents(True)
    rng = np.random.default_rng(1)
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())

    def fly():
        o = eng.positions
        eng.MoveToNextLocation(o.reshape(-1).copy(), (o + rng.normal(size=(n, 3))).reshape(-1).copy(),
                               np.ones(n, np.int8), rng.integers(1, 17, n) / 8.0)

    fly()
    shape0 = eng.face_current_results(0).shape
    eng.set_current_cosine_bins([0.0, 0.5, 1.0])
    assert eng.current_cosine_bins == 2 and eng.get_option("current_cosine_bins") == 2
    fly()
    before = eng.face_current_results(0)
    assert before.shape == shape0[:2] + (2,) + shape0[2:]
    assert eng.leakage(0).shape == (1, 1, 2)
    bad = ([0.5], [0.0, 0.0, 1.0], [0.5, 0.2], [-0.1, 1.0], [0.0, 1.1], [0.0, np.nan], [0.0, np.inf],
           np.linspace(0.0, 1.0, 66))
    for edges in bad:
        with pytest.raises(ValueError):
            eng.set_current_cosine_bins(edges)
        assert eng.current_cosine_bins == 2
        np.testing.assert_array_equal(eng.face_current_results(0), before)
    from pumiumtally_b200.tally import _dp

    assert eng._L.pumitally_set_current_cosine_bins(eng._h, None, 3) != 0
    buf = np.empty(before.size // 2)
    assert eng._L.pumitally_get_face_current_results(eng._h, 0, 0, buf.ctypes.data_as(_dp), buf.size) != 0
    assert eng._L.pumitally_get_leakage(eng._h, 0, buf.ctypes.data_as(_dp), 1) != 0
    np.testing.assert_array_equal(eng.face_current_results(0), before)
    eng.set_current_cosine_bins(np.linspace(0.0, 1.0, 65))  # 64 bins: the most
    assert eng.current_cosine_bins == 64
    eng.set_current_cosine_bins(None)
    assert eng.current_cosine_bins == 0
    assert eng.face_current_results(0).shape == shape0 and eng.leakage(0).shape == (1, 1)


def test_refused_after_comm_init():
    coords, t2v, _ = box_case((4, 4, 4), 1)
    eng = engine(coords, t2v, 1000, 8)
    eng.set_face_currents(True)
    eng.comm_init(0, 1, PumiTally.nccl_unique_id())
    with pytest.raises(ValueError):
        eng.set_current_cosine_bins([0.0, 1.0])
    assert eng.current_cosine_bins == 0


def test_vtk_arrays(tmp_path):
    from vtk_reader import read_vtu_cell_data

    coords, t2v, _ = box_case((4, 4, 3), 1)
    n = 2000
    eng = engine(coords, t2v, n, 8)
    eng.set_score_bins(2)
    eng.set_face_currents(True)
    eng.set_current_cosine_bins([0.0, 0.4, 1.0])
    rng = np.random.default_rng(2)
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
    o = eng.positions
    eng.MoveToNextLocationBinned(o.reshape(-1).copy(), (o + rng.normal(size=(n, 3))).reshape(-1).copy(),
                                 np.ones(n, np.int8), rng.integers(1, 17, n) / 8.0, _bins(n, 2, 0))
    path = str(tmp_path / "r.vtu")
    eng.WriteTallyResults(path)
    with open(os.path.join(path, "pieces", "piece_0.vtu"), "rb") as f:
        text = f.read()
    for name in (b"current_out", b"current_in", b"current_out_mu0", b"current_out_mu1", b"current_in_mu0",
                 b"current_in_mu1"):
        assert b'Name="' + name + b'" NumberOfComponents="4"' in text, name
    assert b"current_out_mu2" not in text
    arrays = read_vtu_cell_data(os.path.join(path, "pieces", "piece_0.vtu"))
    for d in ("out", "in"):
        tot = arrays[f"current_{d}"]
        np.testing.assert_array_equal(arrays[f"current_{d}_mu0"] + arrays[f"current_{d}_mu1"], tot)
        assert tot.sum() > 0


@pytest.mark.skipif(shutil.which("cmake") is None or shutil.which("ninja") is None, reason="cmake/ninja not available")
def test_cxx_program_against_the_installed_package(tmp_path):
    """A C++ caller of SetCurrentCosineBins (tests/current_cosines_demo.cpp), built with find_package(pumitally)
    against the installed CMake package and run."""
    build, inst, app = tmp_path / "build", tmp_path / "inst", tmp_path / "app"
    build.mkdir(); app.mkdir()
    common = ["-G", "Ninja", "-DCMAKE_CXX_COMPILER=/usr/bin/g++"]
    subprocess.check_call(["cmake", *common, "-DCMAKE_CUDA_COMPILER=/usr/local/cuda/bin/nvcc",
                           "-DCMAKE_CUDA_HOST_COMPILER=/usr/bin/g++", f"-DCMAKE_INSTALL_PREFIX={inst}", ROOT],
                          cwd=build, stdout=subprocess.DEVNULL)
    subprocess.check_call(["ninja", "install"], cwd=build, stdout=subprocess.DEVNULL)
    (app / "CMakeLists.txt").write_text(
        "cmake_minimum_required(VERSION 3.20)\nproject(app CXX)\n"
        "find_package(pumitally REQUIRED)\n"
        f"add_executable(app {os.path.join(ROOT, 'tests', 'current_cosines_demo.cpp')})\n"
        "target_compile_features(app PRIVATE cxx_std_17)\n"
        "target_link_libraries(app PRIVATE pumitally::pumitally)\n")
    appb = tmp_path / "appbuild"
    appb.mkdir()
    subprocess.check_call(["cmake", *common, f"-DCMAKE_PREFIX_PATH={inst}", str(app)], cwd=appb,
                          stdout=subprocess.DEVNULL)
    subprocess.check_call(["ninja"], cwd=appb, stdout=subprocess.DEVNULL)
    out = subprocess.check_output([str(appb / "app")], cwd=str(tmp_path), text=True)
    assert "CURRENT_COSINES_OK" in out, out


def _two_gpu(eng, c, t, rank, world, n):
    rng = np.random.default_rng(77)
    init = _interior_points(rng, c, t, n)
    mine = slice(rank, n, world)
    eng.CopyInitialPosition(init[mine].reshape(-1).copy())
    for _ in range(2):
        o = _interior_points(rng, c, t, n)
        d = o + rng.normal(size=(n, 3)) * 1.5
        w = rng.integers(1, 17, n) / 8.0
        m = len(init[mine])
        eng.MoveToNextLocation(o[mine].reshape(-1).copy(), d[mine].reshape(-1).copy(), np.ones(m, np.int8),
                               w[mine].copy())
        eng.end_batch()
    return [eng.face_current_results(dr, k) for dr in (0, 1) for k in (1, 2)] + [eng.leakage(1), eng.leakage(2)]


def _two_gpu_worker(rank, world, port, q):
    import sys

    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pumiumtally_b200.distributed import broadcast_unique_id

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    c, t = kuhn_box(5, 5, 5)
    eng = PumiTally.from_arrays(c, t, 2000 // world, device=rank)
    eng.set_face_currents(True)
    eng.set_current_cosine_bins([0.0, 0.5, 1.0])
    eng.set_batch_statistics(True)
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    q.put((rank, _two_gpu(eng, c, t, rank, world, 2000)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpus_give_the_one_rank_results():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 517) % 1000
    procs = [ctx.Process(target=_two_gpu_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    c, t = kuhn_box(5, 5, 5)
    one = PumiTally.from_arrays(c, t, 2000)
    one.set_face_currents(True)
    one.set_current_cosine_bins([0.0, 0.5, 1.0])
    one.set_batch_statistics(True)
    want = _two_gpu(one, c, t, 0, 1, 2000)
    for rank in range(2):
        for got, w in zip(res[rank][1], want):
            np.testing.assert_allclose(got, w, rtol=1e-12, atol=0.0, err_msg=f"rank {rank}")
