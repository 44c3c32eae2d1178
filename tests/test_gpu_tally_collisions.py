"""Collision estimator (pumitally_set_collision_estimator): events scored at located points or at the particles'
positions into a collision tally of the track-length tally's configuration.  Checked against the numpy reference
(tests/collisions_ref.py); the collision calls must change nothing else, and on a homogeneous box the collision and
track-length estimates of the same flux must agree."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from collisions_ref import assert_close, event_mix, reference_collisions
from helpers import ROOT
from locate_ref import MESHES
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_moments import _configure, _move
from test_gpu_scores import assert_same_particles, responses
from time_bins_ref import time_workload

pytestmark = pytest.mark.gpu

EDGES = np.array([0.0, 1.0, 2.0, 3.0, 4.0])  # 4 time bins
CASES = {  # nscores, nbins, time edges, moments
    "s1": (1, 1, None, 0),
    "s1_b3_mo": (1, 3, None, 1),
    "s3_b3_t": (3, 3, EDGES, 0),
    "s8_t_mo": (8, 1, EDGES, 1),
    "s3_b3_t_mo": (3, 3, EDGES, 1),
}
_dp = C.POINTER(C.c_double)


def _centre(coords):
    c = np.asarray(coords)
    return 0.5 * (c.min(axis=0) + c.max(axis=0))


def _geometry(coords, t2v):
    """vertex-average centroids [E, 3], volumes [E] and second-moment matrices M [E, 3, 3] (linear_moments())"""
    v = np.asarray(coords, dtype=np.float64)[np.asarray(t2v)]
    cen = v.mean(axis=1)
    d = v - cen[:, None, :]
    vol = np.abs(np.einsum("ij,ij->i", d[:, 1] - d[:, 0], np.cross(d[:, 2] - d[:, 0], d[:, 3] - d[:, 0]))) / 6.0
    return cen, vol, vol[:, None, None] / 20.0 * np.einsum("eqa,eqb->eab", d, d)


def _engine(c, t, n, nscores, nbins, edges, moments):
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_collision_estimator(True)
    _configure(eng, nscores, edges, moments=moments, nbins=nbins)
    assert eng.collision_estimator and eng.get_option("collision_estimator") == 1
    return eng


def _to_device(*arrays):
    import torch

    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def check_results(eng, coords, t2v, wm0, wR, a0, aR, moments, label, modes=((0, 1.0), (1, 1.0), (2, 37.0))):
    """kinds 0-3 against the reference: raw, raw / volume / divisor, m1 = R - (c_e - C) m0, M^-1 m1 / divisor."""
    cen, vol, M = _geometry(coords, t2v)
    raw = eng.collision_results(0)
    assert_close(raw, wm0, a0, f"{label} kind 0")
    want_m1 = None
    if moments:
        rel = cen - _centre(coords)
        want_m1 = wR - rel[None, None, None] * wm0[..., None]
        m1 = eng.collision_results(2)
        assert_close(m1, want_m1, aR + np.abs(rel)[None, None, None] * a0[..., None], f"{label} kind 2")
    else:
        for kind in (2, 3):
            with pytest.raises(RuntimeError):
                eng.collision_results(kind)
    for mode, value in modes:
        eng.set_source_normalization(mode, value)
        per = eng.source_normalization()
        np.testing.assert_allclose(eng.collision_results(1), raw / vol / per, rtol=1e-13, atol=0, err_msg=label)
        if moments:
            g = eng.collision_results(3)
            want = np.linalg.solve(M, m1[..., None])[..., 0] / per
            np.testing.assert_allclose(g, want, rtol=1e-9, atol=1e-12 * np.abs(want).max(), err_msg=label)
    eng.set_source_normalization(0)


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mesh", list(MESHES))
def test_located_events_match_the_reference(mesh, case, path):
    import torch

    nscores, nbins, edges, moments = CASES[case]
    c, t = MESHES[mesh]()
    eng = _engine(c, t, 16, nscores, nbins, edges, moments)
    eng.set_option("chunk", 1024)  # several chunks, the last one partial
    rng = np.random.default_rng(len(mesh) * 31 + len(case))
    pts, elem, w, r, bins, times = event_mix(mesh, c, t, rng, 2999, nscores, nbins, edges)
    r_in = None if nscores == 1 and case == "s1" else r
    b_in = None if nbins == 1 else bins
    if path == "host":
        eng.tally_collisions(pts, w, r_in, b_in, times)
    else:
        eng.tally_collisions_device(*_to_device(pts, w, r_in, b_in, times))
        torch.cuda.synchronize()
    wm0, wR, a0, aR, counts = reference_collisions(elem, pts, w, r_in, b_in, times, nbins, edges, len(t), _centre(c))
    assert (eng.get_option("collisions"), eng.get_option("collisions_outside"),
            eng.get_option("collisions_rejected")) == counts
    assert counts[0] > 600 and counts[1] > 50 and counts[2] >= 7
    check_results(eng, c, t, wm0, wR, a0, aR, moments, f"{mesh} {case} {path}")
    assert (eng.flux_time == 0).all() and eng.stats()["moves"] == 0


def _moved_engine(nscores, nbins, edges, moments, n=5000, seed=3, collision=True):
    c, t = kuhn_box(6, 5, 4)
    wl = SyntheticWorkload(box=(6.0, 5.0, 4.0), num_particles=n, mean_length=1.0, seed=seed)
    eng = PumiTally.from_arrays(c, t, n)
    if collision:
        eng.set_collision_estimator(True)
    _configure(eng, nscores, edges, moments=moments, nbins=nbins)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    rng = np.random.default_rng(seed)
    for _ in range(2):
        o, d, f, w = wl.next_step()
        if edges is not None:
            tt, vv = time_workload(rng, o, d, 6.0, edges)
            _move(eng, "timed", o, d, f, w, responses(rng, n, nscores), tt, vv, rng.integers(0, nbins, n).astype(np.int32))
        elif nscores > 1:
            _move(eng, "scored", o, d, f, w, responses(rng, n, nscores), bins=rng.integers(0, nbins, n).astype(np.int32))
        elif nbins > 1:
            _move(eng, "binned", o, d, f, w, bins=rng.integers(0, nbins, n).astype(np.int32))
        else:
            _move(eng, "plain", o, d, f, w)
    return eng, c, t, wl, rng


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("case", list(CASES))
def test_events_at_the_particles_match_the_reference(case, path):
    import torch

    nscores, nbins, edges, moments = CASES[case]
    eng, c, t, wl, rng = _moved_engine(nscores, nbins, edges, moments)
    n = wl.n
    collided = (rng.random(n) < 0.4).astype(np.int8)
    w = rng.uniform(0.1, 2.0, n)
    r = rng.uniform(-1.0, 2.0, (n, nscores))
    bins = rng.integers(-1, nbins + 1, n).astype(np.int32)
    times = None if edges is None else rng.uniform(-0.5, 4.5, n)
    elem, pos = eng.elem_ids, eng.positions
    if path == "host":
        eng.tally_collisions_at_particles(collided, w, r, bins, times)
    else:
        eng.tally_collisions_at_particles_device(*_to_device(collided, w, r, bins, times))
        torch.cuda.synchronize()
    sel = collided != 0
    wm0, wR, a0, aR, counts = reference_collisions(elem[sel], pos[sel], w[sel], r[sel], bins[sel],
                                                   None if times is None else times[sel], nbins, edges, len(t), _centre(c))
    assert counts[1] == counts[2] == 0 and counts[0] > 0.1 * n
    assert (eng.get_option("collisions"), eng.get_option("collisions_outside"),
            eng.get_option("collisions_rejected")) == counts
    check_results(eng, c, t, wm0, wR, a0, aR, moments, f"{case} {path}",
                  modes=((0, 1.0), (1, 1.0), (2, 37.0), (3, 1.0)))
    assert (collided == (sel * 1)).all()  # not zeroed


def test_collision_calls_change_nothing_else(tmp_path):
    import torch
    from vtk_reader import read_vtu_cell_data

    nscores, nbins, edges, moments = CASES["s3_b3_t_mo"]
    eng, c, t, wl, rng = _moved_engine(nscores, nbins, edges, moments, seed=4)
    twin, *_ = _moved_engine(nscores, nbins, edges, moments, seed=4, collision=False)

    def snapshot(e):
        return (e.stats(), [e.get_option(k) for k in ("variant", "launches", "autotune", "chunk", "pinned_path")]), \
            e.elem_ids, e.positions, e.flux_time, e.flux_moments()

    s0 = snapshot(eng)
    n = wl.n
    pts, _, w, r, bins, times = event_mix("kuhn", c, t, rng, 3000, nscores, nbins, edges)
    eng.tally_collisions(pts, w, r, bins, times)
    eng.tally_collisions_device(*_to_device(pts, w, r, bins, times))
    cw, cr, cb, ct = (rng.uniform(0.5, 1.5, n), rng.uniform(0.0, 1.0, (n, nscores)),
                      rng.integers(0, nbins, n).astype(np.int32), rng.uniform(0.0, 4.0, n))
    eng.tally_collisions_at_particles(np.ones(n, dtype=np.int8), cw, cr, cb, ct)
    eng.tally_collisions_at_particles_device(*_to_device(np.ones(n, dtype=np.int8), cw, cr, cb, ct))
    torch.cuda.synchronize()
    s1 = snapshot(eng)
    assert s0[0] == s1[0]
    for what, u, v in zip(("elements", "positions", "flux", "moments"), s0[1:], s1[1:]):
        np.testing.assert_array_equal(u, v, err_msg=what)
    # the same moves on an engine without the estimator: the same particles and track-length tally
    assert_same_particles(eng, twin, "twin")
    # within the order of the reductions: the first moments cancel, so their tolerance is relative to the largest
    for what, a, b in (("flux", eng.flux_time, twin.flux_time), ("moments", eng.flux_moments(), twin.flux_moments()),
                       ("normalised", eng.normalized_flux_time()[0], twin.normalized_flux_time()[0])):
        np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-11 * np.abs(b).max(), err_msg=what)
    d_out = torch.empty(eng.flux_time.size, dtype=torch.float64, device="cuda")
    eng.get_flux_device(d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(d_out.cpu().numpy().reshape(eng.flux_time.shape), eng.flux_time)
    # VTK: the old names plus the collision_ twins of all of them but the volume
    out, out_twin = str(tmp_path / "coll.vtk"), str(tmp_path / "twin.vtk")
    eng.WriteTallyResults(out)
    twin.WriteTallyResults(out_twin)
    cells = read_vtu_cell_data(os.path.join(out, "pieces", "piece_0.vtu"))
    cells_twin = read_vtu_cell_data(os.path.join(out_twin, "pieces", "piece_0.vtu"))
    assert set(cells) == set(cells_twin) | {"collision_" + k for k in cells_twin if k.startswith(("flux", "score"))}
    for k in cells_twin:
        np.testing.assert_allclose(cells[k], cells_twin[k], rtol=1e-9, atol=1e-11 * np.abs(cells_twin[k]).max(), err_msg=k)
    E = len(t)
    nf, g = eng.collision_results(1), eng.collision_results(3)  # [T, B, S, E] and [..., 3]

    def close(name, want):  # sums of values of both signs: the tolerance is relative to the largest
        np.testing.assert_allclose(cells[name].reshape(want.shape), want, rtol=1e-12, atol=1e-12 * np.abs(want).max(),
                                   err_msg=name)

    for k in range(nscores):
        name = "flux" if k == 0 else f"score{k}"
        close(f"collision_{name}", nf[:, :, k].sum(axis=(0, 1)))
        close(f"collision_{name}_grad", g[:, :, k].sum(axis=(0, 1)))
        for b in range(nbins):
            close(f"collision_{name}_bin{b}", nf[:, b, k].sum(axis=0))
        for j in range(len(edges) - 1):
            for b in range(nbins):
                np.testing.assert_array_equal(cells[f"collision_{name}_t{j}_bin{b}"], nf[j, b, k])
    # without scores, time bins or moments: the plain writer, the same rule
    plain, *_ = _moved_engine(1, 2, None, 0, seed=5)
    plain.tally_collisions_at_particles(np.ones(n, dtype=np.int8), np.ones(n))
    plain.WriteTallyResults(str(tmp_path / "plain.vtk"))
    pc = read_vtu_cell_data(os.path.join(str(tmp_path / "plain.vtk"), "pieces", "piece_0.vtu"))
    assert {k for k in pc if k.startswith(("flux", "score", "collision"))} == {
        "flux", "flux_bin0", "flux_bin1", "collision_flux", "collision_flux_bin0", "collision_flux_bin1"}
    pnf = plain.collision_results(1)
    np.testing.assert_allclose(pc["collision_flux"], pnf[0, :, 0].sum(axis=0), rtol=1e-12, atol=1e-300)
    np.testing.assert_array_equal(pc["collision_flux_bin1"], pnf[0, 1, 0])


def _octant_track_lengths(a, b, lo, hi):
    """[n, 8] length of every segment a -> b inside each octant box of [lo, hi] (slab clipping)"""
    mid = 0.5 * (lo + hi)
    d = b - a
    out = np.zeros((len(a), 8))
    for q in range(8):
        bits = [(q >> ax) & 1 for ax in range(3)]
        blo = np.array([lo[ax] if not bits[ax] else mid[ax] for ax in range(3)])
        bhi = np.array([mid[ax] if not bits[ax] else hi[ax] for ax in range(3)])
        t0, t1 = np.zeros(len(a)), np.ones(len(a))
        for ax in range(3):
            with np.errstate(divide="ignore", invalid="ignore"):
                ta, tb = (blo[ax] - a[:, ax]) / d[:, ax], (bhi[ax] - a[:, ax]) / d[:, ax]
            lo_t, hi_t = np.minimum(ta, tb), np.maximum(ta, tb)
            par = d[:, ax] == 0
            inside = (a[:, ax] >= blo[ax]) & (a[:, ax] <= bhi[ax])
            lo_t = np.where(par, np.where(inside, -np.inf, np.inf), lo_t)
            hi_t = np.where(par, np.where(inside, np.inf, -np.inf), hi_t)
            t0, t1 = np.maximum(t0, lo_t), np.minimum(t1, hi_t)
        out[:, q] = np.maximum(t1 - t0, 0.0) * np.linalg.norm(d, axis=1)
    return out


def test_collision_and_track_length_estimates_agree():
    """Homogeneous Kuhn box, Sigma_t = 1.3: particles born uniformly, isotropic, flights of Exp(Sigma_t) length.  Per
    octant, the track-length estimate (a move of weight 1) and the collision estimate (weights 1 / Sigma_t at the
    flights that end inside the box) agree within 5 sigma of the paired per-particle differences."""
    sig = 1.3
    cells = (8, 8, 8)
    c, t = kuhn_box(*cells)
    n = 200_000
    rng = np.random.default_rng(2024)
    o = rng.uniform(0.0, 8.0, (n, 3))
    mu = rng.uniform(-1.0, 1.0, n)
    phi = rng.uniform(0.0, 2 * np.pi, n)
    s = np.sqrt(1.0 - mu * mu)
    u = np.column_stack([s * np.cos(phi), s * np.sin(phi), mu])
    d = o + rng.exponential(1.0 / sig, n)[:, None] * u
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_collision_estimator(True)
    eng.CopyInitialPosition(o.reshape(-1).copy())
    _move(eng, "plain", o, d, np.ones(n, dtype=np.int8), np.ones(n))
    inside = ((d > 0.0) & (d < 8.0)).all(axis=1)
    pos = eng.positions
    np.testing.assert_array_equal(pos[inside], d[inside])
    eng.tally_collisions_at_particles(inside.astype(np.int8), np.full(n, 1.0 / sig))
    tl, col = eng.flux, eng.collision_results(0)[0, 0, 0]
    cen = np.asarray(c)[np.asarray(t)].mean(axis=1)
    oct_of_elem = ((cen >= 4.0).astype(int) * np.array([1, 2, 4])).sum(axis=1)
    ell = _octant_track_lengths(o, pos, np.zeros(3), np.full(3, 8.0))  # [n, 8]
    oct_of_dest = ((d >= 4.0).astype(int) * np.array([1, 2, 4])).sum(axis=1)
    for q in range(8):
        diff = ell[:, q] - (inside & (oct_of_dest == q)) / sig
        sigma = np.sqrt(n * diff.var())
        a, b = tl[oct_of_elem == q].sum(), col[oct_of_elem == q].sum()
        assert abs(a - ell[:, q].sum()) <= 1e-9 * a  # the host clip is the walk's track length
        assert abs(a - b) <= 5 * sigma, (q, a, b, sigma)
        assert sigma < 0.02 * a


def test_refusals_and_counters():
    nscores, nbins = 2, 2
    eng, c, t, wl, rng = _moved_engine(1, 1, None, 0, collision=False)
    n = wl.n
    L, h = eng._L, eng._h
    pts = rng.uniform(0.5, 3.5, (100, 3))
    w = np.ones(100)
    with pytest.raises(RuntimeError):  # the estimator is off
        eng.tally_collisions(pts, w)
    with pytest.raises(RuntimeError):
        eng.tally_collisions_at_particles(np.ones(n, dtype=np.int8), np.ones(n))
    with pytest.raises(RuntimeError):
        eng.collision_results(0)
    assert not eng.collision_estimator
    with pytest.raises(ValueError):
        eng.set_collision_estimator(2)
    eng.set_collision_estimator(True)
    eng.set_scores(nscores)
    eng.set_score_bins(nbins)
    eng.tally_collisions(pts, w, np.ones((100, nscores)))
    assert eng.get_option("collisions") == 100
    before = eng.collision_results(0)
    before_counts = [eng.get_option(k) for k in ("collisions", "collisions_outside", "collisions_rejected")]
    p = np.ascontiguousarray(pts)
    refused = [
        lambda: L.pumitally_tally_collisions(h, p.ctypes.data_as(_dp), 100, w.ctypes.data_as(_dp), None, None, None),
        lambda: L.pumitally_tally_collisions(h, p.ctypes.data_as(_dp), -1, w.ctypes.data_as(_dp),
                                             np.ones(200).ctypes.data_as(_dp), None, None),
        lambda: L.pumitally_tally_collisions_at_particles(h, np.ones(n, dtype=np.int8).ctypes.data_as(C.POINTER(C.c_int8)),
                                                          np.ones(n).ctypes.data_as(_dp), np.ones(2 * n).ctypes.data_as(_dp),
                                                          None, None, n - 1),
        lambda: L.pumitally_tally_collisions_at_particles(h, np.ones(n, dtype=np.int8).ctypes.data_as(C.POINTER(C.c_int8)),
                                                          np.ones(n).ctypes.data_as(_dp), None, None, None, n),
        lambda: L.pumitally_get_collision_results(h, 2, np.empty(3 * len(t)).ctypes.data_as(_dp), 3 * len(t)),
        lambda: L.pumitally_get_collision_results(h, 4, np.empty(len(t)).ctypes.data_as(_dp), len(t)),
        lambda: L.pumitally_get_collision_results(h, 0, np.empty(len(t) + 1).ctypes.data_as(_dp), len(t) + 1),
    ]
    for k, call in enumerate(refused):
        assert call() != 0, k
        np.testing.assert_array_equal(eng.collision_results(0), before)
        assert [eng.get_option(q) for q in ("collisions", "collisions_outside", "collisions_rejected")] == before_counts
    r2 = np.ones(2)
    assert L.pumitally_tally_collisions(h, p.ctypes.data_as(_dp), 0, w.ctypes.data_as(_dp), r2.ctypes.data_as(_dp), None,
                                        None) == 0
    assert eng.get_option("collisions") == 100
    eng.set_time_bins(EDGES)
    with pytest.raises(RuntimeError):  # times are required while time bins are set
        eng.tally_collisions(pts, w, np.ones((100, nscores)))
    # exact counters: 100 inside, 3 outside, 2 rejected (non-finite coordinate and time), 4 skipped (bin, time)
    q = np.concatenate([pts, [[-1.0, 1.0, 1.0], [1.0, 9.0, 1.0], [1e300, 0.0, 0.0], [np.nan, 1.0, 1.0], [1.0, 1.0, 1.0]],
                        pts[:4]])
    tt = np.concatenate([np.full(100, 0.5), [0.5, 0.5, 0.5, 0.5, np.inf], [-0.1, 4.0, 1.0, 1.0]])
    bb = np.concatenate([np.zeros(105, dtype=np.int32), [0, 0, -1, 2]]).astype(np.int32)
    eng.tally_collisions(q, np.ones(len(q)), np.ones((len(q), nscores)), bb, tt)
    assert [eng.get_option(k) for k in ("collisions", "collisions_outside", "collisions_rejected")] == [100, 3, 2]
    eng.reset_tally()
    assert [eng.get_option(k) for k in ("collisions", "collisions_outside", "collisions_rejected")] == [0, 0, 0]
    assert not eng.collision_results(0).any()
    eng.tally_collisions(q, np.ones(len(q)), np.ones((len(q), nscores)), bb, tt)
    eng.set_collision_estimator(True)  # resets
    assert eng.get_option("collisions") == 0 and not eng.collision_results(0).any()
    eng.set_collision_estimator(False)
    assert eng.get_option("collision_estimator") == 0


def test_collision_estimator_refused_after_comm_init():
    import torch
    import torch.distributed as dist

    if not dist.is_available():
        pytest.skip("torch.distributed unavailable")
    eng = PumiTally.from_spec("box:3,3,3", 100)
    try:
        eng.comm_init(0, 1, PumiTally.nccl_unique_id())
    except Exception as exc:  # no NCCL on this machine
        pytest.skip(f"comm_init unavailable: {exc}")
    with pytest.raises(ValueError):
        eng.set_collision_estimator(True)
    assert not eng.collision_estimator
    torch.cuda.synchronize()


def test_config_c2_ten_million_events():
    """Full-size c2 (998,250 tets): 10 M events at the particles after a device move, and 10 M located uniform points,
    against np.add.at with the engine's elements and locate() respectively."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    E = len(t2v)
    n = cfg["particles"]
    wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    eng = PumiTally.from_arrays(coords, t2v, n)
    eng.set_collision_estimator(True)
    s = torch.cuda.current_stream().cuda_stream
    eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
    o, d, f, w = (x.contiguous() for x in wl.next_step())
    eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
    g = torch.Generator(device="cuda").manual_seed(3)
    collided = (torch.rand(n, device="cuda", generator=g) < 0.5).to(torch.int8)
    cw = torch.rand(n, dtype=torch.float64, device="cuda", generator=g) + 0.5
    eng.tally_collisions_at_particles_device(collided, cw)
    torch.cuda.synchronize()
    sel = collided.cpu().numpy() != 0
    want = np.zeros(E)
    np.add.at(want, eng.elem_ids[sel], cw.cpu().numpy()[sel])
    got = eng.collision_results(0)[0, 0, 0]
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    assert eng.get_option("collisions") == sel.sum()
    eng.reset_tally()
    cells = np.array(cfg["cells"], dtype=np.float64)
    pts = (torch.rand((n, 3), dtype=torch.float64, device="cuda", generator=g) * torch.tensor(1.1 * cells, device="cuda")
           - torch.tensor(0.05 * cells, device="cuda")).contiguous()
    pw = torch.rand(n, dtype=torch.float64, device="cuda", generator=g) + 0.5
    eng.tally_collisions_device(pts, pw)
    torch.cuda.synchronize()
    elem = eng.locate(pts.cpu().numpy())
    inn = elem >= 0
    want = np.zeros(E)
    np.add.at(want, elem[inn], pw.cpu().numpy()[inn])
    np.testing.assert_allclose(eng.collision_results(0)[0, 0, 0], want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    assert (eng.get_option("collisions"), eng.get_option("collisions_outside")) == (inn.sum(), (~inn).sum())


def test_cxx_program_with_collisions(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SetCollisionEstimator, TallyCollisionsAtParticles and TallyCollisions next
    to the reference class."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "collisions_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "collisions_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "COLLISIONS_OK" in out, out


def _two_gpu_collisions_worker(rank, world, port, q):
    import sys

    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pumiumtally_b200.distributed import broadcast_unique_id

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    eng = PumiTally.from_spec("box:5,5,5", 100, device=rank)
    eng.set_scores(2)
    eng.set_collision_estimator(True)
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    rng = np.random.default_rng(rank)
    pts = rng.uniform(0.0, 5.0, (20_000, 3))
    eng.tally_collisions(pts, rng.uniform(0.5, 1.5, 20_000), rng.uniform(0.0, 1.0, (20_000, 2)))
    local = eng.collision_results(0)
    eng.exchange_tally()
    summed = eng.collision_results(0)
    q.put((rank, local, summed))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_exchange_sums_the_collision_tallies():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 17) % 1000
    procs = [ctx.Process(target=_two_gpu_collisions_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    total = res[0][1] + res[1][1]
    for _, _, summed in res:
        np.testing.assert_allclose(summed, total, rtol=1e-13, atol=1e-15 * np.abs(total).max())
