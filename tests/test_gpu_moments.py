"""Linear flux moments (pumitally_set_moments): every move also tallies the first spatial moment of each score in
each element.  The moments must match an exact clip-and-sum reference, and apart from them a move must do exactly
what the same move does without moments."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT, box_case
from moments_ref import assert_moments_close, reference_moments, tet_geometry
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_scores import _bins, assert_same_particles, assert_scores_equal, engine, responses
from time_bins_ref import time_pieces, time_workload

pytestmark = pytest.mark.gpu

EDGES = np.linspace(0.0, 4.0, 9)
CUT = 1e-12  # times the box: where a piece starts or ends is known to rounding only (tests/moments_ref.py)


def _move(eng, kind, o, d, f, w, r=None, times=None, speeds=None, bins=None):
    f1 = f.copy()
    args = (o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy())
    if kind == "timed":
        eng.MoveToNextLocationTimed(*args, times, speeds, r, bins)
    elif kind == "scored":
        eng.MoveToNextLocationScored(*args, r, bins)
    elif kind == "binned":
        eng.MoveToNextLocationBinned(*args, bins)
    else:
        eng.MoveToNextLocation(*args)
    assert not f1.any(), "flying[] must be zeroed on return"


def _configure(eng, nscores, edges=None, moments=0, nbins=1):
    if moments:
        eng.set_moments(moments)
    eng.set_scores(nscores)
    if nbins > 1:
        eng.set_score_bins(nbins)
    if edges is not None:
        eng.set_time_bins(edges)


@pytest.mark.parametrize("timed", [False, True], ids=["untimed", "timed"])
@pytest.mark.parametrize("nscores", [1, 3])
@pytest.mark.parametrize("variant", [-1, 0, 8, 16, 24])
def test_moment_move_matches_the_exact_reference(variant, nscores, timed):
    coords, t2v, wl = box_case((6, 6, 5), 12_000, mean_length=2.0)
    rng = np.random.default_rng(10 * nscores + variant + (100 if timed else 0))
    edges = EDGES if timed else None
    kind = "timed" if timed else ("scored" if nscores > 1 else "plain")
    eng, twin = engine(coords, t2v, wl.n, variant), engine(coords, t2v, wl.n, variant)
    _configure(eng, nscores, edges, moments=1)
    _configure(twin, nscores, edges)
    assert eng.moments == 1 == eng.get_option("moments") and twin.moments == 0
    _, diam, _, _ = tet_geometry(coords, t2v)
    init = wl.initial_positions()
    for e in (eng, twin):
        e.CopyInitialPosition(init.reshape(-1).copy())
    nt = len(EDGES) - 1 if timed else 1
    want1 = np.zeros((nt, nscores, len(t2v), 3))
    absum, absw = np.zeros((nt, nscores, len(t2v))), np.zeros((nt, nscores, len(t2v)))
    for step in range(2):
        o, d, f, w = wl.next_step()
        r = responses(rng, wl.n, nscores) if nscores > 1 else None
        times, speeds = time_workload(rng, o, d, 6.0, EDGES) if timed else (None, None)
        _move(eng, kind, o, d, f, w, r, times, speeds)
        occ = eng.get_option("walk_blocks_per_sm")  # (of the last persistent launch in the process)
        _move(twin, kind, o, d, f, w, r, times, speeds)
        assert occ == twin.get_option("walk_blocks_per_sm")
        assert_same_particles(eng, twin, f"variant {variant} step {step}")
        _, a1, ab, aw = reference_moments(coords, t2v, o, eng.positions, f == 1, w,
                                          np.ones((wl.n, 1)) if r is None else r, edges, times, speeds)
        want1, absum, absw = want1 + a1, absum + ab, absw + aw
    m0, m0_twin = eng.flux_time, twin.flux_time
    for j in range(nt):
        for k in range(nscores):
            assert_scores_equal(m0[j, 0, k], m0_twin[j, 0, k], f"variant {variant} time {j} score {k}")
    m1 = eng.flux_moments()
    assert m1.shape == (nt, 1, nscores, len(t2v), 3)
    assert_moments_close(m1[:, 0], want1, absum, diam, f"variant {variant}", cut=CUT * 6.0, abs_w=absw)
    assert np.abs(want1).max() > 0


@pytest.mark.parametrize("kind", ["plain", "binned"])
def test_plain_and_binned_moves_are_the_scored_move_with_unit_responses(kind):
    coords, t2v, wl = box_case((6, 6, 5), 10_000, mean_length=2.0)
    nbins = 3 if kind == "binned" else 1
    a, b = engine(coords, t2v, wl.n), engine(coords, t2v, wl.n)
    for e in (a, b):
        _configure(e, 1, moments=1, nbins=nbins)
    init = wl.initial_positions()
    for e in (a, b):
        e.CopyInitialPosition(init.reshape(-1).copy())
    for step in range(2):
        o, d, f, w = wl.next_step()
        bins = _bins(wl.n, nbins, step) if kind == "binned" else None
        _move(a, kind, o, d, f, w, bins=bins)
        _move(b, "scored", o, d, f, w, r=np.ones(wl.n), bins=bins)
    assert_same_particles(a, b)
    ma, mb = a.flux_moments(), b.flux_moments()
    for q in range(nbins):
        assert_scores_equal(a.flux_time[0, q, 0], b.flux_time[0, q, 0], f"{kind} bin {q}")
        for c in range(3):
            assert_scores_equal(ma[0, q, 0, :, c], mb[0, q, 0, :, c], f"{kind} bin {q} component {c}")


@pytest.mark.parametrize("path", ["staged", "direct", "registered", "device"])
def test_bins_scores_time_bins_and_moments_on_every_upload_path(path):
    import torch

    nbins, nscores, edges = 3, 2, np.array([0.0, 1.0, 2.5, 4.0])
    coords, t2v, wl = box_case((5, 5, 5), 12_000)
    rng = np.random.default_rng(4)
    opts = {"staged": {}, "direct": {"host_path": 0, "chunk": 4096}, "registered": {"host_path": 0, "register_host": 1},
            "device": {}}[path]
    eng, twin = engine(coords, t2v, wl.n, **opts), engine(coords, t2v, wl.n)
    eng.set_time_bins(edges)  # any order
    eng.set_moments(1)
    eng.set_scores(nscores)
    eng.set_score_bins(nbins)
    _configure(twin, nscores, edges, nbins=nbins)
    assert eng.moments == 1 and eng.scores == nscores and eng.score_bins == nbins and eng.time_bins == 3
    _, diam, _, _ = tet_geometry(coords, t2v)
    init = wl.initial_positions()
    for e in (eng, twin):
        e.CopyInitialPosition(init.reshape(-1).copy())
    s = torch.cuda.current_stream().cuda_stream
    nt = len(edges) - 1
    want1 = np.zeros((nt, nbins, nscores, len(t2v), 3))
    absum, absw = np.zeros((nt, nbins, nscores, len(t2v))), np.zeros((nt, nbins, nscores, len(t2v)))
    # the caller's arrays stay alive and are reused for every move (what option register_host asks of the caller)
    o_buf, d_buf, w_buf = np.empty(3 * wl.n), np.empty(3 * wl.n), np.empty(wl.n)
    t_buf, v_buf = np.empty(wl.n), np.empty(wl.n)
    r_buf, b_buf, f_buf = np.empty((wl.n, nscores)), np.empty(wl.n, dtype=np.int32), np.empty(wl.n, dtype=np.int8)
    for step in range(2):
        o, d, f, w = wl.next_step()
        o_buf[:], d_buf[:], w_buf[:] = o.reshape(-1), d.reshape(-1), w
        t_buf[:], v_buf[:] = time_workload(rng, o, d, 5.0, edges)
        r_buf[:], b_buf[:] = responses(rng, wl.n, nscores), _bins(wl.n, nbins, step)
        r, times, speeds, bins = r_buf, t_buf, v_buf, b_buf
        if path == "device":
            dev = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (o_buf, d_buf, f, w_buf, t_buf, v_buf, r_buf,
                                                                              b_buf)]
            eng.move_device_timed(*(x.data_ptr() for x in dev), s)
            torch.cuda.synchronize()
        else:
            f_buf[:] = f
            eng.MoveToNextLocationTimed(o_buf, d_buf, f_buf, w_buf, t_buf, v_buf, r_buf, b_buf)
            assert not f_buf.any()
        _move(twin, "timed", o, d, f, w, r, times, speeds, bins)
        assert_same_particles(eng, twin, f"{path} step {step}")
        for q in range(nbins):
            _, a1, ab, aw = reference_moments(coords, t2v, o, eng.positions, (f == 1) & (bins == q), w, r, edges, times,
                                              speeds)
            want1[:, q] += a1
            absum[:, q] += ab
            absw[:, q] += aw
    m0, m0_twin = eng.flux_time, twin.flux_time
    for idx in np.ndindex(nt, nbins, nscores):
        assert_scores_equal(m0[idx], m0_twin[idx], f"{path} {idx}")
    m1 = eng.flux_moments()
    for q in range(nbins):
        assert_moments_close(m1[:, q], want1[:, q], absum[:, q], diam, f"{path} bin {q}", cut=CUT * 5.0,
                             abs_w=absw[:, q])


def test_accessors_normalisation_reset_and_vtk(tmp_path):
    import torch
    from vtk_reader import read_vtu_cell_data

    nbins, nscores, nt = 2, 2, 3
    coords, t2v, wl = box_case((4, 4, 4), 5000)
    E = len(t2v)
    rng = np.random.default_rng(9)
    eng, twin = engine(coords, t2v, wl.n), engine(coords, t2v, wl.n)
    edges = np.array([0.0, 1.0, 2.0, 3.0])
    _configure(eng, nscores, edges, moments=1, nbins=nbins)
    _configure(twin, nscores, edges, nbins=nbins)
    for e in (eng, twin):
        e.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    times, speeds = time_workload(rng, o, d, 4.0, edges)
    r = responses(rng, wl.n, nscores)
    for e in (eng, twin):
        _move(e, "timed", o, d, f, w, r, times, speeds, _bins(wl.n, nbins, 0))
    ft = eng.flux_time
    m1, g = eng.flux_moments(), eng.flux_gradient()
    assert m1.shape == g.shape == (nt, nbins, nscores, E, 3) and np.isfinite(g).all() and g.any()
    # n = 3E: time 0, bin 0, score 0; anything else but the full size is refused
    first = np.empty(3 * E)
    assert eng._L.pumitally_get_flux_moments(eng._h, first.ctypes.data_as(C.POINTER(C.c_double)), first.size) == 0
    np.testing.assert_array_equal(first.reshape(E, 3), m1[0, 0, 0])
    for wrong in (np.empty(E), np.empty(3 * nt * E)):
        for fn in (eng._L.pumitally_get_flux_moments, eng._L.pumitally_get_flux_gradient):
            assert fn(eng._h, wrong.ctypes.data_as(C.POINTER(C.c_double)), wrong.size) != 0
    # the flux accessors return what they return without moments
    for idx in np.ndindex(nt, nbins, nscores):
        assert_scores_equal(ft[idx], twin.flux_time[idx], str(idx))
    d_out = torch.empty(nt * nbins * nscores * E, dtype=torch.float64, device="cuda")
    eng.get_flux_device(d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(d_out.cpu().numpy().reshape(nt, nbins, nscores, E), ft)
    # the gradient: M_e^-1 m1, divided by the source normalisation
    cen, _, _, _ = tet_geometry(coords, t2v)
    v = np.asarray(coords)[np.asarray(t2v)] - cen[:, None, :]
    vol = np.abs(np.einsum("ij,ij->i", v[:, 1] - v[:, 0], np.cross(v[:, 2] - v[:, 0], v[:, 3] - v[:, 0]))) / 6.0
    M = vol[:, None, None] / 20.0 * np.einsum("eqa,eqb->eab", v, v)
    for mode, value in ((0, 1.0), (1, 1.0), (2, 123.0), (3, 1.0)):
        eng.set_source_normalization(mode, value)
        per = eng.source_normalization()
        gn = eng.flux_gradient()
        np.testing.assert_allclose(gn, np.linalg.solve(M, m1[..., None])[..., 0] / per, rtol=1e-9,
                                   atol=1e-12 * np.abs(gn).max())
        nf, vol_ = eng.normalized_flux_time()
        tw, _ = twin.normalized_flux_time() if mode == 0 else (None, None)
        if tw is not None:
            np.testing.assert_allclose(nf, tw, rtol=1e-12, atol=1e-15 * np.abs(tw).max())
    eng.set_source_normalization(0)
    g = eng.flux_gradient()
    nf, _ = eng.normalized_flux_time()
    out, out_twin = str(tmp_path / "moments.vtk"), str(tmp_path / "plain.vtk")
    eng.WriteTallyResults(out)
    twin.WriteTallyResults(out_twin)
    cells = read_vtu_cell_data(os.path.join(out, "pieces", "piece_0.vtu"))
    cells_twin = read_vtu_cell_data(os.path.join(out_twin, "pieces", "piece_0.vtu"))
    assert set(cells) == set(cells_twin) | {n + "_grad" for n in cells_twin if n.startswith(("flux", "score"))}
    for name in cells_twin:  # the existing arrays, up to the order of the reductions
        np.testing.assert_allclose(cells[name], cells_twin[name], rtol=1e-12, atol=1e-15 * np.abs(cells_twin[name]).max())
    untimed = g.sum(axis=0)  # [bin][score][element][3]: the gradient of a sum is the sum of the gradients
    for k in range(nscores):
        name = "flux" if k == 0 else f"score{k}"
        np.testing.assert_allclose(cells[f"{name}_grad"].reshape(E, 3), untimed[:, k].sum(axis=0), rtol=1e-12)
        for b in range(nbins):
            np.testing.assert_allclose(cells[f"{name}_bin{b}_grad"].reshape(E, 3), untimed[b, k], rtol=1e-12)
        for j in range(nt):
            np.testing.assert_allclose(cells[f"{name}_t{j}_grad"].reshape(E, 3), g[j, :, k].sum(axis=0), rtol=1e-12)
            for b in range(nbins):
                np.testing.assert_array_equal(cells[f"{name}_t{j}_bin{b}_grad"].reshape(E, 3), g[j, b, k])
    head = open(os.path.join(out, "pieces.pvtu")).read()
    assert 'Name="flux_grad" NumberOfComponents="3"' in head and 'Name="flux" NumberOfComponents="1"' in head
    eng.reset_tally()
    assert not eng.flux_time.any() and not eng.flux_moments().any()
    eng.set_moments(0)  # back to the layout without moments
    assert eng.moments == 0 and eng.flux_time.shape == (nt, nbins, nscores, E)
    with pytest.raises(RuntimeError):
        eng.flux_moments()


def test_refusals_touch_nothing():
    coords, t2v, wl = box_case((4, 4, 4), 2000)
    eng = engine(coords, t2v, wl.n)
    eng.set_moments(1)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    _move(eng, "plain", o, d, f, w)
    m0, m1 = eng.flux.copy(), eng.flux_moments()
    for bad in (-1, 2, 7):
        with pytest.raises(ValueError):
            eng.set_moments(bad)
        assert eng.moments == 1
    np.testing.assert_array_equal(eng.flux, m0)
    np.testing.assert_array_equal(eng.flux_moments(), m1)
    # the refusal rules of scores and time bins are unchanged with moments
    eng.set_scores(2)
    f1 = f.copy()
    with pytest.raises(RuntimeError):
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy())
    assert (f1 == f).all()
    eng.set_scores(1)
    eng.set_time_bins([0.0, 1.0])
    with pytest.raises(RuntimeError):
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy())
    assert (f1 == f).all() and eng.moments == 1
    plain = engine(coords, t2v, wl.n)
    with pytest.raises(RuntimeError):
        plain.flux_moments()
    with pytest.raises(RuntimeError):
        plain.flux_gradient()


def test_moments_refused_after_comm_init():
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
        eng.set_moments(1)
    assert eng.moments == 0
    torch.cuda.synchronize()


def test_non_finite_inputs_are_lost_flights_that_add_nothing():
    coords, t2v, wl = box_case((6, 6, 5), 4000)
    eng, ref = engine(coords, t2v, wl.n), engine(coords, t2v, wl.n)
    for e in (eng, ref):
        e.set_moments(1)
    init = wl.initial_positions()
    for e in (eng, ref):
        e.CopyInitialPosition(init.reshape(-1).copy())
    o, d, f, w = wl.next_step()
    f[:] = 1
    bad = np.arange(10, 70)
    wb, db = w.copy(), d.copy()
    wb[bad[:20]] = np.nan
    db[bad[20:40], 0] = np.inf
    wb[bad[40:]] = -np.inf
    _move(eng, "plain", o, db, f, wb)
    fr = f.copy()
    fr[bad] = 0
    _move(ref, "plain", o, d, fr, w)  # the good flights only
    assert eng.stats()["lost"] == len(bad)
    m1, g = eng.flux_moments(), eng.flux_gradient()
    assert np.isfinite(m1).all() and np.isfinite(g).all() and np.isfinite(eng.positions).all()
    np.testing.assert_allclose(m1, ref.flux_moments(), rtol=1e-12, atol=1e-14 * np.abs(m1).max())
    np.testing.assert_allclose(eng.flux, ref.flux, rtol=1e-12, atol=1e-14 * np.abs(ref.flux).max())
    good = np.ones(wl.n, dtype=bool)
    good[bad] = False
    np.testing.assert_array_equal(eng.positions[good], ref.positions[good])
    np.testing.assert_array_equal(eng.positions[bad], o.reshape(-1, 3)[bad])  # relocated to the origin, no further


def test_cxx_program_with_moments(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SetMoments, then the reference class's own MoveToNextLocation."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "moments_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "moments_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "MOMENTS_OK" in out, out


def test_config_c2_full_size_moments_conserve_the_first_moment():
    """BASELINE configs[1] (998,250 tets, 10 M particles), device-resident, default kernel, 2 scores x 4 time bins
    with moments: sum_e (m1_e + (c_e - C) m0_e) = sum_i w_i r_ik l_i (mid_i - C) per score and time bin, and m0 is
    the timed move's without moments."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n, nscores = cfg["particles"], 2
    edges = np.array([0.0, 1.0, 2.0, 3.0, 4.0])
    wl = SyntheticWorkload(box=tuple(float(c) for c in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    eng, twin = PumiTally.from_arrays(coords, t2v, n), PumiTally.from_arrays(coords, t2v, n)
    _configure(eng, nscores, edges, moments=1)
    _configure(twin, nscores, edges)
    s = torch.cuda.current_stream().cuda_stream
    init = wl.initial_positions().contiguous()
    for e in (eng, twin):
        e.copy_initial_position_device(init.data_ptr(), s)
    o, d, f, w = (x.contiguous() for x in wl.next_step())
    g = torch.Generator(device="cuda").manual_seed(5)
    r = (torch.rand((n, nscores), dtype=torch.float64, device="cuda", generator=g) * 2.0).contiguous()
    on, dn = o.cpu().numpy().reshape(-1, 3), d.cpu().numpy().reshape(-1, 3)
    times, speeds = time_workload(np.random.default_rng(6), on, dn, 10.0, edges)
    tt, vt = torch.from_numpy(times).cuda(), torch.from_numpy(speeds).cuda()
    for e in (eng, twin):
        e.move_device_timed(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), tt.data_ptr(), vt.data_ptr(),
                            r.data_ptr(), None, s)
    torch.cuda.synchronize()
    assert eng.get_option("variant") == twin.get_option("variant")
    assert_same_particles(eng, twin, "c2")
    m0, m0_twin = eng.flux_time[:, 0], twin.flux_time[:, 0]
    for j in range(len(edges) - 1):
        for k in range(nscores):
            assert_scores_equal(m0[j, k], m0_twin[j, k], f"c2 time {j} score {k}")
    m1 = eng.flux_moments()[:, 0]
    cen = np.asarray(coords)[np.asarray(t2v)].mean(axis=1)
    C0 = 0.5 * (np.asarray(coords).min(axis=0) + np.asarray(coords).max(axis=0))
    end = eng.positions
    fn, wn, rn = f.cpu().numpy(), w.cpu().numpy(), r.cpu().numpy()
    for j, (a, b, ids) in enumerate(time_pieces(on, end, times, speeds, edges, fn == 1)):
        ell = np.linalg.norm(b - a, axis=1)
        rel = 0.5 * (a + b) - C0
        for k in range(nscores):
            wrl = wn[ids] * rn[ids, k] * ell
            want = (wrl[:, None] * rel).sum(axis=0)
            got = (m1[j, k] + (cen - C0)[:, :] * m0[j, k][:, None]).sum(axis=0)
            scale = (np.abs(wrl)[:, None] * np.abs(rel)).sum(axis=0)
            assert (np.abs(got - want) <= 1e-10 * scale).all(), (j, k, got, want, scale)


def _two_gpu_moments_worker(rank, world, port, q):
    import sys

    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pumiumtally_b200.distributed import broadcast_unique_id, particle_stripe

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    n_total, nbins, nscores = 30_000, 2, 2
    b, e = particle_stripe(n_total, rank, world)
    eng = PumiTally.from_spec("box:7,7,7", e - b, device=rank)
    eng.set_score_bins(nbins)
    eng.set_scores(nscores)
    eng.set_time_bins(EDGES)
    eng.set_moments(1)  # before comm_init: the exchange buffers are sized for the moments
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    wl = SyntheticWorkload(box=(7.0, 7.0, 7.0), num_particles=e - b, mean_length=2.0, id_offset=b)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1))
    for k in range(2):
        o, d, f, w = wl.next_step()
        rng = np.random.default_rng(k)
        r = rng.uniform(0.0, 2.0, (n_total, nscores))[b:e].copy()
        t = rng.uniform(-1.0, 5.0, n_total)[b:e].copy()
        v = rng.uniform(0.5, 4.0, n_total)[b:e].copy()
        eng.MoveToNextLocationTimed(o.reshape(-1), d.reshape(-1), f, w, t, v, r, _bins(n_total, nbins, k)[b:e].copy())
        (eng.allreduce_tally if k == 0 else eng.reduce_tally_to_owners)()
    m1 = eng.flux_moments()
    if rank == 0:
        q.put(m1)
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_moments_exchange_equals_single_gpu():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 11) % 1000
    procs = [ctx.Process(target=_two_gpu_moments_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    m2 = q.get(timeout=180)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    n_total, nbins, nscores = 30_000, 2, 2
    coords, t2v, wl = box_case((7, 7, 7), n_total, mean_length=2.0)
    one = PumiTally.from_spec("box:7,7,7", n_total)
    _configure(one, nscores, EDGES, moments=1, nbins=nbins)
    one.CopyInitialPosition(wl.initial_positions().reshape(-1))
    for k in range(2):
        o, d, f, w = wl.next_step()
        rng = np.random.default_rng(k)
        r = rng.uniform(0.0, 2.0, (n_total, nscores))
        t = rng.uniform(-1.0, 5.0, n_total)
        v = rng.uniform(0.5, 4.0, n_total)
        one.MoveToNextLocationTimed(o.reshape(-1), d.reshape(-1), f, w, t, v, r, _bins(n_total, nbins, k))
    m1 = one.flux_moments()
    np.testing.assert_allclose(m2, m1, rtol=1e-10, atol=1e-12 * np.abs(m1).max())
