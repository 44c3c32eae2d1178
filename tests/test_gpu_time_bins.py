"""Time filter: track-length scores split between the time bins each flight spans (pumitally_set_time_bins).
Time bin j of a timed move must be the tally of the flights' pieces that lie in bin j, and the move must move the
particles exactly as a plain or scored move does."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT, assert_flux_close, box_case
from oracle.oracle import OraclePumiTally
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_scores import _bins, assert_same_particles, assert_scores_equal, engine, responses
from time_bins_ref import edge_crossings, reference_time_tally, time_pieces, time_workload

pytestmark = pytest.mark.gpu

EDGES = np.linspace(0.0, 4.0, 9)


def _move_timed(eng, o, d, f, w, times, speeds, r=None, bins=None):
    f1 = f.copy()
    eng.MoveToNextLocationTimed(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy(), times, speeds, r, bins)
    assert not f1.any(), "flying[] must be zeroed on return"


@pytest.mark.parametrize("nscores", [1, 3])
@pytest.mark.parametrize("variant", [-1, 0, 8, 16, 24])
def test_timed_move_matches_the_cut_flights(variant, nscores):
    cells = (6, 6, 5)
    coords, t2v, wl = box_case(cells, 12_000, mean_length=2.0)
    rng = np.random.default_rng(10 * nscores + variant)
    eng = engine(coords, t2v, wl.n, variant)
    eng.set_scores(nscores)
    eng.set_time_bins(EDGES)
    assert eng.time_bins == len(EDGES) - 1 == eng.get_option("time_bins")
    twin = engine(coords, t2v, wl.n, variant)  # the plain (one score) or scored move of the same inputs
    twin.set_scores(nscores)
    init = wl.initial_positions()
    for e in (eng, twin):
        e.CopyInitialPosition(init.reshape(-1).copy())
    want = np.zeros((len(EDGES) - 1, nscores, len(t2v)))
    crossings = []
    for step in range(2):
        o, d, f, w = wl.next_step()
        r = responses(rng, wl.n, nscores)
        times, speeds = time_workload(rng, o, d, 6.0, EDGES)
        _move_timed(eng, o, d, f, w, times, speeds, r if nscores > 1 else None)
        if nscores > 1:
            twin.MoveToNextLocationScored(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy(), r)
        else:
            twin.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
        alive = f == 1
        want += reference_time_tally(coords, t2v, o, twin.positions, times, speeds, EDGES, alive, w,
                                     r if nscores > 1 else np.ones((wl.n, 1)))
        crossings.append(edge_crossings(o, d, times, speeds, EDGES, alive)[alive])
        assert_same_particles(eng, twin, f"variant {variant} step {step}")
    ft = eng.flux_time
    assert ft.shape == (len(EDGES) - 1, 1, nscores, len(t2v))
    for j in range(len(EDGES) - 1):
        for k in range(nscores):
            assert_flux_close(ft[j, 0, k], want[j, k], f"variant {variant} time {j} score {k}")
    cr = np.concatenate(crossings)
    assert (cr >= 1).mean() > 0.4 and (cr >= 2).mean() > 0.05
    if variant in (8, 16, 24):
        plain = engine(coords, t2v, wl.n, variant)
        plain.CopyInitialPosition(init.reshape(-1).copy())
        o, d, f, w = wl.next_step()
        plain.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
        plain_occupancy = plain.get_option("walk_blocks_per_sm")  # (of the last persistent launch in the process)
        times, speeds = time_workload(rng, o, d, 6.0, EDGES)
        _move_timed(eng, o, d, f, w, times, speeds, responses(rng, wl.n, nscores) if nscores > 1 else None)
        assert eng.get_option("walk_blocks_per_sm") == plain_occupancy > 0


@pytest.mark.parametrize("variant", [-1, 0, 8, 16, 24])
def test_one_enclosing_bin_equals_the_scored_move(variant):
    coords, t2v, wl = box_case((6, 6, 5), 10_000, mean_length=2.0)
    nscores = 3
    rng = np.random.default_rng(3 + variant)
    eng, scored = engine(coords, t2v, wl.n, variant), engine(coords, t2v, wl.n, variant)
    for e in (eng, scored):
        e.set_scores(nscores)
    eng.set_time_bins([-1e3, 1e3])
    init = wl.initial_positions()
    for e in (eng, scored):
        e.CopyInitialPosition(init.reshape(-1).copy())
    for _ in range(2):
        o, d, f, w = wl.next_step()
        r = responses(rng, wl.n, nscores)
        times, speeds = time_workload(rng, o, d, 6.0, np.array([0.0, 1.0]))
        _move_timed(eng, o, d, f, w, times, speeds, r)
        scored.MoveToNextLocationScored(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy(), r)
    ft, fs = eng.flux_time, scored.flux_scores
    for k in range(nscores):
        assert_scores_equal(ft[0, 0, k], fs[0, k], f"variant {variant} score {k}")
    assert_same_particles(eng, scored)


@pytest.mark.parametrize("path", ["staged", "direct", "registered", "device"])
def test_bins_times_scores_on_every_upload_path(path):
    import torch

    nbins, nscores, edges = 3, 2, np.array([0.0, 1.0, 2.5, 4.0])
    coords, t2v, wl = box_case((5, 5, 5), 12_000)
    rng = np.random.default_rng(4)
    opts = {"staged": {}, "direct": {"host_path": 0, "chunk": 4096}, "registered": {"host_path": 0, "register_host": 1},
            "device": {}}[path]
    eng = engine(coords, t2v, wl.n, **opts)
    eng.set_time_bins(edges)  # any order
    eng.set_scores(nscores)
    eng.set_score_bins(nbins)
    assert eng.scores == nscores and eng.score_bins == nbins and eng.time_bins == 3
    twin = engine(coords, t2v, wl.n)
    twin.set_scores(nscores)
    twin.set_score_bins(nbins)
    init = wl.initial_positions()
    for e in (eng, twin):
        e.CopyInitialPosition(init.reshape(-1).copy())
    s = torch.cuda.current_stream().cuda_stream
    o_buf, d_buf, w_buf = np.empty(3 * wl.n), np.empty(3 * wl.n), np.empty(wl.n)
    t_buf, v_buf = np.empty(wl.n), np.empty(wl.n)
    r_buf, b_buf, f_buf = np.empty((wl.n, nscores)), np.empty(wl.n, dtype=np.int32), np.empty(wl.n, dtype=np.int8)
    want = np.zeros((len(edges) - 1, nbins, nscores, len(t2v)))
    h2d = 0.0
    for step in range(2):
        o, d, f, w = wl.next_step()
        o_buf[:], d_buf[:], w_buf[:] = o.reshape(-1), d.reshape(-1), w
        t_buf[:], v_buf[:] = time_workload(rng, o, d, 5.0, edges)
        r_buf[:], b_buf[:] = responses(rng, wl.n, nscores), _bins(wl.n, nbins, step)
        if path == "device":
            t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (o_buf, d_buf, f, w_buf, t_buf, v_buf, r_buf, b_buf)]
            eng.move_device_timed(*(x.data_ptr() for x in t), s)
            torch.cuda.synchronize()
        else:
            before = eng.stats()["h2d_bytes"]
            f_buf[:] = f
            eng.MoveToNextLocationTimed(o_buf, d_buf, f_buf, w_buf, t_buf, v_buf, r_buf, b_buf)
            h2d = eng.stats()["h2d_bytes"] - before
        twin.MoveToNextLocationScored(o_buf.copy(), d_buf.copy(), f.copy(), w_buf.copy(), r_buf, b_buf.copy())
        for b in range(nbins):
            alive = (f == 1) & (b_buf == b)
            want[:, b] += reference_time_tally(coords, t2v, o, twin.positions, t_buf, v_buf, edges, alive, w_buf, r_buf)
    if path != "device":  # the times and speeds, the responses and the bins travel too
        assert h2d >= 16.0 * wl.n + 8.0 * nscores * wl.n + 4.0 * wl.n
    ft = eng.flux_time
    assert ft.shape == (len(edges) - 1, nbins, nscores, len(t2v))
    for j in range(len(edges) - 1):
        for b in range(nbins):
            for k in range(nscores):
                assert_flux_close(ft[j, b, k], want[j, b, k], f"{path} time {j} bin {b} score {k}")
    np.testing.assert_array_equal(eng.elem_ids, twin.elem_ids)
    np.testing.assert_array_equal(eng.positions, twin.positions)


def test_accessors_normalisation_reset_and_vtk(tmp_path):
    import torch
    from vtk_reader import read_vtu_cell_data

    nbins, nscores, nt = 2, 2, 3
    coords, t2v, wl = box_case((4, 4, 4), 5000)
    E = len(t2v)
    rng = np.random.default_rng(9)
    eng = engine(coords, t2v, wl.n)
    eng.set_score_bins(nbins)
    eng.set_scores(nscores)
    edges = np.array([0.0, 1.0, 2.0, 3.0])
    eng.set_time_bins(edges)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    times, speeds = time_workload(rng, o, d, 4.0, edges)
    _move_timed(eng, o, d, f, w, times, speeds, responses(rng, wl.n, nscores), _bins(wl.n, nbins, 0))
    ft = eng.flux_time
    assert ft.shape == (nt, nbins, nscores, E) and ft[1:].any() and ft[:, 1:, 1:].any()
    np.testing.assert_array_equal(eng.flux, ft[0, 0, 0])  # n = E: time 0, bin 0, score 0
    for wrong in (np.empty(nbins * nscores * E), np.empty(nt * E)):
        assert eng._L.pumitally_get_flux(eng._h, wrong.ctypes.data_as(C.POINTER(C.c_double)), wrong.size) != 0
        assert eng._L.pumitally_get_normalized_flux(eng._h, wrong.ctypes.data_as(C.POINTER(C.c_double)), None,
                                                    wrong.size) != 0
    d_out = torch.empty(nt * nbins * nscores * E, dtype=torch.float64, device="cuda")
    eng.get_flux_device(d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(d_out.cpu().numpy().reshape(nt, nbins, nscores, E), ft)
    for mode, value in ((0, 1.0), (1, 1.0), (2, 123.0), (3, 1.0)):  # no division by the bin width
        eng.set_source_normalization(mode, value)
        nf, vol = eng.normalized_flux_time()
        per = eng.source_normalization()
        if mode == 3:
            np.testing.assert_allclose(per, w[f == 1].sum(), rtol=1e-12)
        np.testing.assert_allclose(nf, ft / vol / per, rtol=1e-14)
        f0, v0 = eng.normalized_flux()
        np.testing.assert_array_equal(f0, nf[0, 0, 0])
    eng.set_source_normalization(0)
    nf, vol = eng.normalized_flux_time()
    out = str(tmp_path / "timed.vtk")
    eng.WriteTallyResults(out)
    cells = read_vtu_cell_data(os.path.join(out, "pieces", "piece_0.vtu"))
    untimed = nf.sum(axis=0)  # [bin][score][element]
    np.testing.assert_allclose(cells["flux"], untimed[:, 0].sum(axis=0), rtol=1e-13)
    for k in range(nscores):
        name = "flux" if k == 0 else f"score{k}"
        if k > 0:
            np.testing.assert_allclose(cells[name], untimed[:, k].sum(axis=0), rtol=1e-13)
        for b in range(nbins):
            np.testing.assert_allclose(cells[f"{name}_bin{b}"], untimed[b, k], rtol=1e-13)
        for j in range(nt):
            np.testing.assert_allclose(cells[f"{name}_t{j}"], nf[j, :, k].sum(axis=0), rtol=1e-13)
            for b in range(nbins):
                np.testing.assert_array_equal(cells[f"{name}_t{j}_bin{b}"], nf[j, b, k])
    assert f"flux_t{nt}" not in cells and f"score{nscores}" not in cells
    eng.reset_tally()
    assert not eng.flux_time.any()
    eng.set_time_bins(None)  # the filter removed: back to the scored layout
    assert eng.time_bins == 0 and eng.flux_time.shape == (1, nbins, nscores, E)


def test_refusals_touch_nothing():
    import torch

    coords, t2v, wl = box_case((4, 4, 4), 2000)
    eng = engine(coords, t2v, wl.n)
    for bad in ([0.0], [1.0, 1.0], [2.0, 1.0], [0.0, np.nan], [0.0, np.inf], [-np.inf, 0.0], np.arange(1026.0)):
        with pytest.raises(ValueError):
            eng.set_time_bins(bad)
        assert eng.time_bins == 0
    assert eng._L.pumitally_set_time_bins(eng._h, None, 3) != 0
    eng.set_time_bins(np.arange(1025.0))  # 1024 bins is the limit
    assert eng.time_bins == 1024
    eng.set_time_bins([0.0, 1.0, 2.0])
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    times, speeds = time_workload(np.random.default_rng(1), o, d, 4.0, np.array([0.0, 1.0, 2.0]))
    elems, pos, stats = eng.elem_ids, eng.positions, eng.stats()
    f1 = f.copy()
    with pytest.raises(RuntimeError):
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy())
    np.testing.assert_array_equal(f1, f)  # flying[] untouched
    with pytest.raises(RuntimeError):
        eng.MoveToNextLocationScored(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy(), np.ones(wl.n))
    np.testing.assert_array_equal(f1, f)
    eng.set_score_bins(2)
    with pytest.raises(RuntimeError):
        eng.MoveToNextLocationBinned(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy(), _bins(wl.n, 2, 0))
    np.testing.assert_array_equal(f1, f)
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (o, d, f, w, times, speeds, _bins(wl.n, 2, 0))]
    s = torch.cuda.current_stream().cuda_stream
    with pytest.raises(RuntimeError):
        eng.move_device(*(x.data_ptr() for x in t[:4]), s)
    with pytest.raises(RuntimeError):
        eng.move_device_binned(*(x.data_ptr() for x in t[:4]), t[6].data_ptr(), s)
    with pytest.raises(RuntimeError):
        eng.move_device_scored(*(x.data_ptr() for x in t[:4]), t[4].data_ptr(), None, s)
    with pytest.raises(RuntimeError):  # NULL speeds
        eng.move_device_timed(*(x.data_ptr() for x in t[:5]), None, None, None, s)
    eng.set_scores(2)
    with pytest.raises(RuntimeError):  # NULL responses with two scores
        eng.MoveToNextLocationTimed(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy(), times, speeds)
    np.testing.assert_array_equal(f1, f)
    eng.set_time_bins(None)
    eng.set_scores(1)
    with pytest.raises(RuntimeError):  # a timed move without time bins
        eng.MoveToNextLocationTimed(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy(), times, speeds)
    with pytest.raises(RuntimeError):
        eng.move_device_timed(*(x.data_ptr() for x in t[:6]), None, None, s)
    np.testing.assert_array_equal(f1, f)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(eng.elem_ids, elems)
    np.testing.assert_array_equal(eng.positions, pos)
    assert eng.stats()["segments"] == stats["segments"] and not eng.flux_time.any()


def test_time_bins_refused_after_comm_init():
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
        eng.set_time_bins([0.0, 1.0])
    assert eng.time_bins == 0
    torch.cuda.synchronize()


def test_non_finite_times_and_speeds_are_lost_flights():
    coords, t2v, wl = box_case((6, 6, 5), 4000)
    rng = np.random.default_rng(2)
    eng, plain = engine(coords, t2v, wl.n), engine(coords, t2v, wl.n)
    eng.set_time_bins(EDGES)
    init = wl.initial_positions()
    for e in (eng, plain):
        e.CopyInitialPosition(init.reshape(-1).copy())
    o, d, f, w = wl.next_step()
    f[:] = 1
    times, speeds = time_workload(rng, o, d, 6.0, EDGES)
    bad = np.arange(10, 70)
    times[bad[:15]] = np.nan
    times[bad[15:30]] = np.inf
    speeds[bad[30:45]] = 0.0
    speeds[bad[45:]] = -np.inf
    _move_timed(eng, o, d, f, w, times, speeds)
    wbad = w.copy()
    wbad[bad] = np.nan  # a plain engine treats a non-finite weight exactly so: zero-length flight, counted as lost
    plain.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), wbad)
    assert np.isfinite(eng.flux_time).all() and np.isfinite(eng.positions).all()
    assert_same_particles(eng, plain)
    assert eng.stats()["lost"] == len(bad)
    ok = np.ones(wl.n, dtype=bool)
    ok[bad] = False
    want = reference_time_tally(coords, t2v, o, plain.positions, times, speeds, EDGES, ok, w, np.ones((wl.n, 1)))
    ft = eng.flux_time
    for j in range(len(EDGES) - 1):
        assert_flux_close(ft[j, 0, 0], want[j, 0], f"time {j}")


def test_cxx_program_with_time_bins(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SetTimeBins + MoveToNextLocationTimed next to the reference class."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "time_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "time_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "TIME_OK" in out, out


def test_config_c2_full_size_time_bins_on_the_default_kernel():
    """BASELINE configs[1] (998,250 tets, 10 M particles), device-resident, default kernel: 4 time bins x 2 scores
    against the per-particle oracle run once per time bin on the cut flights, and against a plain engine."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n, nscores = cfg["particles"], 2
    edges = np.array([0.0, 1.0, 2.0, 3.0, 4.0])
    wl = SyntheticWorkload(box=tuple(float(c) for c in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    eng = PumiTally.from_arrays(coords, t2v, n)
    eng.set_scores(nscores)
    eng.set_time_bins(edges)
    plain = PumiTally.from_arrays(coords, t2v, n)
    s = torch.cuda.current_stream().cuda_stream
    init = wl.initial_positions().contiguous()
    for e in (eng, plain):
        e.copy_initial_position_device(init.data_ptr(), s)
    torch.cuda.synchronize()
    start_xyz, start_elem = eng.positions, eng.elem_ids
    o, d, f, w = (x.contiguous() for x in wl.next_step())
    g = torch.Generator(device="cuda").manual_seed(5)
    r = (torch.rand((n, nscores), dtype=torch.float64, device="cuda", generator=g) * 2.0).contiguous()
    r[:, 0] = 1.0
    on, dn = o.cpu().numpy().reshape(-1, 3), d.cpu().numpy().reshape(-1, 3)
    times, speeds = time_workload(np.random.default_rng(6), on, dn, 10.0, edges)
    tt, vt = torch.from_numpy(times).cuda(), torch.from_numpy(speeds).cuda()
    eng.move_device_timed(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), tt.data_ptr(), vt.data_ptr(),
                          r.data_ptr(), None, s)
    plain.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
    torch.cuda.synchronize()
    assert eng.get_option("variant") == plain.get_option("variant")
    assert_same_particles(eng, plain, "c2")
    ft = eng.flux_time[:, 0]
    fn, wn, rn = f.cpu().numpy(), w.cpu().numpy(), r.cpu().numpy()
    end = eng.positions
    # conservation: score 0 (r = 1) summed over the time bins is the plain tally of the part inside [T_0, T_n)
    length = np.linalg.norm(end - on, axis=1)
    alive = fn == 1
    t1 = times + length / speeds
    inside = alive & (times >= edges[0]) & (t1 <= edges[-1])
    assert inside.mean() > 0.05
    for j, (a, b, ids) in enumerate(time_pieces(on, end, times, speeds, edges, alive)):
        orc = OraclePumiTally(coords, t2v, n)
        orc.set_state(start_xyz, start_elem)
        fo = np.zeros(n, dtype=np.int8)
        fo[ids] = 1
        oo, dd = start_xyz.copy(), start_xyz.copy()
        oo[ids], dd[ids] = a, b
        for k in range(nscores):
            if k > 0:
                orc.reset_flux()
                orc.set_state(start_xyz, start_elem)
            orc.MoveToNextLocation(oo.reshape(-1).copy(), dd.reshape(-1).copy(), fo.copy(), wn * rn[:, k])
            assert_flux_close(ft[j, k], orc.flux, f"c2 time {j} score {k}")
    # a plain engine fed only the flights that lie wholly inside [T_0, T_n) tallies what their time bins sum to
    whole = PumiTally.from_arrays(coords, t2v, n)
    whole.copy_initial_position_device(init.data_ptr(), s)
    fw = torch.from_numpy(inside.astype(np.int8)).cuda()
    whole.move_device(o.data_ptr(), d.data_ptr(), fw.data_ptr(), w.data_ptr(), s)
    part = PumiTally.from_arrays(coords, t2v, n)
    part.set_time_bins(edges)
    part.copy_initial_position_device(init.data_ptr(), s)
    part.move_device_timed(o.data_ptr(), d.data_ptr(), fw.data_ptr(), w.data_ptr(), tt.data_ptr(), vt.data_ptr(),
                           None, None, s)
    torch.cuda.synchronize()
    assert_flux_close(part.flux_time[:, 0, 0].sum(axis=0), whole.flux, "c2 conservation")


def _two_gpu_time_worker(rank, world, port, q):
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
    eng.set_time_bins(EDGES)  # before comm_init: the exchange buffers are sized for every time bin
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
    flux = eng.flux_time
    if rank == 0:
        q.put(flux)
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_time_bins_exchange_equals_single_gpu():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 7) % 1000
    procs = [ctx.Process(target=_two_gpu_time_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    flux2 = q.get(timeout=180)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    n_total, nbins, nscores = 30_000, 2, 2
    coords, t2v, wl = box_case((7, 7, 7), n_total, mean_length=2.0)
    one = PumiTally.from_spec("box:7,7,7", n_total)
    one.set_score_bins(nbins)
    one.set_scores(nscores)
    one.set_time_bins(EDGES)
    one.CopyInitialPosition(wl.initial_positions().reshape(-1))
    for k in range(2):
        o, d, f, w = wl.next_step()
        rng = np.random.default_rng(k)
        r = rng.uniform(0.0, 2.0, (n_total, nscores))
        t = rng.uniform(-1.0, 5.0, n_total)
        v = rng.uniform(0.5, 4.0, n_total)
        one.MoveToNextLocationTimed(o.reshape(-1), d.reshape(-1), f, w, t, v, r, _bins(n_total, nbins, k))
    ft = one.flux_time
    for j in range(len(EDGES) - 1):
        for b in range(nbins):
            for k in range(nscores):
                assert_flux_close(flux2[j, b, k], ft[j, b, k], f"2-GPU time {j} bin {b} score {k} vs 1 GPU")
