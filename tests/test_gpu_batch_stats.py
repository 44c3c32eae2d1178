"""Batch statistics (pumitally_set_batch_statistics, pumitally_end_batch): the per-source results of every batch are
folded on the device into a running mean and variance.  Every check captures what the plain accessors return just
before each end_batch and compares the engine's mean, standard error, relative error, gradient of the mean and
max-relative-error trigger with numpy statistics of those captures."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_moments import _configure, _move
from test_gpu_scores import assert_same_particles, responses
from test_gpu_tally_collisions import CASES, _geometry
from time_bins_ref import time_workload

pytestmark = pytest.mark.gpu

_dp = C.POINTER(C.c_double)
MODES = {0: 1.0, 1: 1.0, 2: 37.0, 3: 1.0}  # source-normalisation mode -> value


def numpy_stats(x):
    """x [B, ...] -> mean, std(ddof=1) / sqrt(B), relative error (0 where the mean is 0)"""
    m = x.mean(axis=0)
    s = x.std(axis=0, ddof=1) / np.sqrt(len(x))
    return m, s, np.divide(s, np.abs(m), out=np.zeros_like(s), where=m != 0)


def assert_stats(got, want, label):
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-14 * np.abs(want).max(), err_msg=label)


class Batches:
    """An engine of one CASES configuration with the collision estimator on, fed batch by batch on the Kuhn box."""

    def __init__(self, case, mode=0, path="host", n=4000, seed=5, stats=True):
        import torch

        self.nscores, self.nbins, self.edges, self.moments = CASES[case]
        self.c, self.t = kuhn_box(6, 5, 4)
        self.wl = SyntheticWorkload(box=(6.0, 5.0, 4.0), num_particles=n, mean_length=1.0, seed=seed)
        self.eng = PumiTally.from_arrays(self.c, self.t, n)
        self.eng.set_collision_estimator(True)
        if stats:
            self.eng.set_batch_statistics(True)
        _configure(self.eng, self.nscores, self.edges, moments=self.moments, nbins=self.nbins)
        self.eng.set_source_normalization(mode, MODES[mode])
        self.eng.CopyInitialPosition(self.wl.initial_positions().reshape(-1).copy())
        self.rng = np.random.default_rng(seed)
        self.path, self.n, self.torch = path, n, torch

    def kind(self):
        return "timed" if self.edges is not None else "scored" if self.nscores > 1 else \
            "binned" if self.nbins > 1 else "plain"

    def move(self, scale=1.0):
        """One move of the workload (weights times `scale`), then collision events at 40 % of the particles."""
        o, d, f, w = self.wl.next_step()
        w = w * scale
        n, rng, kind = self.n, self.rng, self.kind()
        r = responses(rng, n, self.nscores)
        bins = rng.integers(0, self.nbins, n).astype(np.int32)
        tt = vv = None
        if self.edges is not None:
            tt, vv = time_workload(rng, o, d, 6.0, self.edges)
        if self.path == "host":
            _move(self.eng, kind, o, d, f, w, r, tt, vv, bins)
        else:
            T = lambda a: None if a is None else self.torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
            do, dd, df, dw, dr, db, dt, dv = (T(a) for a in (o.reshape(-1), d.reshape(-1), f, w, r, bins, tt, vv))
            p = lambda a: a.data_ptr()  # noqa: E731
            s = self.torch.cuda.current_stream().cuda_stream
            if kind == "timed":
                self.eng.move_device_timed(p(do), p(dd), p(df), p(dw), p(dt), p(dv), p(dr), p(db), s)
            elif kind == "scored":
                self.eng.move_device_scored(p(do), p(dd), p(df), p(dw), p(dr), p(db), s)
            elif kind == "binned":
                self.eng.move_device_binned(p(do), p(dd), p(df), p(dw), p(db), s)
            else:
                self.eng.move_device(p(do), p(dd), p(df), p(dw), s)
            self.torch.cuda.synchronize()
        collided = (rng.random(n) < 0.4).astype(np.int8)
        times = None if self.edges is None else rng.uniform(-0.5, 4.5, n)
        self.eng.tally_collisions_at_particles(collided, rng.uniform(0.1, 2.0, n) * scale,
                                               rng.uniform(0.0, 2.0, (n, self.nscores)), bins, times)

    def capture(self):
        """What the plain accessors give for the open batch: normalised results of both tallies (and gradients)."""
        e = self.eng
        out = [e.normalized_flux_time()[0], e.collision_results(1)]
        if self.moments:
            out += [e.flux_gradient(), e.collision_results(3)]
        return out


def test_one_batch():
    b = Batches("s3_b3_t_mo", mode=3)
    b.move()
    before = b.capture()
    b.eng.end_batch()
    assert b.eng.batches == 1 == b.eng.get_option("batches")
    np.testing.assert_allclose(b.eng.batch_results(0, 0), before[0], rtol=1e-14, atol=0)
    np.testing.assert_allclose(b.eng.batch_results(1, 0), before[1], rtol=1e-14, atol=0)
    assert not b.eng.flux_time.any() and not b.eng.collision_results(0).any()
    for tally in (0, 1):
        for kind in (1, 2):
            with pytest.raises(RuntimeError):
                b.eng.batch_results(tally, kind)
        with pytest.raises(RuntimeError):
            b.eng.batch_max_rel_err(tally, 0)


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("case", list(CASES))
def test_eight_batches_match_numpy(case, mode, path):
    b = Batches(case, mode=mode, path=path, seed=11 + mode)
    caps = []
    for _ in range(8):
        b.move()
        caps.append(b.capture())
        b.eng.end_batch()
    assert b.eng.batches == 8
    for tally in (0, 1):
        x = np.array([c[tally] for c in caps])
        want = numpy_stats(x)
        for kind in range(3):
            assert_stats(b.eng.batch_results(tally, kind), want[kind], f"{case} mode {mode} {path} tally {tally} kind {kind}")
        if b.moments:
            g = np.array([c[2 + tally] for c in caps]).mean(axis=0)
            np.testing.assert_allclose(b.eng.batch_results(tally, 3), g, rtol=1e-9, atol=1e-12 * np.abs(g).max(),
                                       err_msg=f"{case} gradient {tally}")
        else:
            with pytest.raises(RuntimeError):
                b.eng.batch_results(tally, 3)
        for k in range(b.nscores):  # tally trigger: max relative error of score k over the nonzero means
            m, _, rel = (w[:, :, k] for w in want)
            mx, cnt = b.eng.batch_max_rel_err(tally, k)
            assert cnt == int((m != 0).sum()) > 0
            np.testing.assert_allclose(mx, rel[m != 0].max(), rtol=1e-12, atol=0)
    # n == num_elements: time bin 0, bin 0, score 0
    E = len(b.t)
    first = np.empty(E)
    assert b.eng._L.pumitally_get_batch_results(b.eng._h, 0, 1, first.ctypes.data_as(_dp), E) == 0
    np.testing.assert_array_equal(first, b.eng.batch_results(0, 1)[0, 0, 0])


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mode", [0, 3])
@pytest.mark.parametrize("collision", [False, True], ids=["track", "collision"])
def test_odd_element_count(collision, mode, path):
    """One score, no bins and an odd number of elements: without the collision estimator the folded length L = E is
    odd, so the double2 fold ends in its odd tail; with it the collision tally starts at the odd offset E.  Every
    element is scored in every batch (a flight starts at each centroid), so a result the fold or readout skipped
    would show as a zero mean."""
    import torch

    from pumiumtally_b200.mesh import delaunay_box

    c, t = delaunay_box(60, seed=1)
    E = len(t)
    assert E % 2 == 1
    cen = c[t].mean(axis=1)
    n = E + 1000
    rng = np.random.default_rng(7 + mode)
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_collision_estimator(collision)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(mode, MODES[mode])
    start = np.vstack([cen, rng.uniform(0.05, 0.95, (n - E, 3))])
    eng.CopyInitialPosition(start.reshape(-1).copy())
    caps = []
    for _ in range(6):
        o = np.vstack([cen, eng.positions[E:]])  # the first E re-start at the centroids
        d = rng.uniform(0.0, 1.0, (n, 3))
        f = np.ones(n, dtype=np.int8)
        w = rng.uniform(0.5, 1.5, n)
        if path == "host":
            _move(eng, "plain", o, d, f, w)
        else:
            do, dd, df, dw = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (o.reshape(-1), d.reshape(-1), f, w))
            eng.move_device(do.data_ptr(), dd.data_ptr(), df.data_ptr(), dw.data_ptr(),
                            torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
        cap = [eng.normalized_flux()[0]]
        if collision:
            eng.tally_collisions(cen, rng.uniform(0.5, 1.5, E))
            cap.append(eng.collision_results(1)[0, 0, 0])
        caps.append(cap)
        eng.end_batch()
    for tally in range(len(caps[0])):
        x = np.array([cp[tally] for cp in caps])
        assert (x != 0).all()
        want = numpy_stats(x)
        for kind in range(3):
            got = eng.batch_results(tally, kind)[0, 0, 0]
            assert_stats(got, want[kind], f"tally {tally} kind {kind}")
            assert got[E - 1] != 0 and abs(got[E - 1] - want[kind][E - 1]) <= 1e-12 * abs(want[kind][E - 1])
        mx, cnt = eng.batch_max_rel_err(tally, 0)
        assert cnt == E
        np.testing.assert_allclose(mx, want[2].max(), rtol=1e-12, atol=0)


def test_ill_conditioned_batches():
    """The same flights every batch with weights scaled by 1 + 1e-9 b: the standard error is 1e-9 of the mean, and
    still matches numpy's two-pass result to 1e-6."""
    c, t = kuhn_box(6, 5, 4)
    n = 4000
    wl = SyntheticWorkload(box=(6.0, 5.0, 4.0), num_particles=n, mean_length=1.0, seed=9)
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_batch_statistics(True)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    caps = []
    for k in range(12):
        _move(eng, "plain", o, d, f, w * (1.0 + 1e-9 * k))
        caps.append(eng.normalized_flux()[0])
        eng.end_batch()
    x = np.array(caps)
    m, s, rel = numpy_stats(x)
    nz = m != 0
    assert nz.sum() > 0.5 * len(t) and np.median(s[nz] / m[nz]) < 1e-8
    got = eng.batch_results(0, 1)[0, 0, 0]
    np.testing.assert_allclose(got[nz], s[nz], rtol=1e-6, atol=0)
    np.testing.assert_allclose(eng.batch_results(0, 2)[0, 0, 0][nz], rel[nz], rtol=1e-6, atol=0)


def test_nothing_else_changes(tmp_path):
    from vtk_reader import read_vtu_cell_data

    a, b = Batches("s3_b3_t_mo", seed=4), Batches("s3_b3_t_mo", seed=4, stats=False)
    for step in range(3):
        a.move()
        b.move()
        assert_same_particles(a.eng, b.eng, f"step {step}")
        for what, u, v in (("flux", a.eng.flux_time, b.eng.flux_time),
                           ("collision", a.eng.collision_results(0), b.eng.collision_results(0)),
                           ("moments", a.eng.flux_moments(), b.eng.flux_moments())):
            np.testing.assert_allclose(u, v, rtol=1e-9, atol=1e-11 * np.abs(v).max(), err_msg=f"{what} {step}")
        a.eng.end_batch()
        b.eng.reset_tally()
        sa, sb = a.eng.stats(), b.eng.stats()
        assert {k: sa[k] for k in sa if k != "kernel_ms"} == {k: sb[k] for k in sb if k != "kernel_ms"}
        assert not a.eng.flux_time.any() and not a.eng.collision_results(0).any()
        assert a.eng.get_option("collisions") == 0
    assert a.eng.batches == 3
    # switched off: refused, and the VTK file has exactly the arrays of an engine that never had statistics
    a.eng.set_batch_statistics(False)
    assert not a.eng.batch_statistics and a.eng.batches == 0
    with pytest.raises(RuntimeError):
        a.eng.end_batch()
    with pytest.raises(RuntimeError):
        a.eng.batch_results(0, 0)
    with pytest.raises(RuntimeError):
        a.eng.batch_max_rel_err(0, 0)
    a.move()
    b.move()
    pa, pb = str(tmp_path / "a.vtk"), str(tmp_path / "b.vtk")
    a.eng.WriteTallyResults(pa)
    b.eng.WriteTallyResults(pb)
    ca = read_vtu_cell_data(os.path.join(pa, "pieces", "piece_0.vtu"))
    cb = read_vtu_cell_data(os.path.join(pb, "pieces", "piece_0.vtu"))
    assert list(ca) == list(cb)


def test_refusals_and_resets():
    b = Batches("s1", mode=3)
    eng, L, h = b.eng, b.eng._L, b.eng._h
    E = len(b.t)
    with pytest.raises(ValueError):
        eng.set_batch_statistics(2)
    assert eng.batch_statistics
    with pytest.raises(RuntimeError):  # no batch folded yet
        eng.batch_results(0, 0)
    with pytest.raises(RuntimeError):  # mode 3 before any move: the divisor is 0
        eng.end_batch()
    assert eng.batches == 0
    for _ in range(2):
        b.move()
        eng.end_batch()
    b.move()
    open_batch = eng.flux_time.copy()
    mean = eng.batch_results(0, 0)
    out = np.empty(E + 1)
    refused = [
        lambda: L.pumitally_get_batch_results(h, 0, 0, out.ctypes.data_as(_dp), E + 1),
        lambda: L.pumitally_get_batch_results(h, 0, 3, out.ctypes.data_as(_dp), 3 * E),  # no moments
        lambda: L.pumitally_get_batch_results(h, 0, 4, out.ctypes.data_as(_dp), E),
        lambda: L.pumitally_get_batch_results(h, 2, 0, out.ctypes.data_as(_dp), E),
        lambda: L.pumitally_get_batch_max_rel_err(h, 0, 1, C.byref(C.c_double()), C.byref(C.c_int64())),
        lambda: L.pumitally_get_batch_max_rel_err(h, 0, -1, C.byref(C.c_double()), C.byref(C.c_int64())),
    ]
    for k, call in enumerate(refused):
        assert call() != 0, k
    np.testing.assert_array_equal(eng.flux_time, open_batch)
    np.testing.assert_array_equal(eng.batch_results(0, 0), mean)
    eng.set_collision_estimator(False)  # a configuration change discards the batches (and resets the tally)
    assert eng.batches == 0 and eng.batch_statistics
    with pytest.raises(RuntimeError):
        eng.batch_results(1, 0)
    eng.set_source_normalization(0)
    _move(eng, "plain", *b.wl.next_step())
    eng.end_batch()
    assert eng.batches == 1
    with pytest.raises(RuntimeError):  # tally 1 without the estimator
        eng.batch_results(1, 0)
    eng.set_batch_statistics(True)  # again: discards
    assert eng.batches == 0


def test_refused_after_comm_init():
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
        eng.set_batch_statistics(True)
    assert not eng.batch_statistics
    torch.cuda.synchronize()


def test_vtk_arrays(tmp_path):
    from vtk_reader import read_vtu_cell_data

    b = Batches("s3_b3_t", seed=21)
    nscores, nbins, edges = b.nscores, b.nbins, b.edges
    b.move()
    b.eng.end_batch()
    p1 = str(tmp_path / "one.vtk")
    b.eng.WriteTallyResults(p1)
    one = read_vtu_cell_data(os.path.join(p1, "pieces", "piece_0.vtu"))
    assert any(k.endswith("_mean") for k in one) and not any(k.endswith("_rel_err") for k in one)
    for _ in range(3):
        b.move()
        b.eng.end_batch()
    b.move()  # an open batch: the existing arrays hold it
    path = str(tmp_path / "stats.vtk")
    b.eng.WriteTallyResults(path)
    cells = read_vtu_cell_data(os.path.join(path, "pieces", "piece_0.vtu"))
    twin = Batches("s3_b3_t", seed=21, stats=False)
    twin.move()
    tp = str(tmp_path / "twin.vtk")
    twin.eng.WriteTallyResults(tp)
    names = list(read_vtu_cell_data(os.path.join(tp, "pieces", "piece_0.vtu")))
    assert list(cells)[:len(names)] == names  # the existing arrays first, in their order
    np.testing.assert_allclose(cells["flux_t0_bin0"], b.eng.normalized_flux_time()[0][0, 0, 0], rtol=1e-14)
    for tally, prefix in ((0, ""), (1, "collision_")):
        m, rel = b.eng.batch_results(tally, 0), b.eng.batch_results(tally, 2)

        def close(name, want):
            np.testing.assert_allclose(cells[prefix + name], want, rtol=1e-12, atol=1e-12 * np.abs(want).max(),
                                       err_msg=prefix + name)

        for k in range(nscores):
            name = "flux" if k == 0 else f"score{k}"
            close(name + "_mean", m[:, :, k].sum(axis=(0, 1)))
            assert prefix + name + "_rel_err" not in cells  # a sum over bins and time bins
            for bb in range(nbins):
                close(f"{name}_bin{bb}_mean", m[:, bb, k].sum(axis=0))
                assert f"{prefix}{name}_bin{bb}_rel_err" not in cells  # a sum over time bins
            for j in range(len(edges) - 1):
                close(f"{name}_t{j}_mean", m[j, :, k].sum(axis=0))
                assert f"{prefix}{name}_t{j}_rel_err" not in cells  # a sum over bins
                for bb in range(nbins):
                    close(f"{name}_t{j}_bin{bb}_mean", m[j, bb, k])
                    close(f"{name}_t{j}_bin{bb}_rel_err", rel[j, bb, k])
    # one score, no bins, no time bins: the plain writer's "flux" is one result
    p = Batches("s1", seed=22)
    for _ in range(2):
        p.move()
        p.eng.end_batch()
    pp = str(tmp_path / "plain.vtk")
    p.eng.WriteTallyResults(pp)
    pc = read_vtu_cell_data(os.path.join(pp, "pieces", "piece_0.vtu"))
    stats_names = [k for k in pc if k.endswith(("_mean", "_rel_err"))]
    assert stats_names == ["flux_mean", "flux_rel_err", "collision_flux_mean", "collision_flux_rel_err"]
    np.testing.assert_allclose(pc["flux_rel_err"], p.eng.batch_results(0, 2)[0, 0, 0], rtol=1e-12, atol=0)
    np.testing.assert_allclose(pc["collision_flux_mean"], p.eng.batch_results(1, 0)[0, 0, 0], rtol=1e-12, atol=0)


def test_config_c2_ten_batches():
    """Full-size c2 (998,250 tets, 10 M particles): 10 batches of one device move each, against numpy."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n = cfg["particles"]
    wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    eng = PumiTally.from_arrays(coords, t2v, n)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(3)
    s = torch.cuda.current_stream().cuda_stream
    eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
    caps = []
    for _ in range(10):
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
        torch.cuda.synchronize()
        caps.append(eng.normalized_flux()[0])
        eng.end_batch()
    want = numpy_stats(np.array(caps))
    for kind in range(3):
        assert_stats(eng.batch_results(0, kind)[0, 0, 0], want[kind], f"c2 kind {kind}")
    mx, cnt = eng.batch_max_rel_err()
    m, _, rel = want
    assert cnt == int((m != 0).sum())
    np.testing.assert_allclose(mx, rel[m != 0].max(), rtol=1e-12)


def test_cxx_program_with_batch_statistics(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SetBatchStatistics, EndBatch, GetBatchResults and GetBatchMaxRelErr."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "batch_stats_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "batch_stats_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "BATCH_STATS_OK" in out, out


def _two_gpu_batch_worker(rank, world, port, q):
    import sys

    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pumiumtally_b200.distributed import broadcast_unique_id

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    n = 3000
    c, t = kuhn_box(5, 5, 5)
    eng = PumiTally.from_arrays(c, t, n, device=rank)
    eng.set_scores(2)
    eng.set_score_bins(2)
    eng.set_collision_estimator(True)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(3)
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    wl = SyntheticWorkload(box=(5.0, 5.0, 5.0), num_particles=n, mean_length=1.0, seed=100 + rank)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    rng = np.random.default_rng(rank)
    local, weights = [], []
    for _ in range(5):
        o, d, f, w = wl.next_step()
        w = w * rng.uniform(0.5, 1.5)
        bins = rng.integers(0, 2, n).astype(np.int32)
        _move(eng, "scored", o, d, f, w, responses(rng, n, 2), bins=bins)
        pts = rng.uniform(0.0, 5.0, (2000, 3))
        eng.tally_collisions(pts, rng.uniform(0.5, 1.5, 2000), rng.uniform(0.0, 1.0, (2000, 2)),
                             rng.integers(0, 2, 2000).astype(np.int32))
        local.append((eng.flux_time.copy(), eng.collision_results(0).copy()))
        weights.append(float((w * (f == 1)).sum()))
        eng.end_batch()
    results = [[eng.batch_results(tally, kind) for kind in range(3)] for tally in (0, 1)]
    trig = [eng.batch_max_rel_err(tally, k) for tally in (0, 1) for k in range(2)]
    q.put((rank, local, weights, _geometry(c, t)[1], results, trig))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpus_fold_the_summed_batches():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 53) % 1000
    procs = [ctx.Process(target=_two_gpu_batch_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    vol = res[0][3]
    div = np.array(res[0][2]) + np.array(res[1][2])  # mode 3: the whole batch's first-track weight
    for tally in (0, 1):
        x = np.array([(res[0][1][b][tally] + res[1][1][b][tally]) / vol / div[b] for b in range(5)])
        want = numpy_stats(x)
        for rank in (0, 1):
            for kind in range(3):
                assert_stats(res[rank][4][tally][kind], want[kind], f"rank {rank} tally {tally} kind {kind}")
            for k in range(2):
                m, _, rel = (w[:, :, k] for w in want)
                mx, cnt = res[rank][5][2 * tally + k]
                assert cnt == int((m != 0).sum())
                np.testing.assert_allclose(mx, rel[m != 0].max(), rtol=1e-12)


# Uneven rank shares: share_ = ceil(L / nranks) odd and not a multiple of the record stride, so every rank after the
# first folds from an odd double (the scalar fold) and its max-relative-error window starts inside a record.  On the
# Delaunay mesh below (E = 731 = 5 mod 6) with the collision estimator on:
#   "s2": 2 scores (stride 2), L = 4 E;  3 ranks: share 975, rank 1 holds the end of the track-length tally and the
#         start of the collision tally;  4 ranks: share 731, rank 2 starts exactly at the collision tally.
#   "s1_b2_mo": 1 score, 2 bins, moments (stride 4), L = 16 E;  3 ranks: share 3899, rank 1 holds both tallies.
UNEVEN = {"s2": (2, 1, 0), "s1_b2_mo": (1, 2, 1)}  # nscores, nbins, moments
UNEVEN_N, UNEVEN_BATCHES = 2500, 5


def _uneven_inputs(rank, nscores, nbins):
    """Every rank's initial positions and, per batch (one more than UNEVEN_BATCHES: the last stays open), its move
    and collision events."""
    wl = SyntheticWorkload(box=(1.0, 1.0, 1.0), num_particles=UNEVEN_N, mean_length=0.3, seed=300 + rank)
    rng = np.random.default_rng(rank)
    init, steps = wl.initial_positions().reshape(-1).copy(), []
    for _ in range(UNEVEN_BATCHES + 1):
        o, d, f, w = wl.next_step()
        k = 1500
        steps.append(dict(o=o, d=d, f=f, w=w * rng.uniform(0.5, 1.5), r=responses(rng, UNEVEN_N, nscores),
                          bins=rng.integers(0, nbins, UNEVEN_N).astype(np.int32), pts=rng.uniform(0.0, 1.0, (k, 3)),
                          cw=rng.uniform(0.5, 1.5, k), cr=rng.uniform(0.0, 1.0, (k, nscores)),
                          cb=rng.integers(0, nbins, k).astype(np.int32)))
    return init, steps


def _uneven_engine(c, t, n, nscores, nbins, moments, device=-1):
    eng = PumiTally.from_arrays(c, t, n, device=device)
    _configure(eng, nscores, moments=moments, nbins=nbins)
    eng.set_collision_estimator(True)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(3)
    return eng


def _uneven_step(eng, s, nscores):
    if nscores > 1:
        _move(eng, "scored", s["o"], s["d"], s["f"], s["w"], s["r"], bins=s["bins"])
    else:
        _move(eng, "binned", s["o"], s["d"], s["f"], s["w"], bins=s["bins"])
    eng.tally_collisions(s["pts"], s["cw"], s["cr"], s["cb"])


def _exchanged(eng, moments, pts):
    """What the accessors return after a batch-end exchange (raw results and point values, mode 0)."""
    out = [eng.flux_time, eng.collision_results(0), eng.evaluate(pts)[0]]
    if moments:
        out += [eng.flux_moments(), eng.collision_results(2)]
    return out


def _uneven_worker(rank, world, port, q, case):
    import sys

    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pumiumtally_b200.distributed import broadcast_unique_id
    from pumiumtally_b200.mesh import delaunay_box

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    nscores, nbins, moments = UNEVEN[case]
    c, t = delaunay_box(120, seed=6)
    eng = _uneven_engine(c, t, UNEVEN_N, nscores, nbins, moments, device=rank)
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    init, steps = _uneven_inputs(rank, nscores, nbins)
    eng.CopyInitialPosition(init)
    local, weights = [], []
    for s in steps[:-1]:
        _uneven_step(eng, s, nscores)
        local.append((eng.flux_time.copy(), eng.collision_results(0).copy()))
        weights.append(float((s["w"] * (s["f"] == 1)).sum()))
        eng.end_batch()
    kinds = range(4) if moments else range(3)
    results = [[eng.batch_results(tally, kind) for kind in kinds] for tally in (0, 1)]
    trig = [eng.batch_max_rel_err(tally, k) for tally in (0, 1) for k in range(nscores)]
    _uneven_step(eng, steps[-1], nscores)  # an open batch, exchanged both ways
    eng.set_source_normalization(0)
    pts = np.random.default_rng(99).uniform(0.0, 1.0, (500, 3))
    eng.reduce_tally_to_owners()
    owners = _exchanged(eng, moments, pts)
    eng.allreduce_tally()
    summed = _exchanged(eng, moments, pts)
    q.put((rank, local, weights, results, trig, owners, summed))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("case,world,straddle", [("s2", 3, True), ("s2", 4, False), ("s1_b2_mo", 3, True)],
                         ids=["s2-3ranks", "s2-4ranks", "s1_b2_mo-3ranks"])
def test_uneven_rank_shares(case, world, straddle):
    import torch

    from pumiumtally_b200.mesh import delaunay_box
    from test_gpu_stats_kernels import score_stride

    nscores, nbins, moments = UNEVEN[case]
    c, t = delaunay_box(120, seed=6)
    E = len(t)
    stride = score_stride(nscores) * (4 if moments else 1)
    flux_len = nbins * E * stride
    L = 2 * flux_len
    share = -(-L // world)
    # the layout this test is about
    assert share % 2 == 1 and share % stride != 0
    los = [r * share for r in range(world)]
    if straddle:  # one share holds the end of the track-length tally and the start of the collision tally
        assert any(lo < flux_len < lo + share for lo in los)
    else:  # a share starts exactly at the collision tally
        assert flux_len in los
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 17 * world + len(case)) % 1000
    procs = [ctx.Process(target=_uneven_worker, args=(r, world, port, q, case)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in range(world)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    vol = _geometry(c, t)[1]
    div = np.sum([r[2] for r in res], axis=0)  # mode 3: the whole batch's first-track weight
    # the same particles and events on one GPU
    one = _uneven_engine(c, t, world * UNEVEN_N, nscores, nbins, moments)
    inputs = [_uneven_inputs(r, nscores, nbins) for r in range(world)]
    one.CopyInitialPosition(np.concatenate([i for i, _ in inputs]))
    for b in range(UNEVEN_BATCHES + 1):
        s = {k: np.concatenate([steps[b][k] for _, steps in inputs]) for k in inputs[0][1][b]}
        _uneven_step(one, s, nscores)
        if b < UNEVEN_BATCHES:
            one.end_batch()
    for tally in (0, 1):
        x = np.array([sum(r[1][b][tally] for r in res) / vol / div[b] for b in range(UNEVEN_BATCHES)])
        want = numpy_stats(x)
        for rank in range(world):
            for kind in range(3):
                assert_stats(res[rank][3][tally][kind], want[kind], f"rank {rank} tally {tally} kind {kind}")
                assert_stats(res[rank][3][tally][kind], one.batch_results(tally, kind), f"one GPU {tally} {kind}")
            if moments:
                g = one.batch_results(tally, 3)
                np.testing.assert_allclose(res[rank][3][tally][3], g, rtol=1e-9, atol=1e-12 * np.abs(g).max(),
                                           err_msg=f"rank {rank} gradient {tally}")
            for k in range(nscores):
                m, _, rel = (w[:, :, k] for w in want)
                mx, cnt = res[rank][4][nscores * tally + k]
                assert cnt == int((m != 0).sum()) > 0
                np.testing.assert_allclose(mx, rel[m != 0].max(), rtol=1e-12)
                one_mx, one_cnt = one.batch_max_rel_err(tally, k)
                assert cnt == one_cnt
                np.testing.assert_allclose(mx, one_mx, rtol=1e-12, atol=0)
    one.set_source_normalization(0)
    want = _exchanged(one, moments, np.random.default_rng(99).uniform(0.0, 1.0, (500, 3)))
    for rank in range(world):
        for how, got in (("reduce_tally_to_owners", res[rank][5]), ("allreduce_tally", res[rank][6])):
            for j, (g, w) in enumerate(zip(got, want)):
                fin = np.isfinite(w)
                np.testing.assert_array_equal(np.isfinite(g), fin)
                tol = 1e-12 * np.abs(w[fin]) + 1e-15 * np.abs(w[fin]).sum()
                assert (np.abs(g[fin] - w[fin]) <= tol).all(), f"rank {rank} {how} array {j}"
