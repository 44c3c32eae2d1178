"""Weight windows (pumitally_set_weight_windows, _generate_weight_windows and the lookups): MAGIC windows generated on
the device from the batch statistics must equal numpy's, built from batch_results kinds 0 and 2, bit for bit; the
lookups must equal a numpy gather through the particles' elements or through locate(); every refusal and every lookup
must leave the engine's tally state and the table bit-identical."""
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT
from locate_ref import MESHES, generic_points, non_finite_points, outside_points
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_batch_stats import MODES, Batches
from test_gpu_checkpoint import assert_same, snapshot
from test_gpu_tally_collisions import CASES

pytestmark = pytest.mark.gpu
INF = float("inf")


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def numpy_windows(eng, tally, score, time_bin, ratio, max_rel_err):
    """The MAGIC windows of pumitally_generate_weight_windows from the engine's batch results: [nbins, E] each."""
    phi = eng.batch_results(tally, 0)[time_bin, :, score]
    r = eng.batch_results(tally, 2)[time_bin, :, score]
    ok = (phi > 0) & np.isfinite(phi) & (r <= max_rel_err)
    pm = np.where(ok, phi, 0.0).max(axis=1)
    c = 2.0 / (ratio + 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        lo = (phi / pm[:, None]) * c
    hi = lo * ratio
    return np.where(ok, lo, -1.0), np.where(ok, hi, -1.0)


def full_snapshot(b):
    s = snapshot(b)
    for k in ("launches", "variant"):
        s[k] = np.int64(b.eng.get_option(k))
    s["elem"], s["pos"] = b.eng.elem_ids, b.eng.positions
    return s


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("case", list(CASES))
def test_generate_matches_numpy(case, mode):
    b = Batches(case, mode=mode, seed=4)
    for _ in range(3):
        b.move()
        b.eng.end_batch()
    b.move()  # an open batch: generation reads the folded batches only
    before = full_snapshot(b)
    nt = max(b.eng.time_bins, 1)
    for tally in (0, 1):
        for score in sorted({0, b.nscores - 1}):
            for tb in sorted({0, nt - 1}):
                for ratio, mre in ((5.0, INF), (2.0, 0.3), (1.0 + 2.0 ** -40, 0.05), (1e6, 1.0)):
                    b.eng.generate_weight_windows(tally, score, tb, ratio, mre)
                    assert b.eng.weight_window_groups == b.nbins
                    lo, hi = b.eng.weight_windows()
                    want_lo, want_hi = numpy_windows(b.eng, tally, score, tb, ratio, mre)
                    label = f"{case} mode {mode} tally {tally} score {score} time bin {tb} ratio {ratio} mre {mre}"
                    np.testing.assert_array_equal(bits(lo), bits(want_lo), err_msg=label)
                    np.testing.assert_array_equal(bits(hi), bits(want_hi), err_msg=label)
    # the lookups change nothing either
    b.eng.weight_windows_at_particles(np.arange(b.n, dtype=np.int32) % (b.nbins + 1))
    b.eng.weight_windows_at_particles_device()
    b.eng.weight_windows_at_points(np.random.default_rng(1).uniform(-1, 7, (500, 3)))
    import torch
    torch.cuda.synchronize()
    assert_same(before, full_snapshot(b), f"{case} mode {mode}")


def _engine_with_particles(n, seed=3, box=(6, 5, 4)):
    c, t = kuhn_box(*box)
    eng = PumiTally.from_arrays(c, t, n)
    wl = SyntheticWorkload(box=tuple(float(x) for x in box), num_particles=n, mean_length=1.0, seed=seed)
    return eng, wl, c, t


def random_table(rng, G, E):
    lo = rng.uniform(0.01, 2.0, (G, E))
    lo[rng.random((G, E)) < 0.2] = 0.0
    lo[rng.random((G, E)) < 0.05] = -3.0
    hi = lo * rng.uniform(1.5, 10.0, (G, E))
    hi[lo <= 0] = np.nan  # unread where there is no window
    stored_lo, stored_hi = np.where(lo > 0, lo, -1.0), np.where(lo > 0, hi, -1.0)
    return lo, hi, stored_lo, stored_hi


def gather(table, elems, groups):
    lo, hi = table
    G = lo.shape[0]
    ok = (groups >= 0) & (groups < G) & (elems >= 0)
    gi, ei = np.where(ok, groups, 0), np.where(ok, elems, 0)
    return np.where(ok, lo[gi, ei], -1.0), np.where(ok, hi[gi, ei], -1.0)


def test_set_get_round_trip_and_refusals(capfd):
    import ctypes as C

    eng, wl, c, t = _engine_with_particles(1000)
    E = eng.num_elements
    rng = np.random.default_rng(2)
    assert eng.weight_window_groups == 0
    lo0, hi0 = eng.weight_windows()
    assert lo0.shape == (0, E)
    lo, hi, slo, shi = random_table(rng, 3, E)
    eng.set_weight_windows(lo, hi)
    assert eng.weight_window_groups == 3
    got = eng.weight_windows()
    np.testing.assert_array_equal(bits(got[0]), bits(slo))
    np.testing.assert_array_equal(bits(got[1]), bits(shi))

    def refused(fn, why):
        capfd.readouterr()
        with pytest.raises((ValueError, RuntimeError)):
            fn()
        err = capfd.readouterr().err
        assert why in err, err
        now = eng.weight_windows()
        np.testing.assert_array_equal(bits(now[0]), bits(slo), err_msg=why)
        np.testing.assert_array_equal(bits(now[1]), bits(shi), err_msg=why)

    good = np.where(lo > 0, lo, 1.0), np.where(lo > 0, hi, 2.0)
    for i, (a, bb) in enumerate(((np.nan, 1.0), (1.0, np.nan), (np.inf, np.inf), (1.0, np.inf), (2.0, 2.0), (2.0, 1.0))):
        l2, h2 = good[0].copy(), good[1].copy()
        l2[i % 3, (37 * i) % E], h2[i % 3, (37 * i) % E] = a, bb
        refused(lambda: eng.set_weight_windows(l2, h2), "needs finite bounds")
    L = eng._L
    dp = C.POINTER(C.c_double)
    ptr = lambda a: a.ctypes.data_as(dp)  # noqa: E731
    for args, why in (((ptr(good[0]), ptr(good[1]), 3 * E - 1, 3), "ngroups * num_elements"),
                      ((ptr(good[0]), None, 3 * E, 3), "null bound array"),
                      ((ptr(good[0]), ptr(good[1]), 3 * E, 0), "ngroups must be >= 1"),
                      ((ptr(good[0]), ptr(good[1]), -3 * E, -3), "ngroups must be >= 1")):
        def call(a=args):
            if L.pumitally_set_weight_windows(eng._h, *a):
                raise RuntimeError("refused")
        refused(call, why)
    # generation is refused without batch statistics, leaving the table alone
    refused(lambda: eng.generate_weight_windows(), "batch statistics are off")
    # lookups at the particles are refused before CopyInitialPosition and with the wrong n
    refused(lambda: eng.weight_windows_at_particles(), "before CopyInitialPosition")
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    out = np.empty(2000)
    assert L.pumitally_get_weight_windows_at_particles(eng._h, None, ptr(out), ptr(out[1000:]), 999) != 0
    assert L.pumitally_get_weight_windows_at_points(eng._h, None, -1, None, None, None) != 0
    assert L.pumitally_get_weight_windows(eng._h, ptr(out), ptr(out), 3 * E - 1) != 0
    # removal
    eng.set_weight_windows(None)
    assert eng.weight_window_groups == 0 and eng.weight_windows()[0].size == 0
    lo_p, hi_p = eng.weight_windows_at_particles()
    assert (lo_p == -1).all() and (hi_p == -1).all()


def test_generate_refusals_change_nothing(capfd):
    b = Batches("s3_b3_t", mode=0, seed=6)
    b.move()
    b.eng.end_batch()
    table = random_table(np.random.default_rng(3), 2, b.eng.num_elements)
    b.eng.set_weight_windows(table[0], table[1])
    ref = full_snapshot(b)

    def refused(args, why):
        capfd.readouterr()
        with pytest.raises(RuntimeError):
            b.eng.generate_weight_windows(*args)
        assert why in capfd.readouterr().err
        now = b.eng.weight_windows()
        np.testing.assert_array_equal(bits(now[0]), bits(table[2]), err_msg=why)
        np.testing.assert_array_equal(bits(now[1]), bits(table[3]), err_msg=why)
        assert_same(ref, full_snapshot(b), why)

    refused((0, 0, 0, 5.0, INF), "at least two batches")
    b.move()
    b.eng.end_batch()
    ref = full_snapshot(b)
    for args, why in (((2, 0, 0, 5.0, INF), "tally must be"), ((-1, 0, 0, 5.0, INF), "tally must be"),
                      ((0, 3, 0, 5.0, INF), "score must be"), ((0, -1, 0, 5.0, INF), "score must be"),
                      ((0, 0, 4, 5.0, INF), "time_bin must be"), ((0, 0, -1, 5.0, INF), "time_bin must be"),
                      ((0, 0, 0, 1.0, INF), "ratio must be"), ((0, 0, 0, INF, INF), "ratio must be"),
                      ((0, 0, 0, float("nan"), INF), "ratio must be"), ((0, 0, 0, 0.5, INF), "ratio must be"),
                      ((0, 0, 0, 5.0, 0.0), "max_rel_err must be"), ((0, 0, 0, 5.0, -1.0), "max_rel_err must be"),
                      ((0, 0, 0, 5.0, float("nan")), "max_rel_err must be")):
        refused(args, why)
    # the collision tally without the estimator
    c, t = kuhn_box(3, 3, 3)
    e = PumiTally.from_arrays(c, t, 100)
    e.set_batch_statistics(True)
    wl = SyntheticWorkload(box=(3.0, 3.0, 3.0), num_particles=100, mean_length=1.0, seed=1)
    e.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    for _ in range(2):
        o, d, f, w = wl.next_step()
        e.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
        e.end_batch()
    capfd.readouterr()
    with pytest.raises(RuntimeError):
        e.generate_weight_windows(1)
    assert "collision estimator is off" in capfd.readouterr().err
    e.generate_weight_windows(0)
    assert e.weight_window_groups == 1


@pytest.mark.parametrize("n", [3001, 4096 + 77])
def test_particle_lookup_host_and_device(n):
    import torch

    eng, wl, c, t = _engine_with_particles(n)
    eng.set_option("chunk", 1024)  # several chunks, the last one partial
    E = eng.num_elements
    rng = np.random.default_rng(n)
    _, _, slo, shi = random_table(rng, 3, E)
    eng.set_weight_windows(np.where(slo > 0, slo, 0.0), np.where(slo > 0, shi, 0.0))
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    groups = rng.integers(-2, 5, n).astype(np.int32)  # 3 and 4 and the negatives are out of range
    groups[:3] = [-(2 ** 31), 2 ** 31 - 1, 3]
    for step, path in enumerate(("host", "device", "host", "device")):
        o, d, f, w = wl.next_step()
        if path == "host":
            eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
        else:
            T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
            do, dd, df, dw = T(o.reshape(-1)), T(d.reshape(-1)), T(f), T(w)
            eng.move_device(do.data_ptr(), dd.data_ptr(), df.data_ptr(), dw.data_ptr(),
                            torch.cuda.current_stream().cuda_stream)
        # device lookup straight behind the move, on the same stream, before anything synchronises
        dlo, dhi = eng.weight_windows_at_particles_device(torch.from_numpy(groups).cuda())
        d0lo, d0hi = eng.weight_windows_at_particles_device(device=0)
        torch.cuda.synchronize()
        elems = eng.elem_ids
        want = gather((slo, shi), elems, groups)
        want0 = gather((slo, shi), elems, np.zeros(n, np.int32))
        for got, w_, label in ((eng.weight_windows_at_particles(groups), want, "host"),
                               ((dlo.cpu().numpy(), dhi.cpu().numpy()), want, "device"),
                               (eng.weight_windows_at_particles(), want0, "host NULL groups"),
                               ((d0lo.cpu().numpy(), d0hi.cpu().numpy()), want0, "device NULL groups")):
            np.testing.assert_array_equal(bits(got[0]), bits(w_[0]), err_msg=f"step {step} {label}")
            np.testing.assert_array_equal(bits(got[1]), bits(w_[1]), err_msg=f"step {step} {label}")


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mesh", list(MESHES))
def test_point_lookup(mesh, path):
    import torch

    c, t = MESHES[mesh]()
    eng = PumiTally.from_arrays(c, t, 16)
    eng.set_option("chunk", 1024)
    rng = np.random.default_rng(5)
    _, _, slo, shi = random_table(rng, 2, eng.num_elements)
    eng.set_weight_windows(np.where(slo > 0, slo, 0.0), np.where(slo > 0, shi, 0.0))
    pts, _ = generic_points(mesh, c, t, 2999, rng)
    pts = np.concatenate([pts, outside_points(mesh, c, rng), non_finite_points()])
    groups = rng.integers(-1, 3, len(pts)).astype(np.int32)
    elems = eng.locate(pts)
    assert (elems[-len(non_finite_points()):] == -1).all() and (elems == -1).sum() > 100
    for g, gg in ((groups, groups), (None, np.zeros(len(pts), np.int32))):
        want = gather((slo, shi), elems, gg)
        if path == "host":
            got = eng.weight_windows_at_points(pts, g)
        else:
            dg = None if g is None else torch.from_numpy(g).cuda()
            lo, hi = eng.weight_windows_at_points_device(torch.from_numpy(pts).cuda(), dg)
            torch.cuda.synchronize()
            got = lo.cpu().numpy(), hi.cpu().numpy()
        np.testing.assert_array_equal(bits(got[0]), bits(want[0]))
        np.testing.assert_array_equal(bits(got[1]), bits(want[1]))
    assert eng.stats()["moves"] == 0 and (eng.flux == 0).all()


def test_windows_survive_resets_batches_configuration_and_checkpoints(tmp_path):
    b = Batches("s1_b3_mo", mode=1, seed=9)
    for _ in range(2):
        b.move()
        b.eng.end_batch()
    b.eng.generate_weight_windows(0, 0, 0, 4.0, INF)
    want = b.eng.weight_windows()
    assert (want[0] > 0).any()

    def same(label):
        got = b.eng.weight_windows()
        np.testing.assert_array_equal(bits(got[0]), bits(want[0]), err_msg=label)
        np.testing.assert_array_equal(bits(got[1]), bits(want[1]), err_msg=label)

    b.eng.reset_tally()
    same("reset_tally")
    b.move()
    b.eng.end_batch()
    same("end_batch")
    p = str(tmp_path / "x.ckpt")
    b.eng.save_checkpoint(p)
    b.eng.load_checkpoint(p)
    same("checkpoint")
    for call in (lambda: b.eng.set_scores(2), lambda: b.eng.set_score_bins(2), lambda: b.eng.set_time_bins([0.0, 1.0]),
                 lambda: b.eng.set_moments(0), lambda: b.eng.set_batch_statistics(False),
                 lambda: b.eng.set_collision_estimator(False)):
        call()
        same("set_*")


def test_vtk_arrays(tmp_path):
    from vtk_reader import read_vtu_cell_data

    b = Batches("s1", mode=0, seed=12)
    for _ in range(2):
        b.move()
        b.eng.end_batch()
    piece = lambda p: os.path.join(p, "pieces", "piece_0.vtu")  # noqa: E731
    plain = str(tmp_path / "plain.vtk")
    b.eng.WriteTallyResults(plain)
    with open(piece(plain), "rb") as f:
        plain_bytes = f.read()
    names_before = list(read_vtu_cell_data(piece(plain)))
    b.eng.generate_weight_windows(0, 0, 0, 5.0, INF)
    lo, hi = b.eng.weight_windows()
    one = str(tmp_path / "one.vtk")
    b.eng.WriteTallyResults(one)
    cells = read_vtu_cell_data(piece(one))
    assert list(cells)[:len(names_before)] == names_before
    assert list(cells)[len(names_before):] == ["ww_lower", "ww_upper"]
    np.testing.assert_array_equal(bits(np.asarray(cells["ww_lower"]).reshape(-1)), bits(lo[0]))
    np.testing.assert_array_equal(bits(np.asarray(cells["ww_upper"]).reshape(-1)), bits(hi[0]))
    E = b.eng.num_elements
    _, _, slo, shi = random_table(np.random.default_rng(4), 3, E)
    b.eng.set_weight_windows(np.where(slo > 0, slo, 0.0), np.where(slo > 0, shi, 0.0))
    three = str(tmp_path / "three.vtk")
    b.eng.WriteTallyResults(three)
    cells = read_vtu_cell_data(piece(three))
    assert list(cells)[len(names_before):] == [f"ww_{k}_g{g}" for g in range(3) for k in ("lower", "upper")]
    for g in range(3):
        np.testing.assert_array_equal(bits(np.asarray(cells[f"ww_lower_g{g}"]).reshape(-1)), bits(slo[g]))
        np.testing.assert_array_equal(bits(np.asarray(cells[f"ww_upper_g{g}"]).reshape(-1)), bits(shi[g]))
    b.eng.set_weight_windows(None)
    again = str(tmp_path / "again.vtk")
    b.eng.WriteTallyResults(again)
    with open(piece(again), "rb") as f:
        assert f.read() == plain_bytes


def test_forward_beam_windows_fall_with_depth():
    """Tracks enter a 4 x 4 x 12 Kuhn box through its z = 0 face, mostly along +z, with exponential lengths: the flux falls
    with depth, so must the slab-averaged lower bounds, and the element with the most flux has lower = 2 / (ratio + 1)."""
    box = (4, 4, 12)
    c, t = kuhn_box(*box)
    n = 200_000
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_batch_statistics(True)
    rng = np.random.default_rng(8)
    o0 = np.column_stack([rng.uniform(0.01, 3.99, n), rng.uniform(0.01, 3.99, n), np.full(n, 1e-3)])
    eng.CopyInitialPosition(o0.reshape(-1).copy())
    for _ in range(4):
        o = np.column_stack([rng.uniform(0.01, 3.99, n), rng.uniform(0.01, 3.99, n), np.full(n, 1e-3)])
        mu = rng.uniform(0.7, 1.0, n)
        phi = rng.uniform(0.0, 2 * np.pi, n)
        s = np.sqrt(1 - mu * mu)
        u = np.column_stack([s * np.cos(phi), s * np.sin(phi), mu])
        d = o + rng.exponential(2.5, n)[:, None] * u
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), np.ones(n, np.int8), np.ones(n))
        eng.end_batch()
    ratio = 5.0
    eng.generate_weight_windows(0, 0, 0, ratio, INF)
    lo, hi = eng.weight_windows()
    lo, hi = lo[0], hi[0]
    mean = eng.batch_results(0, 0)[0, 0, 0]
    top = np.argmax(mean)
    assert lo[top] == 2.0 / (ratio + 1.0) and hi[top] == lo[top] * ratio
    assert lo.max() == lo[top]
    z = np.asarray(c)[np.asarray(t)].mean(axis=1)[:, 2]
    slabs = [lo[(z >= k) & (z < k + 1)] for k in range(8)]
    assert all((s > 0).all() for s in slabs)
    avg = [s.mean() for s in slabs]
    assert all(a > b for a, b in zip(avg, avg[1:])), avg


def test_config_c2_full_size():
    """Full-size c2 with 16 score bins as energy groups and 10 M particles: the generated table against numpy, and the
    device and host particle lookups against a gather through elem_ids()."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n = cfg["particles"]
    eng = PumiTally.from_arrays(coords, t2v, n)
    eng.set_batch_statistics(True)
    eng.set_score_bins(16)
    eng.set_source_normalization(1)
    wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
    g = torch.Generator(device="cuda").manual_seed(3)
    for _ in range(3):
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        bins = torch.randint(0, 16, (n,), device="cuda", dtype=torch.int32, generator=g)
        eng.move_device_binned(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), bins.data_ptr(), s)
        torch.cuda.synchronize()
        eng.end_batch()
    eng.generate_weight_windows(0, 0, 0, 5.0, 0.2)
    assert eng.weight_window_groups == 16
    lo, hi = eng.weight_windows()
    want = numpy_windows(eng, 0, 0, 0, 5.0, 0.2)
    np.testing.assert_array_equal(bits(lo), bits(want[0]))
    np.testing.assert_array_equal(bits(hi), bits(want[1]))
    assert (lo > 0).any()
    groups = torch.randint(-1, 17, (n,), device="cuda", dtype=torch.int32, generator=g)
    dlo, dhi = eng.weight_windows_at_particles_device(groups)
    torch.cuda.synchronize()
    gh = groups.cpu().numpy()
    w_lo, w_hi = gather((lo, hi), eng.elem_ids, gh)
    np.testing.assert_array_equal(bits(dlo.cpu().numpy()), bits(w_lo))
    np.testing.assert_array_equal(bits(dhi.cpu().numpy()), bits(w_hi))
    h_lo, h_hi = eng.weight_windows_at_particles(gh)
    np.testing.assert_array_equal(bits(h_lo), bits(w_lo))
    np.testing.assert_array_equal(bits(h_hi), bits(w_hi))


def test_cxx_program_with_weight_windows(tmp_path):
    """A C++ caller of PumiTallyExtras.h: GenerateWeightWindows, the lookups, SetWeightWindows and GetWeightWindows."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "ww_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "ww_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "WEIGHT_WINDOWS_OK" in out, out


def _centroid_batches(eng, c, t, seeds):
    """One collision batch per seed list entry: for every seed one event at every element's centroid (two ranks' events
    at one address add in either order to the same bits), then end_batch."""
    cen = np.asarray(c)[np.asarray(t)].mean(axis=1)
    for batch in seeds:
        for seed in batch:
            r = np.random.default_rng(seed)
            eng.tally_collisions(cen, r.uniform(0.0, 2.0, len(cen)) * (r.random(len(cen)) < 0.8),
                                 bins=r.integers(0, 2, len(cen)).astype(np.int32))
        eng.end_batch()


def _two_gpu_ww_worker(rank, world, port, q):
    import sys

    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pumiumtally_b200.distributed import broadcast_unique_id

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    c, t = kuhn_box(5, 5, 5)
    eng = PumiTally.from_arrays(c, t, 16, device=rank)
    eng.set_collision_estimator(True)
    eng.set_batch_statistics(True)
    eng.set_score_bins(2)
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    _centroid_batches(eng, c, t, [[100 * b + rank] for b in range(4)])
    eng.generate_weight_windows(1, 0, 0, 5.0, 0.5)
    q.put((rank, eng.weight_windows()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpus_generate_the_one_rank_table():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 211) % 1000
    procs = [ctx.Process(target=_two_gpu_ww_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    c, t = kuhn_box(5, 5, 5)
    one = PumiTally.from_arrays(c, t, 16)
    one.set_collision_estimator(True)
    one.set_batch_statistics(True)
    one.set_score_bins(2)
    _centroid_batches(one, c, t, [[100 * b, 100 * b + 1] for b in range(4)])
    one.generate_weight_windows(1, 0, 0, 5.0, 0.5)
    want = one.weight_windows()
    for rank in range(2):
        for k in range(2):
            np.testing.assert_array_equal(bits(res[rank][1][k]), bits(want[k]), err_msg=f"rank {rank}")
