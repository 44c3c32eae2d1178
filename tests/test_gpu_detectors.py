"""Point detectors (pumitally_set_point_detectors): next-event estimates of the flux at fixed points, with the optical
depth of every ray traced through the mesh.  Checked against exact uncollided fluxes, against the numpy reference
(tests/detectors_ref.py), and statistically against an independent quadrature; the detector calls must change nothing
else."""
import math
import os
import subprocess

import numpy as np
import pytest

from detectors_ref import reference_detectors
from helpers import ROOT
from locate_ref import MESHES, generic_points
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

pytestmark = pytest.mark.gpu


def _to_device(*arrays):
    import torch

    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _engine(c, t, n, det, r0, sigma, nbins=1, nscores=1, edges=None):
    eng = PumiTally.from_arrays(c, t, n)
    if nbins > 1:
        eng.set_score_bins(nbins)
    if nscores > 1:
        eng.set_scores(nscores)
    if edges is not None:
        eng.set_time_bins(edges)
    eng.set_point_detectors(det, r0)
    eng.set_detector_cross_sections(sigma)
    assert eng.point_detectors == len(det) == eng.get_option("point_detectors")
    return eng


def _tally(eng, path, pts, w, **kw):
    if path == "host":
        eng.tally_detectors(pts, w, **kw)
    elif path == "device":
        import torch

        dev = {k: (None if v is None else _to_device(v)[0]) for k, v in kw.items()}
        eng.tally_detectors_device(*_to_device(pts, w), **dev)
        torch.cuda.synchronize()
    else:  # the particles, placed at the points in the elements that contain them
        import torch

        x, el = _to_device(pts, eng.locate(pts).astype(np.int32))
        eng.set_state_device(x.data_ptr(), el.data_ptr(), 0, len(pts))
        torch.cuda.synchronize()
        flag = np.ones(len(pts), dtype=np.int8)
        if path == "particles":
            eng.tally_detectors_at_particles(flag, w, **kw)
        else:
            import torch

            dev = {k: (None if v is None else _to_device(v)[0]) for k, v in kw.items()}
            eng.tally_detectors_at_particles_device(*_to_device(flag, w), **dev)
            torch.cuda.synchronize()


PATHS = ["host", "device", "particles", "particles_device"]


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("slabs", [False, True], ids=["homogeneous", "two_slab"])
def test_exact_uncollided_flux(slabs, path):
    """Isotropic point sources score w exp(-tau) / (4 pi R^2), tau = S1 l1 + S2 l2 along the line, to rtol 1e-12."""
    c, t = kuhn_box(6, 5, 4)
    s1, s2 = 0.4, (1.3 if slabs else 0.4)
    cen = c[t].mean(1)
    sigma = np.where(cen[:, 0] < 3.0, s1, s2)[None, :]
    rng = np.random.default_rng(5)
    n = 400
    pts = rng.uniform([0.05, 0.05, 0.05], [5.95, 4.95, 3.95], size=(n, 3))
    w = rng.uniform(0.5, 2.0, n)
    det = np.array([[4.7, 2.3, 1.9]])
    eng = _engine(c, t, n, det, np.zeros(1), sigma)
    _tally(eng, path, pts, w)
    u = det[0] - pts
    R = np.sqrt((u ** 2).sum(1))
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.where(pts[:, 0] < 3.0, (3.0 - pts[:, 0]) / u[:, 0], 0.0)  # fraction of the line with x < 3 (det at x > 3)
    tau = s1 * f * R + s2 * (1.0 - f) * R
    want = math.fsum(w * np.exp(-tau) / (4 * math.pi * R ** 2))
    got = eng.detector_results(0)[0, 0, 0, 0]
    assert got == pytest.approx(want, rel=1e-12)
    assert eng.get_option("detector_rays") == n
    assert eng.get_option("detector_crossings") > n


@pytest.mark.parametrize("D", [1, 37])
@pytest.mark.parametrize("mesh", ["kuhn", "void"])
def test_device_calls_match_the_reference(mesh, D):
    """Random Sigma, pdfs, responses, two scores, score bins and time bins whose edges the arrival times cross; with D =
    1, more events than one "chunk" (1024) of the host call."""
    c, t = MESHES[mesh]()
    rng = np.random.default_rng(D + len(mesh))
    pts, _ = generic_points(mesh, c, t, 150 if D > 1 else 1100, rng)
    det, _ = generic_points(mesh, c, t, D, rng)
    n, nbins, nscores = len(pts), 2, 2
    edges = np.array([0.0, 0.5, 1.0, 2.0, 5.0])
    sigma = rng.uniform(0.05, 1.0, size=(nbins, len(t)))
    r0 = rng.uniform(0.0, 0.8, D) if D > 1 else np.array([1.5])
    w = rng.uniform(0.5, 2.0, n)
    pdf = rng.uniform(0.0, 0.3, size=(n, D))
    r = rng.uniform(0.2, 2.0, size=(n, nscores))
    bins = rng.integers(0, nbins + 1, n).astype(np.int32)
    times = rng.uniform(0.0, 1.5, n)
    speeds = rng.uniform(1.0, 4.0, n)
    eng = _engine(c, t, n, det, r0, sigma, nbins, nscores, edges)
    elem = eng.locate(pts)
    want, wcnt = reference_detectors(c, t, elem, pts, w, pdf, r, bins, times, speeds, edges, nbins, nscores, sigma, det,
                                     r0)
    names = ["detector_rays", "detector_rays_shadowed", "detector_rays_lost", "detector_inside_r0", None,
             "detector_events_outside", "detector_events_rejected"]
    for path in ("device", "host", "particles", "particles_device"):
        eng.reset_tally()
        eng.set_option("chunk", 1024)
        _tally(eng, path, pts, w, pdf=pdf, responses=r, bins=bins, times=times, speeds=speeds)
        got = eng.detector_results(0)
        np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-14 * np.abs(want).max())
        assert tuple(eng.get_option(k) if k else None for k in names) == wcnt, path
    assert wcnt[0] > 0 and wcnt[3] > 0


def test_statistics_against_quadrature():
    """A uniform isotropic volume source in a homogeneous box: the batch mean at each detector lies within 5 standard
    errors of (1 / (4 pi V Sigma)) int (1 - exp(-Sigma l(Omega))) dOmega, with a standard error below 1 %; kinds 1-3
    are numpy's statistics of the kind-0 results of each batch."""
    import torch
    from scipy import integrate

    L = np.array([6.0, 5.0, 4.0])
    c, t = kuhn_box(6, 5, 4)
    sig = 0.5
    det = np.array([[3.0, 2.5, 2.0], [1.7, 3.1, 1.4]])
    r0 = np.array([0.5, 0.3])
    N, B = 1 << 20, 20
    eng = _engine(c, t, N, det, r0, np.full((1, len(t)), sig))
    eng.set_batch_statistics(True)
    eng.set_source_normalization(2, float(N))
    g = torch.Generator(device="cuda").manual_seed(11)
    Lt = torch.tensor(L, dtype=torch.float64, device="cuda")
    w = torch.ones(N, dtype=torch.float64, device="cuda")
    per_batch = []
    for _ in range(B):
        pts = (torch.rand((N, 3), dtype=torch.float64, device="cuda", generator=g) * Lt).contiguous()
        eng.tally_detectors_device(pts, w)
        torch.cuda.synchronize()
        per_batch.append(eng.detector_results(0)[0, 0, 0].copy())
        eng.end_batch()
    x = np.array(per_batch)
    mean, se, rel = (eng.detector_results(k)[0, 0, 0] for k in (1, 2, 3))
    np.testing.assert_allclose(mean, x.mean(0), rtol=1e-12)
    np.testing.assert_allclose(se, x.std(0, ddof=1) / math.sqrt(B), rtol=1e-9)
    np.testing.assert_allclose(rel, se / mean, rtol=1e-12)
    V = float(np.prod(L))
    for d in range(len(det)):
        p = det[d]

        def ell(th, ph):
            u = np.array([math.sin(th) * math.cos(ph), math.sin(th) * math.sin(ph), math.cos(th)])
            with np.errstate(divide="ignore"):
                s = np.where(u > 0, (L - p) / u, np.where(u < 0, -p / u, np.inf))
            return s.min()

        val, _ = integrate.dblquad(lambda th, ph: (1.0 - math.exp(-sig * ell(th, ph))) * math.sin(th), 0.0, 2 * math.pi,
                                   0.0, math.pi, epsabs=1e-12, epsrel=1e-10)
        want = val / (4 * math.pi * V * sig)
        assert se[d] < 0.01 * mean[d], (d, se[d], mean[d])
        assert abs(mean[d] - want) < 5 * se[d], (d, mean[d], want, se[d])


def test_detector_calls_change_nothing_else():
    c, t = kuhn_box(6, 5, 4)
    n = 3000
    wl = SyntheticWorkload(box=(6.0, 5.0, 4.0), num_particles=n, mean_length=1.0, seed=2)
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_collision_estimator(True)
    eng.set_batch_statistics(True)
    eng.set_point_detectors(np.array([[2.0, 2.0, 2.0], [4.5, 1.0, 3.0]]), np.array([0.1, 0.0]))
    eng.set_detector_cross_sections(np.full((1, len(t)), 0.3))
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    eng.MoveToNextLocation(o.copy(), d.copy(), f.copy(), w.copy())
    eng.tally_collisions(np.reshape(d, (-1, 3))[:100], np.ones(100))
    eng.end_batch()
    eng.MoveToNextLocation(d.copy(), (o * 0.5 + d * 0.5).copy(), np.ones(n, dtype=np.int8), w.copy())

    def snapshot():
        return [eng.flux.copy(), eng.collision_results(0).copy(), eng.collision_results(1).copy(), eng.positions.copy(),
                eng.elem_ids.copy(), eng.batch_results(0, 0).copy(), dict(eng.stats()),
                eng.get_option("variant"), eng.get_option("launches"), eng.get_option("collisions")]

    before = snapshot()
    rng = np.random.default_rng(1)
    eng.tally_detectors(rng.uniform(0, 4, size=(500, 3)), np.ones(500))
    eng.tally_detectors_at_particles(np.ones(n, dtype=np.int8), np.ones(n))
    after = snapshot()
    for a, b in zip(before, after):
        if isinstance(a, np.ndarray):
            assert np.array_equal(a, b)
        elif isinstance(a, dict):
            assert {k: v for k, v in a.items() if k != "kernel_ms"} == {k: v for k, v in b.items() if k != "kernel_ms"}
        else:
            assert a == b
    assert eng.detector_results(0).sum() > 0


def test_refusals_resets_and_counters(tmp_path):
    c, t = kuhn_box(4, 4, 4)
    E = len(t)
    eng = PumiTally.from_arrays(c, t, 64)
    pts = np.array([[1.0, 1.0, 1.0], [2.5, 2.5, 2.5]])
    with pytest.raises(RuntimeError):  # no detectors
        eng.tally_detectors(pts, np.ones(2))
    for bad in ((np.array([[5.0, 1.0, 1.0]]), [0.0]), (np.array([[np.nan, 1.0, 1.0]]), [0.0]),
                (np.array([[1.0, 1.0, 1.0]]), [-1.0]), (np.array([[1.0, 1.0, 1.0]]), [np.inf]),
                (np.tile([[1.0, 1.0, 1.0]], (257, 1)), np.zeros(257))):
        with pytest.raises(ValueError):
            eng.set_point_detectors(*bad)
        assert eng.point_detectors == 0
    eng.set_point_detectors(pts, np.array([0.0, 1.0]))
    with pytest.raises(RuntimeError):  # no table
        eng.tally_detectors(pts, np.ones(2))
    for bad in (np.full((1, E), -1.0), np.full((1, E), np.nan), np.ones((1, E - 1))):
        with pytest.raises(ValueError):
            eng.set_detector_cross_sections(bad)
    eng.set_detector_cross_sections(np.full((1, E), 0.2))
    rng = np.random.default_rng(4)
    ev = np.concatenate([rng.uniform(0.01, 3.99, size=(300, 3)), [[9.0, 1.0, 1.0], [np.nan, 1.0, 1.0]]])
    w = np.ones(len(ev))
    w[5] = np.inf
    pdf = np.full((len(ev), 2), 0.05)
    pdf[7, 1] = -0.1    # a negative pdf rejects the event
    pdf[8, 0] = np.nan  # so does a non-finite one
    ev[9] = pts[0]      # an event on detector 0 (r0 == 0) is rejected
    bins = np.zeros(len(ev), dtype=np.int32)
    bins[10:20] = 1     # outside [0, 1): skipped, not counted
    eng.tally_detectors(ev, w, pdf=pdf, bins=bins)
    rays = sum(eng.get_option(k) for k in ("detector_rays", "detector_rays_shadowed", "detector_rays_lost",
                                           "detector_inside_r0"))
    assert eng.get_option("detector_events_outside") == 1 and eng.get_option("detector_events_rejected") == 5
    assert rays == 2 * (len(ev) - 6) - 2 * 10
    assert eng.get_option("detector_inside_r0") > 0
    before = eng.detector_results(0)
    with pytest.raises(ValueError):
        eng.set_detector_cross_sections(np.ones((2, E)))
    assert np.array_equal(eng.detector_results(0), before)
    eng.reset_tally()
    assert not eng.detector_results(0).any() and eng.get_option("detector_rays") == 0
    eng.set_score_bins(2)  # another number of groups drops the table
    with pytest.raises(RuntimeError):
        eng.tally_detectors(pts, np.ones(2))
    eng.set_detector_cross_sections(np.ones((2, E)))
    eng.tally_detectors(pts, np.ones(2), bins=np.array([1, 5], dtype=np.int32))
    assert eng.detector_results(0).shape == (1, 2, 1, 2)
    eng.set_point_detectors(None, None)
    assert eng.point_detectors == 0


@pytest.mark.parametrize("D", [1, 8])
def test_config_c2_ten_million_events(D):
    """Full-size c2: 10 M isotropic events at D detectors; every event inside the mesh makes D rays, and the homogeneous
    estimate of the near detector is close to the sum of exp(-Sigma R) / (4 pi R^2) over a numpy subsample."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    cells = np.array(cfg["cells"], dtype=np.float64)
    n = 10_000_000
    rng = np.random.default_rng(D)
    det = rng.uniform(0.2 * cells, 0.8 * cells, size=(D, 3))
    eng = _engine(coords, t2v, 16, det, np.full(D, 0.5), np.full((1, len(t2v)), 0.05))
    g = torch.Generator(device="cuda").manual_seed(3)
    pts = (torch.rand((n, 3), dtype=torch.float64, device="cuda", generator=g) * torch.tensor(cells, device="cuda"))
    w = torch.ones(n, dtype=torch.float64, device="cuda")
    eng.tally_detectors_device(pts.contiguous(), w)
    torch.cuda.synchronize()
    total = sum(eng.get_option(k) for k in ("detector_rays", "detector_rays_shadowed", "detector_rays_lost",
                                            "detector_inside_r0"))
    assert total == D * n and eng.get_option("detector_rays_lost") == 0 and eng.get_option("detector_rays_shadowed") == 0
    got = eng.detector_results(0)[0, 0, 0]
    p = pts.cpu().numpy()
    for d in range(D):
        R = np.sqrt(((p - det[d]) ** 2).sum(1))
        far = R >= 0.5
        want = np.sum(np.exp(-0.05 * R[far]) / (4 * math.pi * R[far] ** 2)) + \
            (~far).sum() * 3 * (-math.expm1(-0.05 * 0.5) / (0.05 * 0.5)) / (4 * math.pi * 0.25)
        assert got[d] == pytest.approx(want, rel=1e-9)


def test_cxx_program_with_detectors(tmp_path):
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "detectors_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "detectors_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "DETECTORS_OK" in out, out


def _checkpoint_engine(det=((1.0, 1.0, 1.0), (2.5, 2.5, 2.5)), r0=(0.0, 1.0), sig=0.2):
    c, t = kuhn_box(4, 4, 4)
    eng = PumiTally.from_arrays(c, t, 64)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(2, 100.0)
    eng.set_point_detectors(np.array(det), np.array(r0))
    eng.set_detector_cross_sections(np.full((1, len(t)), sig))
    return eng


def test_checkpoints_save_load_and_merge(tmp_path):
    """The open detector tally, its counters and its batch statistics round-trip bit for bit in a version-3 file; a
    merge combines the statistics; other detectors or another table are refused with a message that names them."""
    rng = np.random.default_rng(8)
    a = _checkpoint_engine()
    for _ in range(3):
        a.tally_detectors(rng.uniform(0.01, 3.99, size=(500, 3)), rng.uniform(0.5, 1.5, 500))
        a.end_batch()
    a.tally_detectors(rng.uniform(0.01, 3.99, size=(200, 3)), np.ones(200))  # the open batch
    path = str(tmp_path / "a.ckpt")
    a.save_checkpoint(path)
    assert open(path, "rb").read()[8:12] == (3).to_bytes(4, "little")
    names = ("detector_rays", "detector_rays_shadowed", "detector_inside_r0", "detector_crossings",
             "detector_events_outside", "detector_events_rejected")
    b = _checkpoint_engine()
    b.load_checkpoint(path)
    for k in range(4):
        assert np.array_equal(a.detector_results(k), b.detector_results(k)), k
    assert [a.get_option(k) for k in names] == [b.get_option(k) for k in names]
    # merge: a file saved at a batch end, into an engine with batches of its own
    c = _checkpoint_engine()
    xs = []
    for _ in range(2):
        c.tally_detectors(rng.uniform(0.01, 3.99, size=(500, 3)), np.ones(500))
        xs.append(c.detector_results(0)[0, 0, 0].copy())
        c.end_batch()
    c.save_checkpoint(str(tmp_path / "c.ckpt"))
    d = _checkpoint_engine()
    for _ in range(3):
        d.tally_detectors(rng.uniform(0.01, 3.99, size=(500, 3)), np.ones(500))
        xs.append(d.detector_results(0)[0, 0, 0].copy())
        d.end_batch()
    d.merge_checkpoint(str(tmp_path / "c.ckpt"))
    x = np.array(xs)
    np.testing.assert_allclose(d.detector_results(1)[0, 0, 0], x.mean(0), rtol=1e-13)
    np.testing.assert_allclose(d.detector_results(2)[0, 0, 0], x.std(0, ddof=1) / np.sqrt(5), rtol=1e-10)
    assert d.batches == 5
    for kw in ({"r0": (0.0, 1.0 + 1e-15)}, {"sig": 0.2000001}, {"det": ((1.0, 1.0, 1.0), (2.5, 2.5, 2.4))},
               {"det": ((1.0, 1.0, 1.0),), "r0": (0.0,)}):
        e = _checkpoint_engine(**kw)
        before = e.detector_results(0)
        for call in (e.load_checkpoint, e.merge_checkpoint):
            with pytest.raises(RuntimeError):
                call(str(tmp_path / "c.ckpt"))
        assert np.array_equal(e.detector_results(0), before)


def test_removing_the_detectors_keeps_the_previous_file_bytes(tmp_path):
    """An engine whose detectors were set and removed writes the same bytes as one that never had them (version 1)."""
    rng = np.random.default_rng(2)
    pts = rng.uniform(0.01, 3.99, size=(64, 3))
    files = []
    for with_det in (False, True):
        c, t = kuhn_box(4, 4, 4)
        e = PumiTally.from_arrays(c, t, 64)
        e.set_batch_statistics(True)
        if with_det:
            e.set_point_detectors(np.array([[1.0, 1.0, 1.0]]), np.array([0.0]))
            e.set_detector_cross_sections(np.full((1, len(t)), 0.2))
            e.set_point_detectors(None, None)
        e.CopyInitialPosition(pts.reshape(-1).copy())
        e.end_batch()
        p = str(tmp_path / f"f{int(with_det)}.ckpt")
        e.save_checkpoint(p)
        files.append(open(p, "rb").read())
    assert files[0] == files[1] and files[0][8:12] == (1).to_bytes(4, "little")


def _two_gpu_detectors_worker(rank, world, port, q):
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
    eng.set_batch_statistics(True)
    eng.set_point_detectors(np.array([[2.5, 2.5, 2.5], [1.0, 4.0, 2.0]]), np.array([0.5, 0.0]))
    eng.set_detector_cross_sections(np.full((1, eng.num_elements), 0.3))
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    rng = np.random.default_rng(rank)
    out = {"local": [], "allreduce": [], "owners": [], "batch": []}
    for b in range(3):
        pts = rng.uniform(0.0, 5.0, (20_000, 3))
        eng.tally_detectors(pts, rng.uniform(0.5, 1.5, 20_000), responses=rng.uniform(0.0, 1.0, (20_000, 2)))
        out["local"].append(eng.detector_results(0))
        eng.allreduce_tally()
        out["allreduce"].append(eng.detector_results(0))
        eng.reduce_tally_to_owners()
        out["owners"].append(eng.detector_results(0))
        eng.end_batch()
    out["batch"] = [eng.detector_results(k) for k in (1, 2, 3)]
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_exchange_sums_the_detector_tallies():
    """After each exchange kind 0 is the sum over the ranks on every rank; after end_batch kinds 1-3 are the statistics
    of those sums, the same on every rank."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 41) % 1000
    procs = [ctx.Process(target=_two_gpu_detectors_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    a, b = res[0][1], res[1][1]
    sums = [x + y for x, y in zip(a["local"], b["local"])]
    for r in (a, b):
        for k in ("allreduce", "owners"):
            for got, want in zip(r[k], sums):
                np.testing.assert_allclose(got, want, rtol=1e-13)
    x = np.array(sums)
    for r in (a, b):
        np.testing.assert_allclose(r["batch"][0], x.mean(0), rtol=1e-12)
        np.testing.assert_allclose(r["batch"][1], x.std(0, ddof=1) / np.sqrt(3), rtol=1e-9)
    for k in range(3):
        assert np.array_equal(a["batch"][k], b["batch"][k])
