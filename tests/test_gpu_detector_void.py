"""The detector void (pumitally_set_detector_void): point-detector rays through the space outside the mesh, detectors
outside the hull and re-entry across concave parts of it.  Checked against the void reference
(tests/detector_void_ref.py), against exact uncollided fluxes, bit for bit against the mode off where no ray leaves the
mesh, and for its refusals, resets and checkpoints."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from detector_void_ref import comb_mesh, reference_void
from helpers import ROOT, carve
from locate_ref import MESHES, generic_points
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_host_emul_detector_void import cavity_points, outside_points

pytestmark = pytest.mark.gpu

COUNTERS = ["detector_rays", "detector_rays_shadowed", "detector_rays_lost", "detector_inside_r0", None,
            "detector_events_outside", "detector_events_rejected"]


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
    eng.set_detector_void(True)
    eng.set_point_detectors(det, r0)
    eng.set_detector_cross_sections(sigma)
    assert eng.detector_void and eng.get_option("detector_void") == 1
    return eng


def _tally(eng, path, pts, w, **kw):
    import torch

    if path == "host":
        eng.tally_detectors(pts, w, **kw)
    elif path == "device":
        dev = {k: (None if v is None else _to_device(v)[0]) for k, v in kw.items()}
        eng.tally_detectors_device(*_to_device(pts, w), **dev)
        torch.cuda.synchronize()
    else:  # the particles, placed at the points (inside the mesh) in the elements that contain them
        el = eng.locate(pts).astype(np.int32)
        assert (el >= 0).all()
        x, el = _to_device(pts, el)
        eng.set_state_device(x.data_ptr(), el.data_ptr(), 0, len(pts))
        torch.cuda.synchronize()
        flag = np.ones(len(pts), dtype=np.int8)
        if path == "particles":
            eng.tally_detectors_at_particles(flag, w, **kw)
        else:
            dev = {k: (None if v is None else _to_device(v)[0]) for k, v in kw.items()}
            eng.tally_detectors_at_particles_device(*_to_device(flag, w), **dev)
            torch.cuda.synchronize()


PATHS = ["device", "host", "particles", "particles_device"]
VOID_MESHES = {"l_shape": MESHES["l_shape"], "void": MESHES["void"], "comb": comb_mesh}


@pytest.mark.parametrize("D", [1, 37])
@pytest.mark.parametrize("mesh", list(VOID_MESHES))
def test_four_calls_match_the_void_reference(mesh, D):
    """Events inside, in the notch, cavity or slots and beyond the box; detectors anywhere; random Sigma, pdfs, two
    scores, score bins and time bins the arrival times cross; with D = 1 more events than one "chunk" (1024)."""
    c, t = VOID_MESHES[mesh]()
    rng = np.random.default_rng(D + 3 * len(mesh))
    ni = 900 if D == 1 else 60
    pts = np.concatenate([generic_points(mesh, c, t, ni, rng)[0], cavity_points(mesh, c, rng, ni // 4),
                          outside_points(c, rng, ni // 4, far=3.0)])
    det = np.concatenate([generic_points(mesh, c, t, max(D // 3, 1), rng)[0], cavity_points(mesh, c, rng, D // 3),
                          outside_points(c, rng, D, far=50.0)])[:D]
    if D == 1:
        det = cavity_points(mesh, c, rng, 1)
    n, nbins, nscores = len(pts), 2, 2
    edges = np.array([0.0, 0.5, 1.0, 2.0, 80.0])
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
    assert (elem < 0).sum() > 0
    # a particle is always in an element: the particle calls take the events inside the mesh (their rays still leave
    # it and come back), the located calls all of them
    inn = elem >= 0
    args = {True: (pts, w, pdf, r, bins, times, speeds), False: tuple(a[inn] for a in (pts, w, pdf, r, bins, times, speeds))}
    eng_p = _engine(c, t, int(inn.sum()), det, r0, sigma, nbins, nscores, edges)
    for path in PATHS:
        located = path in ("device", "host")
        p_, w_, pdf_, r_, b_, t_, v_ = args[located]
        eng = eng if located else eng_p
        want, wcnt = reference_void(c, t, elem if located else elem[inn], p_, w_, pdf_, r_, b_, t_, v_, edges, nbins,
                                    nscores, sigma, det, r0)
        eng.reset_tally()
        assert eng.detector_hull_entries == 0
        eng.set_option("chunk", 1024)
        _tally(eng, path, p_, w_, pdf=pdf_, responses=r_, bins=b_, times=t_, speeds=v_)
        got = eng.detector_results(0)
        np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-14 * np.abs(want).max())
        cnt = tuple(eng.get_option(k) if k else None for k in COUNTERS)
        assert cnt == wcnt, path
        assert cnt[1] == cnt[2] == cnt[5] == 0
        assert eng.detector_hull_entries > 0 or not located  # the outside events' rays enter
    assert wcnt[0] > 0 and wcnt[3] > 0


@pytest.mark.parametrize("path", PATHS)
def test_convex_box_detectors_outside_are_exact(path):
    """Detectors outside a Kuhn box: w exp(-Sigma l_inside) / (4 pi R^2) to rtol 1e-12, l_inside from the slab clip."""
    c, t = kuhn_box(6, 5, 4)
    L = np.array([6.0, 5.0, 4.0])
    sig = 0.45
    rng = np.random.default_rng(12)
    n = 500
    pts = rng.uniform(0.05, L - 0.05, size=(n, 3))
    w = rng.uniform(0.5, 2.0, n)
    det = np.array([[9.0, 2.1, 1.7], [-4.0, -3.0, 11.0], [3.0, 2.5, -500.0]])
    eng = _engine(c, t, n, det, np.zeros(3), np.full((1, len(t)), sig))
    _tally(eng, path, pts, w)
    got = eng.detector_results(0)[0, 0, 0]
    for d in range(3):
        u = det[d] - pts
        R = np.sqrt((u ** 2).sum(1))
        with np.errstate(divide="ignore"):
            s = np.where(u > 0, (L - pts) / u, np.where(u < 0, -pts / u, np.inf)).min(1)  # exit parameter
        want = math.fsum(w * np.exp(-sig * s * R) / (4 * math.pi * R ** 2))
        assert got[d] == pytest.approx(want, rel=1e-12), d
    assert eng.get_option("detector_rays") == 3 * n and eng.detector_hull_entries == 0


@pytest.mark.parametrize("path", PATHS)
def test_convex_box_all_inside_is_bit_for_bit_the_mode_off(path):
    """Every event and detector inside a convex box: each ray's score and the counters with the mode on equal those with
    it off bit for bit, and no ray enters through the hull.  One event per call, so that every slot holds one ray's score
    (the order of the aggregation's atomic additions is not fixed, and the two modes run in blocks of different size)."""
    c, t = kuhn_box(6, 5, 4)
    rng = np.random.default_rng(4)
    n, D = 40, 5
    pts = rng.uniform(0.05, [5.95, 4.95, 3.95], size=(n, 3))
    det = rng.uniform(0.3, [5.7, 4.7, 3.7], size=(D, 3))
    r0 = np.array([0.0, 0.3, 0.0, 1.0, 0.2])
    sigma = rng.uniform(0.1, 0.9, size=(1, len(t)))
    w = rng.uniform(0.5, 2.0, n)
    pdf = rng.uniform(0.0, 0.3, size=(n, D))
    res = []
    for on in (False, True):
        eng = PumiTally.from_arrays(c, t, 1)
        eng.set_detector_void(on)
        eng.set_point_detectors(det, r0)
        eng.set_detector_cross_sections(sigma)
        per_event = []
        for i in range(n):
            _tally(eng, path, pts[i:i + 1], w[i:i + 1], pdf=pdf[i:i + 1])
            per_event.append(eng.detector_results(0).copy())
        res.append((np.array(per_event), [eng.get_option(k) for k in COUNTERS if k] +
                    [eng.get_option("detector_crossings"), eng.detector_hull_entries]))
    assert np.array_equal(res[0][0], res[1][0])
    assert res[0][1] == res[1][1] and res[1][1][-1] == 0 and res[1][1][0] > 0


def test_refusals_switching_and_resets():
    c, t = MESHES["l_shape"]()
    n = 200
    wl = SyntheticWorkload(box=(8.0, 8.0, 2.0), num_particles=n, mean_length=1.0, seed=2)
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_collision_estimator(True)
    eng.set_batch_statistics(True)
    outside = np.array([[6.0, 6.0, 1.0], [2.0, 2.0, 1.0]])  # the first in the notch
    with pytest.raises(ValueError):
        eng.set_point_detectors(outside, np.zeros(2))  # the mode is off
    assert eng.point_detectors == 0 and not eng.detector_void
    eng.set_detector_void(True)
    eng.set_point_detectors(outside, np.zeros(2))
    with pytest.raises(ValueError):
        eng.set_point_detectors(np.array([[np.nan, 1.0, 1.0]]), np.zeros(1))
    eng.set_detector_cross_sections(np.full((1, len(t)), 0.3))
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    eng.MoveToNextLocation(o.copy(), d.copy(), f.copy(), w.copy())
    eng.tally_detectors(np.array([[1.0, 1.0, 1.0], [7.0, 3.0, 1.0]]), np.ones(2))
    eng.end_batch()
    eng.tally_detectors(np.array([[1.0, 1.0, 1.0]]), np.ones(1))
    assert eng.get_option("detector_rays") == 2

    def snapshot():
        return [eng.flux.copy(), eng.positions.copy(), eng.elem_ids.copy(), eng.collision_results(0).copy()]

    before = snapshot()
    with pytest.raises(ValueError):
        eng.set_detector_void(False)  # a detector lies outside the mesh
    assert eng.detector_void and eng.get_option("detector_rays") == 2
    eng.set_detector_void(True)  # the mode it has: nothing changes
    assert eng.get_option("detector_rays") == 2 and eng.detector_results(0).any()
    eng.set_point_detectors(np.array([[2.0, 2.0, 1.0]]), np.zeros(1))
    eng.tally_detectors(np.array([[6.0, 6.0, 1.0]]), np.ones(1))  # in the notch: its ray enters the mesh once
    assert eng.detector_hull_entries == 1 and eng.get_option("detector_events_outside") == 0
    eng.set_detector_void(False)  # switching resets the tally and discards the folded batches
    assert not eng.detector_void and eng.get_option("detector_void") == 0
    assert eng.get_option("detector_rays") == 0 and eng.detector_hull_entries == 0
    assert not eng.detector_results(0).any()
    assert eng.get_option("batches") == 0
    with pytest.raises(RuntimeError):
        eng.detector_results(1)
    with pytest.raises(ValueError):
        eng.set_detector_void(2)
    for a, b in zip(before, snapshot()):
        assert np.array_equal(a, b)
    # off: an event in the notch is outside again, and a ray across the notch is shadowed
    eng.set_point_detectors(np.array([[3.0, 7.0, 1.0]]), np.zeros(1))
    eng.tally_detectors(np.array([[6.0, 6.0, 1.0], [7.0, 3.0, 1.0]]), np.ones(2))
    assert eng.get_option("detector_events_outside") == 1 and eng.get_option("detector_rays_shadowed") == 1


def _checkpoint_engine(on, det=((1.0, 1.0, 1.0), (6.0, 6.0, 1.0)), r0=(0.0, 1.0)):
    c, t = MESHES["l_shape"]()
    eng = PumiTally.from_arrays(c, t, 64)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(2, 100.0)
    if on:
        eng.set_detector_void(True)
    eng.set_point_detectors(np.array(det), np.array(r0))
    eng.set_detector_cross_sections(np.full((1, len(t)), 0.2))
    return eng


def test_checkpoints_with_the_void(tmp_path):
    rng = np.random.default_rng(8)
    a = _checkpoint_engine(True)
    for _ in range(3):
        a.tally_detectors(rng.uniform(0.01, 7.99, size=(500, 3)) * [1, 1, 0.25], rng.uniform(0.5, 1.5, 500))
        a.end_batch()
    a.tally_detectors(rng.uniform(0.01, 7.99, size=(200, 3)) * [1, 1, 0.25], np.ones(200))
    path = str(tmp_path / "a.ckpt")
    a.save_checkpoint(path)
    assert open(path, "rb").read()[8:12] == (4).to_bytes(4, "little")
    names = [k for k in COUNTERS if k] + ["detector_crossings", "detector_hull_entries"]
    b = _checkpoint_engine(True)
    b.load_checkpoint(path)
    for k in range(4):
        assert np.array_equal(a.detector_results(k), b.detector_results(k)), k
    assert [a.get_option(k) for k in names] == [b.get_option(k) for k in names]
    assert b.detector_hull_entries > 0
    c = _checkpoint_engine(True)
    c.tally_detectors(rng.uniform(0.01, 7.99, size=(300, 3)) * [1, 1, 0.25], np.ones(300))
    c.end_batch()
    c.save_checkpoint(str(tmp_path / "c.ckpt"))
    d = _checkpoint_engine(True)
    d.tally_detectors(rng.uniform(0.01, 7.99, size=(300, 3)) * [1, 1, 0.25], np.ones(300))
    d.end_batch()
    mean_d = d.detector_results(1).copy()
    d.merge_checkpoint(str(tmp_path / "c.ckpt"))
    np.testing.assert_allclose(d.detector_results(1), 0.5 * (mean_d + c.detector_results(1)), rtol=1e-13)
    # across the two settings: refused, and the message names the detector void
    inside = ((1.0, 1.0, 1.0), (3.0, 2.0, 1.0))
    on, off = _checkpoint_engine(True, inside), _checkpoint_engine(False, inside)
    on.end_batch()
    off.end_batch()
    on.save_checkpoint(str(tmp_path / "on.ckpt"))
    off.save_checkpoint(str(tmp_path / "off.ckpt"))
    for eng, p in ((_checkpoint_engine(False, inside), "on.ckpt"), (_checkpoint_engine(True, inside), "off.ckpt")):
        for call in (eng.load_checkpoint, eng.merge_checkpoint):
            with pytest.raises(RuntimeError):
                call(str(tmp_path / p))


def test_switching_on_and_off_keeps_the_file_bytes(tmp_path):
    c, t = MESHES["l_shape"]()
    paths = []
    for k, switch in enumerate((False, True)):
        eng = PumiTally.from_arrays(c, t, 64)
        eng.set_batch_statistics(True)
        if switch:
            eng.set_detector_void(True)
        eng.set_point_detectors(np.array([[1.0, 1.0, 1.0]]), np.zeros(1))
        if switch:
            eng.set_detector_void(False)
        eng.set_detector_cross_sections(np.full((1, len(t)), 0.2))
        eng.tally_detectors(np.array([[2.0, 3.0, 1.0], [7.0, 2.0, 0.5]]), np.ones(2))
        eng.end_batch()
        eng.tally_detectors(np.array([[3.0, 3.0, 1.0]]), np.ones(1))
        p = str(tmp_path / f"{k}.ckpt")
        eng.save_checkpoint(p)
        paths.append(p)
    a, b = (open(p, "rb").read() for p in paths)
    assert a == b and a[8:12] == (3).to_bytes(4, "little")


def test_refused_checkpoint_message_names_the_void(tmp_path):
    """The refusal's message (on stderr) names the detector void."""
    script = f"""
import sys, numpy as np
sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
from locate_ref import MESHES
from pumiumtally_b200.tally import PumiTally
c, t = MESHES["l_shape"]()
def make(on):
    e = PumiTally.from_arrays(c, t, 64)
    e.set_batch_statistics(True)
    e.set_detector_void(on)
    e.set_point_detectors(np.array([[1.0, 1.0, 1.0]]), np.zeros(1))
    e.set_detector_cross_sections(np.full((1, len(t)), 0.2))
    return e
a = make(True); a.end_batch(); a.save_checkpoint({str(tmp_path / 'v.ckpt')!r})
b = make(False)
for call in (b.load_checkpoint, b.merge_checkpoint):
    try:
        call({str(tmp_path / 'v.ckpt')!r})
    except RuntimeError:
        print("REFUSED", flush=True)
"""
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=300)
    assert r.stdout.count("REFUSED") == 2, r.stdout + r.stderr
    assert r.stderr.count("detector void (set_detector_void)") == 2, r.stderr


@pytest.mark.parametrize("D", [8])
def test_config_c2_ten_million_events_detectors_outside(D):
    """Full-size c2 (convex): 10 M events at D detectors outside the box; no ray is lost or shadowed, and each detector's
    estimate is the exact uncollided sum over the events, exp(-Sigma l_inside) / (4 pi R^2)."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    cells = np.array(cfg["cells"], dtype=np.float64)
    n = 10_000_000
    rng = np.random.default_rng(D)
    u = rng.normal(size=(D, 3))
    det = 0.5 * cells + u / np.linalg.norm(u, axis=1)[:, None] * cells * rng.uniform(1.0, 3.0, (D, 1))
    sig = 0.05
    eng = _engine(coords, t2v, 16, det, np.zeros(D), np.full((1, len(t2v)), sig))
    g = torch.Generator(device="cuda").manual_seed(3)
    ct = torch.tensor(cells, device="cuda")
    pts = (torch.rand((n, 3), dtype=torch.float64, device="cuda", generator=g) * ct).contiguous()
    eng.tally_detectors_device(pts, torch.ones(n, dtype=torch.float64, device="cuda"))
    torch.cuda.synchronize()
    assert eng.get_option("detector_rays") == D * n
    assert eng.get_option("detector_rays_lost") == 0 and eng.get_option("detector_rays_shadowed") == 0
    got = eng.detector_results(0)[0, 0, 0]
    for d in range(D):
        dd = torch.tensor(det[d], device="cuda")
        v = dd - pts
        R = v.norm(dim=1)
        s = torch.where(v > 0, (ct - pts) / v, torch.where(v < 0, -pts / v, torch.full_like(v, math.inf))).min(1).values
        want = float((torch.exp(-sig * s * R) / (4 * math.pi * R * R)).sum())
        assert got[d] == pytest.approx(want, rel=1e-9), d


def test_carved_c2_cavity():
    """A c2-size box with a central cubic cavity, homogeneous Sigma: rays through the cavity lose its length, tau = Sigma
    (R - l_cavity); every ray is traced, and re-entries are counted."""
    import torch

    n_cells = CONFIGS["c2"]["cells"]
    c, t = kuhn_box(*n_cells)
    cen = c[t].mean(1)
    lo, hi = np.array([18.0, 18.0, 18.0]), np.array([37.0, 37.0, 37.0])
    c, t = carve(c, t, ~((cen > lo) & (cen < hi)).all(1))
    sig = 0.05
    D, n = 4, 1_000_000
    rng = np.random.default_rng(5)
    det = np.array([[27.5, 27.5, 27.5], [5.0, 27.0, 29.0], [50.0, 30.0, 20.0], [27.0, 2.0, 53.0]])
    eng = _engine(c, t, 16, det, np.zeros(D), np.full((1, len(t)), sig))
    pts = rng.uniform(0.0, 55.0, size=(n, 3))
    eng.tally_detectors_device(*_to_device(pts, np.ones(n)))
    torch.cuda.synchronize()
    cnt = {k: eng.get_option(k) for k in COUNTERS if k}
    assert cnt["detector_rays"] == D * n
    assert cnt["detector_rays_lost"] == cnt["detector_rays_shadowed"] == cnt["detector_events_outside"] == 0
    assert eng.detector_hull_entries > n
    got = eng.detector_results(0)[0, 0, 0]

    def clip_len(a, b, blo, bhi):
        u = b - a
        with np.errstate(divide="ignore", invalid="ignore"):
            t0 = np.where(u != 0, (blo - a) / u, np.where((a >= blo) & (a <= bhi), -np.inf, np.inf))
            t1 = np.where(u != 0, (bhi - a) / u, np.where((a >= blo) & (a <= bhi), np.inf, -np.inf))
        tin = np.clip(np.minimum(t0, t1).max(1), 0.0, 1.0)
        tout = np.clip(np.maximum(t0, t1).min(1), 0.0, 1.0)
        return np.maximum(tout - tin, 0.0) * np.sqrt((u ** 2).sum(1))

    box = np.array([55.0, 55.0, 55.0])
    for d in range(D):
        b = np.broadcast_to(det[d], pts.shape)
        R = np.sqrt(((b - pts) ** 2).sum(1))
        ell = clip_len(pts, b, np.zeros(3), box) - clip_len(pts, b, lo, hi)
        want = math.fsum(np.exp(-sig * ell) / (4 * math.pi * R ** 2))
        assert got[d] == pytest.approx(want, rel=1e-9), d
    # a subsample against the mesh-clipping reference
    sub = pts[:3]
    from detector_void_ref import reference_void as ref
    want, _ = ref(c, t, eng.locate(sub), sub, np.ones(3), None, None, None, None, None, None, 1, 1,
                  np.full((1, len(t)), sig), det[:2], np.zeros(2))
    e2 = _engine(c, t, 16, det[:2], np.zeros(2), np.full((1, len(t)), sig))
    e2.tally_detectors(sub, np.ones(3))
    np.testing.assert_allclose(e2.detector_results(0), want, rtol=1e-11)


def test_cxx_program_with_the_detector_void(tmp_path):
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "detector_void_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "detector_void_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "DETECTOR_VOID_OK" in out, out


def _two_gpu_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from locate_ref import MESHES as M
    from pumiumtally_b200.distributed import broadcast_unique_id

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    c, t = M["l_shape"]()
    eng = PumiTally.from_arrays(c, t, 100, device=rank)
    eng.set_batch_statistics(True)
    eng.set_detector_void(True)
    eng.set_point_detectors(np.array([[6.0, 6.0, 1.0], [1.0, 4.0, 1.0]]), np.array([0.5, 0.0]))
    eng.set_detector_cross_sections(np.full((1, eng.num_elements), 0.3))
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    refused = False
    try:
        eng.set_detector_void(False)
    except ValueError:
        refused = True
    rng = np.random.default_rng(rank)
    out = {"local": [], "allreduce": [], "refused": refused}
    for b in range(2):
        pts = rng.uniform(0.0, 8.0, (20_000, 3)) * [1, 1, 0.25]
        eng.tally_detectors(pts, rng.uniform(0.5, 1.5, 20_000))
        out["local"].append(eng.detector_results(0))
        eng.allreduce_tally()
        out["allreduce"].append(eng.detector_results(0))
        eng.end_batch()
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_exchange_with_the_void():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 53) % 1000
    procs = [ctx.Process(target=_two_gpu_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    a, b = res[0][1], res[1][1]
    assert a["refused"] and b["refused"]
    for got_a, got_b, la, lb in zip(a["allreduce"], b["allreduce"], a["local"], b["local"]):
        np.testing.assert_allclose(got_a, la + lb, rtol=1e-13)
        np.testing.assert_allclose(got_b, la + lb, rtol=1e-13)
