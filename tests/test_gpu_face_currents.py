"""Face currents (pumitally_set_face_currents): every crossing of the tally phase adds the particle's weight to the
outgoing current of the face it leaves through, which is the incoming current of the neighbour's face.  Weights are
dyadic (k / 8), so every sum is exact in any order and the comparisons are bit for bit."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from face_currents_ref import back_faces, face_walk, reference_currents, unit_planes
from helpers import ROOT, box_case, l_shaped_mesh
from pumiumtally_b200.mesh import delaunay_box, kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_scores import _bins, engine

pytestmark = pytest.mark.gpu

EDGES = np.linspace(0.0, 4.0, 9)
KINDS = ["plain", "binned", "scored", "timed", "moment"]


def _configure(eng, kind, currents=True):
    if kind == "moment":
        eng.set_moments(1)
    if kind in ("binned", "scored", "timed"):
        eng.set_score_bins(3)
    if kind == "scored":
        eng.set_scores(2)
    if kind == "timed":
        eng.set_time_bins(EDGES)
    if currents:
        eng.set_face_currents(True)


def _move(eng, kind, o, d, f, w, extra, device):
    bins, r, times, speeds = extra
    if device:
        import torch

        keep = []

        def t(x):  # a device copy, kept alive until the move has run
            if x is None:
                return None
            keep.append(torch.as_tensor(np.ascontiguousarray(x)).cuda())
            return keep[-1].data_ptr()

        args = (t(o.reshape(-1)), t(d.reshape(-1)), t(f), t(w))
        if kind == "timed":
            eng.move_device_timed(*args, t(times), t(speeds), t(r), t(bins))
        elif kind == "scored":
            eng.move_device_scored(*args, t(r), t(bins))
        elif kind == "binned":
            eng.move_device_binned(*args, t(bins))
        else:
            eng.move_device(*args)
        torch.cuda.synchronize()
        eng.synchronize()
        return
    args = (o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
    if kind == "timed":
        eng.MoveToNextLocationTimed(*args, times, speeds, r, bins)
    elif kind == "scored":
        eng.MoveToNextLocationScored(*args, r, bins)
    elif kind == "binned":
        eng.MoveToNextLocationBinned(*args, bins)
    else:
        eng.MoveToNextLocation(*args)


def _interior_points(rng, coords, t2v, n):
    lam = rng.dirichlet(np.ones(4), n)
    lam = 0.02 + 0.92 * lam  # clear of every face
    lam /= lam.sum(axis=1, keepdims=True)
    tets = rng.integers(0, len(t2v), n)
    return np.ascontiguousarray(np.einsum("iq,iqk->ik", lam, coords[t2v[tets]]))


def _run(coords, t2v, n, kind, variant, device, steps=2, seed=0, twin=True):
    """Moves with currents on against the exact reference, and against a twin engine with currents off."""
    rng = np.random.default_rng(seed)
    eng = engine(coords, t2v, n, variant)
    _configure(eng, kind)
    other = engine(coords, t2v, n, variant) if twin else None
    if other:
        _configure(other, kind, currents=False)
    adj = eng.adjacency
    planes = unit_planes(coords, t2v)
    ntime, nbins = (len(EDGES) - 1 if kind == "timed" else 1), eng.score_bins
    want_out = np.zeros((ntime, nbins, len(t2v), 4))
    want_in = np.zeros_like(want_out)
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    init = _interior_points(rng, coords, t2v, n)
    for e in (eng, other) if other else (eng,):
        e.CopyInitialPosition(init.reshape(-1).copy())
    for step in range(steps):
        o = _interior_points(rng, coords, t2v, n)
        w = rng.integers(1, 17, n) / 8.0
        r = np.ascontiguousarray(rng.uniform(0.0, 2.0, (n, eng.scores)))
        bins = _bins(n, nbins, step) if nbins > 1 else None
        ones = np.ones(n, dtype=np.int8)
        extra0 = (bins, r, np.zeros(n), np.ones(n))
        # positioning move: relocation to o, then a flight of length zero.  Weight 0: a relocation that stops on the
        # hull (non-convex mesh) is followed by a flight from there that may cross faces on its way back to o.
        for e in (eng, other) if other else (eng,):
            _move(e, kind, o, o, ones, np.zeros(n), extra0, device)
        ok = (eng.positions == o).all(axis=1)
        start = eng.elem_ids.astype(np.int64)
        u = rng.normal(size=(n, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        d = o + u * rng.exponential(0.6 * (hi - lo).max(), n)[:, None]
        times = rng.uniform(EDGES[0] - 1.0, EDGES[-1] + 0.5, n)
        speeds = rng.uniform(0.3, 3.0, n)
        tpp = np.linalg.norm(d - o, axis=1) / speeds
        fly0 = ok & (rng.random(n) < 0.9)
        cr = face_walk(planes, adj, start, o, d, fly0, times, tpp, EDGES if kind == "timed" else None)
        fly = (fly0 & ~cr[4]).astype(np.int8)
        cr = face_walk(planes, adj, start, o, d, fly.astype(bool), times, tpp, EDGES if kind == "timed" else None)
        assert not cr[4][fly.astype(bool)].any()
        extra = (bins, r, times, speeds)
        for e in (eng, other) if other else (eng,):
            _move(e, kind, o, d, fly, w, extra, device)
        a, b = reference_currents(adj, cr, w, bins, ntime, nbins)
        want_out += a
        want_in += b
    got_out, got_in = eng.face_current_results(0), eng.face_current_results(1)
    np.testing.assert_array_equal(got_out, want_out, err_msg=f"{kind} v{variant} outgoing")
    np.testing.assert_array_equal(got_in, want_in, err_msg=f"{kind} v{variant} incoming")
    hull = adj < 0
    np.testing.assert_array_equal(eng.leakage(0), (want_out * hull).sum(axis=(2, 3)))
    if other:
        np.testing.assert_array_equal(eng.elem_ids, other.elem_ids)
        np.testing.assert_array_equal(eng.positions, other.positions)
        fa, fb = eng.flux_time, other.flux_time
        np.testing.assert_allclose(fa, fb, rtol=1e-12, atol=1e-14 * np.abs(fb).max())
    return eng, adj


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("variant", [-1, 0, 8, 16, 24])
def test_currents_match_the_exact_reference(variant, kind):
    coords, t2v, _ = box_case((6, 6, 5), 1)
    _run(coords, t2v, 6000, kind, variant, device=False, seed=10 + variant + 7 * KINDS.index(kind))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("variant", [0, 8, 16, 24])
def test_device_moves_match_the_exact_reference(variant, kind):
    coords, t2v, _ = box_case((5, 6, 4), 1)
    _run(coords, t2v, 5000, kind, variant, device=True, seed=100 + variant + 7 * KINDS.index(kind))


@pytest.mark.parametrize("variant", [0, 8, 24])
def test_non_convex_mesh(variant):
    coords, t2v = l_shaped_mesh(6, 6, 3)
    _run(coords, t2v, 4000, "plain", variant, device=False, seed=3)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("variant", [0, 8, 16, 24])
def test_delaunay_mesh(variant, kind):
    """Irregular local vertex order: the face numbering and the neighbours' `back` indices of an unstructured mesh."""
    coords, t2v = delaunay_box(600)
    _run(coords, t2v, 4000, kind, variant, device=False, seed=200 + variant + 7 * KINDS.index(kind))


def test_incoming_is_the_neighbours_outgoing():
    coords, t2v, _ = box_case((6, 6, 5), 1)
    eng, adj = _run(coords, t2v, 8000, "binned", 8, device=False, seed=11, twin=False)
    out, inn = eng.face_current_results(0), eng.face_current_results(1)
    back = back_faces(adj)
    e, f = np.nonzero(adj >= 0)
    np.testing.assert_array_equal(inn[:, :, e, f], out[:, :, adj[e, f], back[e, f]])
    np.testing.assert_array_equal(inn[:, :, adj < 0], 0.0)


def test_balance_and_leakage_on_c2():
    """Full-size c2: per element, sum of incoming - outgoing = weight of the flights that reached their destination
    there - weight of the flights that started there; the leakage is the weight of the flights stopped on the hull."""
    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    wl = SyntheticWorkload(cfg["cells"], cfg["particles"], mean_length=cfg["mean_length"], mu_min=cfg["mu_min"])
    eng = engine(coords, t2v, wl.n)
    eng.set_face_currents(True)
    E = len(t2v)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    rng = np.random.default_rng(5)
    net = np.zeros(E)
    leak = 0.0
    for step in range(3):
        o, d, f, _ = wl.next_step()
        w = rng.integers(1, 17, wl.n) / 8.0
        ones = np.ones(wl.n, dtype=np.int8)
        # positioning, weight 0: an origin outside the box ends its relocation on the hull and then flies out of it
        eng.MoveToNextLocation(o.reshape(-1).copy(), o.reshape(-1).copy(), ones, np.zeros(wl.n))
        ok = (eng.positions == o).all(axis=1)
        start = eng.elem_ids.copy()
        fly = (f.astype(bool) & ok).astype(np.int8)
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), fly.copy(), w.copy())
        pos, end = eng.positions, eng.elem_ids
        flew = fly.astype(bool)
        reached = flew & (pos == d).all(axis=1)
        stopped = flew & ~reached
        net += np.bincount(end[reached], weights=w[reached], minlength=E)
        net -= np.bincount(start[flew], weights=w[flew], minlength=E)
        leak += w[stopped].sum()
    out, inn = eng.face_current_results(0)[0, 0], eng.face_current_results(1)[0, 0]
    np.testing.assert_array_equal(inn.sum(axis=1) - out.sum(axis=1), net)
    assert eng.leakage(0)[0, 0] == leak
    assert eng.stats()["lost"] == 0


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_batch_statistics(mode):
    coords, t2v, _ = box_case((5, 5, 4), 1)
    n = 3000
    eng = engine(coords, t2v, n, 8)
    eng.set_score_bins(2)
    eng.set_face_currents(True)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(mode, 3.0 if mode == 2 else 1.0)
    rng = np.random.default_rng(mode)
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
    vals = {0: [], 1: [], "leak": []}
    for b in range(8):
        o = eng.positions
        u = rng.normal(size=(n, 3))
        d = o + u * rng.uniform(0.2, 3.0, (n, 1))
        w = rng.integers(1, 17, n) / 8.0
        bins = _bins(n, 2, b)
        eng.MoveToNextLocationBinned(o.reshape(-1).copy(), d.reshape(-1).copy(), np.ones(n, np.int8), w, bins)
        vals[0].append(eng.face_current_results(0))
        vals[1].append(eng.face_current_results(1))
        vals["leak"].append(eng.leakage(0))
        eng.end_batch()
    for key, got in ((0, lambda k: eng.face_current_results(0, k)), (1, lambda k: eng.face_current_results(1, k)),
                     ("leak", eng.leakage)):
        x = np.stack(vals[key])
        mean, se = x.mean(axis=0), x.std(axis=0, ddof=1) / np.sqrt(len(x))
        scale = np.abs(x).max() + 1e-300
        np.testing.assert_allclose(got(1), mean, rtol=1e-13, atol=1e-14 * scale)
        np.testing.assert_allclose(got(2), se, rtol=1e-9, atol=1e-12 * scale)
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = np.where(mean != 0, se / np.abs(mean), 0.0)
        np.testing.assert_allclose(got(3), rel, rtol=1e-8, atol=1e-12)


def test_checkpoint_round_trip_merge_and_refusals(tmp_path, capfd):
    coords, t2v, _ = box_case((5, 5, 4), 1)
    n = 3000

    def make(currents):
        e = engine(coords, t2v, n, 8)
        e.set_face_currents(currents)
        e.set_batch_statistics(True)
        e.CopyInitialPosition(init.reshape(-1).copy())
        return e

    rng = np.random.default_rng(9)
    init = _interior_points(rng, coords, t2v, n)
    eng = make(True)
    for b in range(3):
        o = eng.positions
        d = o + rng.normal(size=(n, 3))
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), np.ones(n, np.int8),
                               rng.integers(1, 17, n) / 8.0)
        if b < 2:
            eng.end_batch()
    p = str(tmp_path / "a.ckpt")
    eng.save_checkpoint(p)
    loaded = make(True)
    loaded.load_checkpoint(p)
    for k in range(4):
        if k > 0:
            for dr in (0, 1):
                np.testing.assert_array_equal(loaded.face_current_results(dr, k), eng.face_current_results(dr, k))
            np.testing.assert_array_equal(loaded.leakage(k), eng.leakage(k))
    np.testing.assert_array_equal(loaded.face_current_results(0, 0), eng.face_current_results(0, 0))
    p2 = str(tmp_path / "b.ckpt")
    loaded.save_checkpoint(p2)
    assert open(p, "rb").read() == open(p2, "rb").read()
    # merge a batch-end checkpoint into a fresh engine: the same statistics
    eng.end_batch()
    p3 = str(tmp_path / "c.ckpt")
    eng.save_checkpoint(p3)
    merged = make(True)
    merged.merge_checkpoint(p3)
    np.testing.assert_array_equal(merged.face_current_results(0, 1), eng.face_current_results(0, 1))
    np.testing.assert_array_equal(merged.leakage(2), eng.leakage(2))
    # the other currents setting is refused in both directions, with a message that names it, and nothing changes
    off = make(False)
    capfd.readouterr()
    with pytest.raises(RuntimeError):
        off.load_checkpoint(p3)
    assert "face currents differ: the checkpoint was saved with them on" in capfd.readouterr().err
    p4 = str(tmp_path / "d.ckpt")
    off.end_batch()
    off.save_checkpoint(p4)
    before = merged.face_current_results(0, 1)
    capfd.readouterr()
    with pytest.raises(RuntimeError):
        merged.load_checkpoint(p4)
    assert "face currents differ: the checkpoint was saved with them off" in capfd.readouterr().err
    with pytest.raises(RuntimeError):
        merged.merge_checkpoint(p4)
    assert "face currents differ: the checkpoint was saved with them off" in capfd.readouterr().err
    np.testing.assert_array_equal(merged.face_current_results(0, 1), before)


def test_refusals_change_nothing():
    coords, t2v, _ = box_case((4, 4, 4), 1)
    n = 2000
    eng = engine(coords, t2v, n, 8)
    with pytest.raises(Exception):
        eng.face_current_results(0)  # currents off
    with pytest.raises(Exception):
        eng.leakage(0)
    with pytest.raises(ValueError):
        eng.set_face_currents(2)
    assert not eng.face_currents and eng.get_option("face_currents") == 0
    eng.set_face_currents(True)
    assert eng.face_currents
    rng = np.random.default_rng(1)
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
    o = eng.positions
    eng.MoveToNextLocation(o.reshape(-1).copy(), (o + rng.normal(size=(n, 3))).reshape(-1).copy(),
                           np.ones(n, np.int8), rng.integers(1, 17, n) / 8.0)
    before = eng.face_current_results(0)
    for args in ((2, 0), (0, 4), (0, -1), (0, 1), (1, 2), (0, 3)):  # bad direction or kind; batch kinds without stats
        with pytest.raises(Exception):
            eng.face_current_results(*args)
    with pytest.raises(Exception):
        eng.leakage(1)
    from pumiumtally_b200.tally import _dp

    bad = np.empty(before.size - 1)
    assert eng._L.pumitally_get_face_current_results(eng._h, 0, 0, bad.ctypes.data_as(_dp), bad.size) != 0
    assert eng._L.pumitally_get_leakage(eng._h, 0, bad.ctypes.data_as(_dp), 2) != 0
    np.testing.assert_array_equal(eng.face_current_results(0), before)


def test_vtk_arrays(tmp_path):
    coords, t2v, _ = box_case((4, 4, 3), 1)
    n = 2000
    paths = {}
    for on in (False, True):
        eng = engine(coords, t2v, n, 8)
        if on:
            eng.set_face_currents(True)
        rng = np.random.default_rng(2)
        eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
        o = eng.positions
        eng.MoveToNextLocation(o.reshape(-1).copy(), (o + rng.normal(size=(n, 3))).reshape(-1).copy(),
                               np.ones(n, np.int8), rng.integers(1, 17, n) / 8.0)
        paths[on] = str(tmp_path / f"r{int(on)}.vtu")
        eng.WriteTallyResults(paths[on])
    with open(os.path.join(paths[True], "pieces", "piece_0.vtu"), "rb") as f:
        text = f.read()
    assert b'Name="current_out" NumberOfComponents="4"' in text
    assert b'Name="current_in" NumberOfComponents="4"' in text
    with open(os.path.join(paths[False], "pieces", "piece_0.vtu"), "rb") as f:
        assert b"current_out" not in f.read()


@pytest.mark.skipif(shutil.which("cmake") is None or shutil.which("ninja") is None, reason="cmake/ninja not available")
def test_cxx_program_against_the_installed_package(tmp_path):
    """A C++ caller of SetFaceCurrents, GetFaceCurrentResults and GetLeakage (tests/currents_demo.cpp), built with
    find_package(pumitally) against the installed CMake package and run."""
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
        f"add_executable(app {os.path.join(ROOT, 'tests', 'currents_demo.cpp')})\n"
        "target_compile_features(app PRIVATE cxx_std_17)\n"
        "target_link_libraries(app PRIVATE pumitally::pumitally)\n")
    appb = tmp_path / "appbuild"
    appb.mkdir()
    subprocess.check_call(["cmake", *common, f"-DCMAKE_PREFIX_PATH={inst}", str(app)], cwd=appb,
                          stdout=subprocess.DEVNULL)
    subprocess.check_call(["ninja"], cwd=appb, stdout=subprocess.DEVNULL)
    out = subprocess.check_output([str(appb / "app")], cwd=str(tmp_path), text=True)
    assert "FACE_CURRENTS_OK" in out, out


def _two_gpu_currents(eng, c, t, rank, world, n):
    """Two batches; rank r flies particles r, r + world, ... of one fixed set of n (every rank holds n // world)."""
    rng = np.random.default_rng(77)
    init = _interior_points(rng, c, t, n)
    mine = slice(rank, n, world)
    eng.CopyInitialPosition(init[mine].reshape(-1).copy())
    for _ in range(2):
        o = _interior_points(rng, c, t, n)
        d = o + rng.normal(size=(n, 3)) * 1.5
        w = rng.integers(1, 17, n) / 8.0
        bins = (np.arange(n) % 3 - 1).astype(np.int32)  # -1: outside [0, 2), adds nothing
        m = len(init[mine])
        eng.MoveToNextLocationBinned(o[mine].reshape(-1).copy(), d[mine].reshape(-1).copy(), np.ones(m, np.int8),
                                     w[mine].copy(), bins[mine].copy())
        eng.end_batch()
    return [eng.face_current_results(dr, k) for dr in (0, 1) for k in (1, 2)] + [eng.leakage(1), eng.leakage(2)]


def _two_gpu_currents_worker(rank, world, port, q):
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
    eng.set_score_bins(2)
    eng.set_face_currents(True)
    eng.set_batch_statistics(True)
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    q.put((rank, _two_gpu_currents(eng, c, t, rank, world, 2000)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpus_give_the_one_rank_currents():
    """The batch-end exchange carries the currents: leakage summed per rank before the reduce-scatter, the rank shares
    cutting through the current block, and the statistics gathered from every rank's share at readout."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 311) % 1000
    procs = [ctx.Process(target=_two_gpu_currents_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    c, t = kuhn_box(5, 5, 5)
    one = PumiTally.from_arrays(c, t, 2000)
    one.set_score_bins(2)
    one.set_face_currents(True)
    one.set_batch_statistics(True)
    want = _two_gpu_currents(one, c, t, 0, 1, 2000)
    for rank in range(2):
        for got, w in zip(res[rank][1], want):
            # dyadic weights: every sum is exact, so the means are the same bits; the errors agree to rounding
            np.testing.assert_allclose(got, w, rtol=1e-12, atol=0.0, err_msg=f"rank {rank}")
        np.testing.assert_array_equal(res[rank][1][0], want[0])
        np.testing.assert_array_equal(res[rank][1][4], want[4])
