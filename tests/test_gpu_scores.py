"""Scores: several responses per track tallied in one walk (pumitally_set_scores).  A scored move must
give, score by score, what a plain engine moved with weights w * r[:, k] gives, and move the particles
exactly as a plain move does."""
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

pytestmark = pytest.mark.gpu


def engine(coords, t2v, n, variant=-1, **opts):
    e = PumiTally.from_arrays(coords, t2v, n)
    e.set_option("variant", variant)
    for k, v in opts.items():
        e.set_option(k, v)
    return e


def responses(rng, n, nscores, low=0.0):
    """In [low, 2] with exact zeros and ones."""
    r = rng.uniform(low, 2.0, (n, nscores))
    r[rng.random((n, nscores)) < 0.1] = 0.0
    r[rng.random((n, nscores)) < 0.1] = 1.0
    return np.ascontiguousarray(r)


def assert_scores_equal(got, want, label):
    """rtol 1e-12 plus a floor of 1e-15 of the total (the summation order of the reductions differs)."""
    got, want = np.asarray(got), np.asarray(want)
    tol = 1e-12 * np.abs(want) + 1e-15 * np.abs(want).sum()
    bad = np.abs(got - want) > tol
    assert not bad.any(), f"{label}: {int(bad.sum())} of {bad.size} elements differ"


def assert_same_particles(a, b, label=""):
    np.testing.assert_array_equal(a.elem_ids, b.elem_ids, err_msg=label)
    np.testing.assert_array_equal(a.positions, b.positions, err_msg=label)
    sa, sb = a.stats(), b.stats()
    for k in ("segments", "tracks", "relocations", "lost", "moves"):
        assert sa[k] == sb[k], (label, k, sa[k], sb[k])


@pytest.mark.parametrize("nscores", [2, 3, 8])
@pytest.mark.parametrize("variant", [-1, 0, 8, 16, 24])
def test_scores_equal_separate_plain_engines(variant, nscores):
    coords, t2v, wl = box_case((6, 6, 5), 12_000, mean_length=2.0)
    rng = np.random.default_rng(100 * nscores + variant)
    eng = engine(coords, t2v, wl.n, variant)
    eng.set_scores(nscores)
    assert eng.scores == nscores and eng.get_option("scores") == nscores
    plains = [engine(coords, t2v, wl.n, variant) for _ in range(nscores)]
    init = wl.initial_positions()
    for e in [eng] + plains:
        e.CopyInitialPosition(init.reshape(-1).copy())
    for step in range(3):  # the workload re-sources particles from move to move
        o, d, f, w = wl.next_step()
        r = responses(rng, wl.n, nscores)
        f1 = f.copy()
        eng.MoveToNextLocationScored(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy(), r)
        assert not f1.any(), "flying[] must be zeroed on return"
        for k, p in enumerate(plains):
            p.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w * r[:, k])
        fs = eng.flux_scores
        assert fs.shape == (1, nscores, len(t2v))
        for k, p in enumerate(plains):
            assert_scores_equal(fs[0, k], p.flux, f"variant {variant} score {k} step {step}")
        assert_same_particles(eng, plains[0], f"variant {variant} step {step}")
    if variant in (8, 16, 24):
        assert eng.get_option("walk_blocks_per_sm") == plains[0].get_option("walk_blocks_per_sm") > 0


def test_negative_responses_against_the_oracle():
    coords, t2v, wl = box_case((5, 5, 5), 6000)
    nscores = 3
    rng = np.random.default_rng(7)
    eng = engine(coords, t2v, wl.n)
    eng.set_scores(nscores)
    orcs = [OraclePumiTally(coords, t2v, wl.n) for _ in range(nscores)]
    init = wl.initial_positions()
    for e in [eng] + orcs:
        e.CopyInitialPosition(init.reshape(-1).copy())
    for step in range(2):
        o, d, f, w = wl.next_step()
        r = responses(rng, wl.n, nscores, low=-1.5)
        eng.MoveToNextLocationScored(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy(), r)
        for k, orc in enumerate(orcs):
            orc.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w * r[:, k])
    fs = eng.flux_scores[0]
    for k, orc in enumerate(orcs):
        assert_flux_close(fs[k], orc.flux, f"score {k}")
    np.testing.assert_array_equal(eng.elem_ids, orcs[0].elem_ids)


def test_one_score_is_the_plain_move_with_weights_times_responses():
    coords, t2v, wl = box_case((5, 5, 5), 8000)
    rng = np.random.default_rng(1)
    eng, plain = engine(coords, t2v, wl.n), engine(coords, t2v, wl.n)
    eng.set_scores(1)
    init = wl.initial_positions()
    for e in (eng, plain):
        e.CopyInitialPosition(init.reshape(-1).copy())
    for _ in range(2):
        o, d, f, w = wl.next_step()
        r = responses(rng, wl.n, 1)
        eng.MoveToNextLocationScored(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy(), r)
        plain.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w * r[:, 0])
    assert_scores_equal(eng.flux, plain.flux, "one score")
    assert_same_particles(eng, plain)


def test_config_c2_full_size_four_scores_on_the_default_kernel():
    """BASELINE configs[1] (998,250 tets, 10 M particles), device-resident moves on the default kernel (binned
    on an H100): four scores in one walk against four plain engines."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n, nscores = cfg["particles"], 4
    wl = SyntheticWorkload(box=tuple(float(c) for c in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    eng = PumiTally.from_arrays(coords, t2v, n)
    eng.set_scores(nscores)
    plains = [PumiTally.from_arrays(coords, t2v, n) for _ in range(nscores)]
    s = torch.cuda.current_stream().cuda_stream
    init = wl.initial_positions().contiguous()
    for e in [eng] + plains:
        e.copy_initial_position_device(init.data_ptr(), s)
    g = torch.Generator(device="cuda").manual_seed(5)
    for step in range(2):
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        r = torch.rand((n, nscores), dtype=torch.float64, device="cuda", generator=g) * 2.0
        r[r < 0.2] = 0.0
        r[(r > 1.0) & (r < 1.2)] = 1.0
        r = r.contiguous()
        eng.move_device_scored(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), r.data_ptr(), None, s)
        for k, p in enumerate(plains):
            wk = (w * r[:, k]).contiguous()
            p.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), wk.data_ptr(), s)
            torch.cuda.synchronize()
    assert eng.get_option("variant") == plains[0].get_option("variant")
    fs = eng.flux_scores[0]
    for k, p in enumerate(plains):
        assert_scores_equal(fs[k], p.flux, f"c2 score {k}")
    assert_same_particles(eng, plains[0], "c2")
    assert eng.stats()["lost"] == 0


def _bins(n, nbins, step):
    b = (np.arange(n) * 7 + step) % (nbins + 1)
    b[b == nbins] = -1  # a bin outside [0, nbins): flies unscored
    return b.astype(np.int32)


@pytest.mark.parametrize("path", ["staged", "direct", "registered", "device"])
def test_bins_times_scores_on_every_upload_path(path):
    import torch

    nbins, nscores = 3, 3
    coords, t2v, wl = box_case((5, 5, 5), 15_000)
    rng = np.random.default_rng(4)
    opts = {"staged": {}, "direct": {"host_path": 0, "chunk": 4096}, "registered": {"host_path": 0, "register_host": 1},
            "device": {}}[path]
    eng = engine(coords, t2v, wl.n, **opts)
    eng.set_scores(nscores)
    eng.set_score_bins(nbins)  # either order
    assert eng.scores == nscores and eng.score_bins == nbins
    plains = [engine(coords, t2v, wl.n) for _ in range(nscores)]
    for p in plains:
        p.set_score_bins(nbins)
    init = wl.initial_positions()
    for e in [eng] + plains:
        e.CopyInitialPosition(init.reshape(-1).copy())
    s = torch.cuda.current_stream().cuda_stream
    # the same arrays every move (register_host pins the caller's buffers once)
    o_buf, d_buf, w_buf = np.empty(3 * wl.n), np.empty(3 * wl.n), np.empty(wl.n)
    r_buf, b_buf, f_buf = np.empty((wl.n, nscores)), np.empty(wl.n, dtype=np.int32), np.empty(wl.n, dtype=np.int8)
    h2d = 0.0
    for step in range(3):
        o, d, f, w = wl.next_step()
        o_buf[:], d_buf[:], w_buf[:] = o.reshape(-1), d.reshape(-1), w
        r_buf[:], b_buf[:] = responses(rng, wl.n, nscores), _bins(wl.n, nbins, step)
        if path == "device":
            t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (o_buf, d_buf, f, w_buf, r_buf, b_buf)]
            eng.move_device_scored(*(x.data_ptr() for x in t), s)
            torch.cuda.synchronize()
        else:
            before = eng.stats()["h2d_bytes"]
            f_buf[:] = f
            eng.MoveToNextLocationScored(o_buf, d_buf, f_buf, w_buf, r_buf, b_buf)
            h2d = eng.stats()["h2d_bytes"] - before
        for k, p in enumerate(plains):
            p.MoveToNextLocationBinned(o_buf.copy(), d_buf.copy(), f.copy(), w_buf * r_buf[:, k], b_buf.copy())
    if path != "device":
        assert h2d >= 8.0 * nscores * wl.n + 4.0 * wl.n  # the responses and the bins travel too
    fs = eng.flux_scores
    assert fs.shape == (nbins, nscores, len(t2v))
    for k, p in enumerate(plains):
        fb = p.flux_bins
        for b in range(nbins):
            assert_scores_equal(fs[b, k], fb[b], f"{path} bin {b} score {k}")
    np.testing.assert_array_equal(eng.elem_ids, plains[0].elem_ids)
    np.testing.assert_array_equal(eng.positions, plains[0].positions)


def test_accessors_normalisation_reset_and_vtk(tmp_path):
    import torch
    from vtk_reader import read_vtu_cell_data

    nbins, nscores = 2, 3
    coords, t2v, wl = box_case((4, 4, 4), 5000)
    E = len(t2v)
    rng = np.random.default_rng(9)
    eng = engine(coords, t2v, wl.n)
    eng.set_score_bins(nbins)
    eng.set_scores(nscores)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    r = responses(rng, wl.n, nscores)
    eng.MoveToNextLocationScored(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy(), r, _bins(wl.n, nbins, 0))
    fs = eng.flux_scores
    assert fs[:, 1:].any()
    np.testing.assert_array_equal(eng.flux, fs[0, 0])  # n = E: bin 0, score 0
    wrong = np.empty(nbins * E)  # with scores, n is E or nbins * nscores * E
    assert eng._L.pumitally_get_flux(eng._h, wrong.ctypes.data_as(C.POINTER(C.c_double)), wrong.size) != 0
    assert eng._L.pumitally_get_normalized_flux(eng._h, wrong.ctypes.data_as(C.POINTER(C.c_double)), None, wrong.size) != 0
    d_out = torch.empty(nbins * nscores * E, dtype=torch.float64, device="cuda")
    eng.get_flux_device(d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(d_out.cpu().numpy().reshape(nbins, nscores, E), fs)
    # normalisation: every score alike; mode 3 divides by the weights of the first tracks, not the responses
    for mode, value in ((0, 1.0), (1, 1.0), (2, 123.0), (3, 1.0)):
        eng.set_source_normalization(mode, value)
        nf, vol = eng.normalized_flux_scores()
        per = eng.source_normalization()
        if mode == 3:
            np.testing.assert_allclose(per, w[f == 1].sum(), rtol=1e-12)
        np.testing.assert_allclose(nf, fs / vol / per, rtol=1e-14)
        f0, v0 = eng.normalized_flux()
        np.testing.assert_array_equal(f0, nf[0, 0])
    eng.set_source_normalization(0)
    nf, vol = eng.normalized_flux_scores()
    out = str(tmp_path / "scores.vtk")
    eng.WriteTallyResults(out)
    cells = read_vtu_cell_data(os.path.join(out, "pieces", "piece_0.vtu"))
    np.testing.assert_allclose(cells["flux"], nf[:, 0].sum(axis=0), rtol=1e-14)
    for b in range(nbins):
        np.testing.assert_array_equal(cells[f"flux_bin{b}"], nf[b, 0])
    for k in range(1, nscores):
        np.testing.assert_allclose(cells[f"score{k}"], nf[:, k].sum(axis=0), rtol=1e-14)
        for b in range(nbins):
            np.testing.assert_array_equal(cells[f"score{k}_bin{b}"], nf[b, k])
    assert f"score{nscores}" not in cells
    eng.reset_tally()
    assert not eng.flux_scores.any()


def test_refusals_touch_nothing():
    import torch

    coords, t2v, wl = box_case((4, 4, 4), 2000)
    eng = engine(coords, t2v, wl.n)
    for bad in (0, 9, -1):
        with pytest.raises(ValueError):
            eng.set_scores(bad)
        assert eng.scores == 1
    eng.set_scores(2)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    o, d, f, w = wl.next_step()
    elems, pos, stats = eng.elem_ids, eng.positions, eng.stats()
    f1 = f.copy()
    with pytest.raises(RuntimeError):
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy())
    np.testing.assert_array_equal(f1, f)  # flying[] untouched
    eng.set_score_bins(2)
    with pytest.raises(RuntimeError):
        eng.MoveToNextLocationBinned(o.reshape(-1).copy(), d.reshape(-1).copy(), f1, w.copy(), _bins(wl.n, 2, 0))
    np.testing.assert_array_equal(f1, f)
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (o, d, f, w, _bins(wl.n, 2, 0))]
    s = torch.cuda.current_stream().cuda_stream
    with pytest.raises(RuntimeError):
        eng.move_device(*(x.data_ptr() for x in t[:4]), s)
    with pytest.raises(RuntimeError):
        eng.move_device_binned(*(x.data_ptr() for x in t), s)
    with pytest.raises(RuntimeError):  # NULL responses
        eng.move_device_scored(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), None, None, s)
    dp = C.POINTER(C.c_double)
    o1, d1 = o.reshape(-1).copy(), d.reshape(-1).copy()
    rc = eng._L.pumitally_move_to_next_location_scored(eng._h, o1.ctypes.data_as(dp), d1.ctypes.data_as(dp),
                                                       f1.ctypes.data_as(C.POINTER(C.c_int8)), w.ctypes.data_as(dp),
                                                       None, None, 3 * wl.n)
    assert rc != 0
    np.testing.assert_array_equal(f1, f)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(eng.elem_ids, elems)
    np.testing.assert_array_equal(eng.positions, pos)
    assert eng.stats()["segments"] == stats["segments"] and not eng.flux_scores.any()


def test_non_finite_responses_do_not_poison_the_tally_or_the_state():
    coords, t2v, wl = box_case((6, 6, 5), 4000)
    nscores = 3
    rng = np.random.default_rng(2)
    eng = engine(coords, t2v, wl.n)
    eng.set_scores(nscores)
    plains = [engine(coords, t2v, wl.n) for _ in range(nscores)]
    init = wl.initial_positions()
    for e in [eng] + plains:
        e.CopyInitialPosition(init.reshape(-1).copy())
    o, d, f, w = wl.next_step()
    f[:] = 1
    r = responses(rng, wl.n, nscores)
    bad = np.arange(10, 70)
    r[bad[:20], 0] = np.nan
    r[bad[20:40], 2] = np.inf
    r[bad[40:], 1] = -np.inf
    eng.MoveToNextLocationScored(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy(), r)
    # a plain engine treats the non-finite weight w * r exactly so: zero-length flight, counted as lost
    wk_all_bad = np.where(np.isfinite(r).all(axis=1), 1.0, np.nan)
    for k, p in enumerate(plains):
        p.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), np.nan_to_num(w * r[:, k]) * wk_all_bad)
    fs = eng.flux_scores[0]
    assert np.isfinite(fs).all() and np.isfinite(eng.positions).all()
    for k, p in enumerate(plains):
        assert_scores_equal(fs[k], p.flux, f"score {k}")
    assert_same_particles(eng, plains[0])
    assert eng.stats()["lost"] == len(bad)
    o2, d2, f2, w2 = wl.next_step()
    r2 = responses(rng, wl.n, nscores)
    eng.MoveToNextLocationScored(o2.reshape(-1).copy(), d2.reshape(-1).copy(), f2.copy(), w2.copy(), r2)
    for k, p in enumerate(plains):
        p.MoveToNextLocation(o2.reshape(-1).copy(), d2.reshape(-1).copy(), f2.copy(), w2 * r2[:, k])
    fs = eng.flux_scores[0]
    for k, p in enumerate(plains):
        assert_scores_equal(fs[k], p.flux, f"after: score {k}")


def test_cxx_program_with_scores(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SetScores + MoveToNextLocationScored next to the reference class."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "scores_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "scores_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "SCORES_OK" in out, out


def _two_gpu_scores_worker(rank, world, port, q):
    import sys

    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pumiumtally_b200.distributed import broadcast_unique_id, particle_stripe

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    n_total, nbins, nscores = 30_000, 2, 3
    b, e = particle_stripe(n_total, rank, world)
    eng = PumiTally.from_spec("box:7,7,7", e - b, device=rank)
    eng.set_score_bins(nbins)
    eng.set_scores(nscores)  # before comm_init: the exchange buffers are sized for all bins and scores
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    wl = SyntheticWorkload(box=(7.0, 7.0, 7.0), num_particles=e - b, mean_length=2.0, id_offset=b)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1))
    for k in range(2):
        o, d, f, w = wl.next_step()
        r = np.random.default_rng(k).uniform(0.0, 2.0, (n_total, nscores))[b:e].copy()
        eng.MoveToNextLocationScored(o.reshape(-1), d.reshape(-1), f, w, r, _bins(n_total, nbins, k)[b:e].copy())
        (eng.allreduce_tally if k == 0 else eng.reduce_tally_to_owners)()
    flux = eng.flux_scores
    if rank == 0:
        q.put(flux)
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_scores_exchange_equals_single_gpu():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + os.getpid() % 1000
    procs = [ctx.Process(target=_two_gpu_scores_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    flux2 = q.get(timeout=180)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    n_total, nbins, nscores = 30_000, 2, 3
    coords, t2v, wl = box_case((7, 7, 7), n_total, mean_length=2.0)
    one = PumiTally.from_spec("box:7,7,7", n_total)
    one.set_score_bins(nbins)
    one.set_scores(nscores)
    one.CopyInitialPosition(wl.initial_positions().reshape(-1))
    for k in range(2):
        o, d, f, w = wl.next_step()
        r = np.random.default_rng(k).uniform(0.0, 2.0, (n_total, nscores))
        one.MoveToNextLocationScored(o.reshape(-1), d.reshape(-1), f, w, r, _bins(n_total, nbins, k))
    fs = one.flux_scores
    for b in range(nbins):
        for k in range(nscores):
            assert_flux_close(flux2[b, k], fs[b, k], f"2-GPU bin {b} score {k} vs 1 GPU")
