"""Region tallies (pumitally_set_regions): every result summed over caller-defined groups of elements on the device,
and the batch statistics of those sums.  The identity map (region e is element e) must give the per-element accessors
bit for bit; other maps are checked against fsum / numpy references of the per-element arrays, and the region errors
against numpy statistics of the per-batch region sums."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_batch_stats import MODES, Batches, assert_stats, numpy_stats
from test_gpu_moments import _move
from test_gpu_scores import assert_same_particles
from test_gpu_tally_collisions import CASES, _geometry

pytestmark = pytest.mark.gpu

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def assert_bits(got, want, label):
    np.testing.assert_array_equal(bits(got), bits(want), err_msg=label)


def fsum_regions(x, region, nregions):
    """x [..., E] -> [..., nregions], exactly rounded sums over the elements of each region"""
    lead = x.shape[:-1]
    flat = x.reshape(-1, x.shape[-1])
    out = np.empty((flat.shape[0], nregions))
    for g in range(nregions):
        sel = region == g
        for j in range(flat.shape[0]):
            out[j, g] = math.fsum(flat[j, sel])
    return out.reshape(lead + (nregions,))


def slab_map(coords, t2v, nslabs, axis=2):
    """region of every element (caller's numbering): the slab of its centroid along `axis`"""
    cen = np.asarray(coords)[np.asarray(t2v)].mean(axis=1)[:, axis]
    lo, hi = cen.min(), cen.max()
    return np.minimum(((cen - lo) / (hi - lo) * nslabs).astype(np.int32), nslabs - 1)


@pytest.mark.parametrize("case", list(CASES))
def test_identity_map_gives_the_element_results(case):
    b = Batches(case, mode=3, seed=31)
    E = len(b.t)
    b.eng.set_regions(np.arange(E, dtype=np.int32))
    assert b.eng.regions == E and b.eng.batches == 0
    for batch in range(8):
        b.move()
        if batch == 0:
            assert_bits(b.eng.region_volumes(), b.eng.normalized_flux_time()[1], "volumes")
        assert_bits(b.eng.region_results(0, 0), b.eng.flux_time, f"{case} raw {batch}")
        assert_bits(b.eng.region_results(0, 1), b.eng.normalized_flux_time()[0], f"{case} normalised {batch}")
        assert_bits(b.eng.region_results(1, 0), b.eng.collision_results(0), f"{case} collision raw {batch}")
        assert_bits(b.eng.region_results(1, 1), b.eng.collision_results(1), f"{case} collision normalised {batch}")
        b.eng.end_batch()
    for tally in (0, 1):
        for kind in range(3):
            assert_bits(b.eng.region_batch_results(tally, kind), b.eng.batch_results(tally, kind),
                        f"{case} batch tally {tally} kind {kind}")
    # n == nregions: time bin 0, bin 0, score 0
    first = np.empty(E)
    assert b.eng._L.pumitally_get_region_results(b.eng._h, 0, 0, first.ctypes.data_as(_dp), E) == 0
    assert_bits(first, b.eng.region_results(0, 0)[0, 0, 0], "first")
    assert b.eng._L.pumitally_get_region_batch_results(b.eng._h, 1, 2, first.ctypes.data_as(_dp), E) == 0
    assert_bits(first, b.eng.region_batch_results(1, 2)[0, 0, 0], "first batch")


def random_map(E, nregions, seed):
    """ids in [-1, nregions) with region nregions - 1 left empty"""
    rng = np.random.default_rng(seed)
    region = rng.integers(-1, nregions - 1, E).astype(np.int32)
    return region


@pytest.mark.parametrize("case", ["s1", "s3_b3_t_mo"])
def test_random_map_against_fsum(case):
    b = Batches(case, mode=1, seed=41)
    E = len(b.t)
    G = 9
    region = random_map(E, G, 3)
    assert (region == -1).any() and not (region == G - 1).any()
    b.eng.set_regions(region, G)
    vol = b.eng.normalized_flux_time()[1]
    want_vol = fsum_regions(vol, region, G)
    np.testing.assert_allclose(b.eng.region_volumes(), want_vol, rtol=1e-13, atol=0)
    assert b.eng.region_volumes()[G - 1] == 0.0
    d = b.eng.source_normalization()
    for batch in range(3):
        b.move()
        for tally, raw in ((0, b.eng.flux_time), (1, b.eng.collision_results(0))):
            want = fsum_regions(raw, region, G)
            got = b.eng.region_results(tally, 0)
            np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-13 * np.abs(want).max())
            assert (got[..., G - 1] == 0.0).all()
            norm = b.eng.region_results(tally, 1)
            np.testing.assert_allclose(norm[..., :G - 1], want[..., :G - 1] / want_vol[:G - 1] / d, rtol=1e-12)
            assert np.isnan(norm[..., G - 1]).all()  # 0 / 0
        b.eng.end_batch()
    for tally in (0, 1):
        for kind in range(3):
            r = b.eng.region_batch_results(tally, kind)
            assert np.isnan(r[..., G - 1]).all() and np.isfinite(r[..., :G - 1]).all(), (tally, kind)


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mode", list(MODES))
def test_eight_batches_match_numpy(mode, path):
    """Kind 0 and the divisor captured before every end_batch; the engine's mean, standard error and relative error
    of the region sums against numpy's."""
    b = Batches("s3_b3_t", mode=mode, path=path, seed=51 + mode)
    E = len(b.t)
    G = 12
    region = slab_map(b.c, b.t, G - 1)
    region[::7] = -1
    region[region == 5] = G - 1
    b.eng.set_regions(region, G)
    vol = b.eng.region_volumes()
    caps = []
    for _ in range(8):
        b.move()
        d = b.eng.source_normalization()
        caps.append([b.eng.region_results(tally, 0) / d for tally in (0, 1)])
        b.eng.end_batch()
    assert b.eng.batches == 8 and E > G
    for tally in (0, 1):
        x = np.array([c[tally] for c in caps])
        m, s, rel = numpy_stats(x)
        want = (m / vol, s / vol, rel)
        for kind in range(3):
            got = b.eng.region_batch_results(tally, kind)
            live = vol > 0
            assert_stats(got[..., live], want[kind][..., live], f"mode {mode} {path} tally {tally} kind {kind}")
            assert np.isnan(got[..., ~live]).all()


def test_covariances_are_in_the_region_error():
    """Long tracks cross many elements of one slab in the same batch, so the elements' scores rise and fall together:
    the standard error of the slab's sum is far above the quadrature sum of the per-element errors, and it is what
    numpy gives for the per-batch slab sums."""
    c, t = kuhn_box(12, 12, 12)
    n, B = 3000, 16
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(1)
    z = slab_map(c, t, 4)
    region = np.where(z == 1, 0, -1).astype(np.int32)
    eng.set_regions(region, 1)
    assert (region == 0).sum() > 1000
    wl = SyntheticWorkload(box=(12.0, 12.0, 12.0), num_particles=n, mean_length=8.0, seed=61)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    sums = []
    for _ in range(B):
        _move(eng, "plain", *wl.next_step())
        sums.append(eng.region_results(0, 0)[0, 0, 0, 0] / n)
        eng.end_batch()
    vol = eng.region_volumes()[0]
    m, s, rel = numpy_stats(np.array(sums))
    got = [eng.region_batch_results(0, kind)[0, 0, 0, 0] for kind in range(3)]
    np.testing.assert_allclose(got, [m / vol, s / vol, rel], rtol=1e-12)
    se = eng.batch_results(0, 1)[0, 0, 0]
    ev = eng.normalized_flux_time()[1]
    sel = region == 0
    quad = math.sqrt(math.fsum((se[sel] * ev[sel]) ** 2)) / vol
    ratio = got[1] / quad
    print(f"slab standard error {got[1]:.4g}, quadrature of the element errors {quad:.4g}, ratio {ratio:.2f}")
    assert ratio > 1.5


def _centroid_events(eng, c, t, rng):
    """one collision event at every element's centroid: each element's collision tally is a single addition, so two
    engines fed the same events hold bit-identical tallies"""
    cen = np.asarray(c)[np.asarray(t)].mean(axis=1)
    eng.tally_collisions(cen, rng.uniform(0.5, 1.5, len(t)))


def test_determinism():
    c, t = kuhn_box(10, 9, 8)
    E = len(t)
    region = slab_map(c, t, 5)
    engs = []
    for _ in range(2):
        e = PumiTally.from_arrays(c, t, 100)
        e.set_collision_estimator(True)
        e.set_regions(region)
        _centroid_events(e, c, t, np.random.default_rng(70))
        engs.append(e)
    a, b = engs
    assert_bits(a.collision_results(0), b.collision_results(0), "the two raw tallies")
    assert_bits(a.region_results(1, 0), a.region_results(1, 0), "the same call twice")
    assert_bits(a.region_results(1, 0), b.region_results(1, 0), "two engines")
    assert_bits(a.region_results(1, 1), b.region_results(1, 1), "two engines, normalised")
    assert_bits(a.region_volumes(), b.region_volumes(), "volumes")
    b.set_regions(np.arange(E, dtype=np.int32))  # one element per region: the element's value itself
    assert_bits(b.region_results(1, 0), b.collision_results(0), "identity")


def test_refusals_and_resets():
    b = Batches("s1", mode=0, seed=81)
    eng, L, h = b.eng, b.eng._L, b.eng._h
    E = len(b.t)
    out = np.empty(E)
    with pytest.raises(RuntimeError):  # regions unset
        eng.region_results()
    assert L.pumitally_get_region_volumes(h, out.ctypes.data_as(_dp), 1) != 0
    assert eng.regions == 0
    good = (np.arange(E) % 4).astype(np.int32)
    bad = [
        (good[:-1], 4),                                   # wrong n
        (np.where(good == 0, -2, good).astype(np.int32), 4),  # below -1
        (good, 3),                                        # an id at nregions
        (good, 0),                                        # nregions out of range
        (good, E + 1),
    ]
    for k, (m, g) in enumerate(bad):
        assert L.pumitally_set_regions(h, np.ascontiguousarray(m).ctypes.data_as(_ip), len(m), g) != 0, k
        assert eng.regions == 0
    assert L.pumitally_set_regions(h, None, E, 4) != 0
    b.move()
    b.eng.end_batch()
    b.move()
    open_batch = eng.flux_time.copy()
    eng.set_regions(good, 4)  # resets the tally and discards the batches
    assert eng.regions == 4 and eng.batches == 0 and not eng.flux_time.any()
    assert open_batch.any()
    with pytest.raises(RuntimeError):  # no batch folded
        eng.region_batch_results(0, 0)
    for _ in range(2):
        b.move()
        eng.end_batch()
    b.move()
    raw = eng.region_results(0, 0).copy()
    mean = eng.region_batch_results(0, 0).copy()
    for m, g in bad:  # refused inputs change nothing
        assert L.pumitally_set_regions(h, np.ascontiguousarray(m).ctypes.data_as(_ip), len(m), g) != 0
    assert eng.regions == 4 and eng.batches == 2
    np.testing.assert_array_equal(eng.region_results(0, 0), raw)
    np.testing.assert_array_equal(eng.region_batch_results(0, 0), mean)
    refused = [
        lambda: L.pumitally_get_region_results(h, 0, 2, out.ctypes.data_as(_dp), 4),
        lambda: L.pumitally_get_region_results(h, 2, 0, out.ctypes.data_as(_dp), 4),
        lambda: L.pumitally_get_region_results(h, 0, 0, out.ctypes.data_as(_dp), 5),
        lambda: L.pumitally_get_region_batch_results(h, 0, 3, out.ctypes.data_as(_dp), 4),
        lambda: L.pumitally_get_region_batch_results(h, 0, 0, out.ctypes.data_as(_dp), E),
        lambda: L.pumitally_get_region_volumes(h, out.ctypes.data_as(_dp), 3),
    ]
    for k, call in enumerate(refused):
        assert call() != 0, k
    eng.set_collision_estimator(False)
    for call in (lambda: eng.region_results(1, 0), lambda: eng.region_batch_results(1, 0)):
        with pytest.raises(RuntimeError):  # tally 1 without the estimator
            call()
    _move(eng, "plain", *b.wl.next_step())
    eng.end_batch()
    for kind in (1, 2):
        with pytest.raises(RuntimeError):  # errors need two batches
            eng.region_batch_results(0, kind)
    eng.region_batch_results(0, 0)
    eng.set_batch_statistics(False)
    with pytest.raises(RuntimeError):
        eng.region_batch_results(0, 0)
    eng.region_results(0, 0)  # the open tally's sums need no statistics
    eng.set_regions(None)
    assert eng.regions == 0
    with pytest.raises(RuntimeError):
        eng.region_results(0, 0)


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
        eng.set_regions(np.zeros(eng.num_elements, dtype=np.int32))
    assert eng.regions == 0
    torch.cuda.synchronize()


def test_nothing_else_changes(tmp_path):
    from vtk_reader import read_vtu_cell_data

    a, b = Batches("s3_b3_t_mo", seed=4), Batches("s3_b3_t_mo", seed=4)
    a.eng.set_regions(slab_map(a.c, a.t, 6))
    b.eng.set_batch_statistics(True)  # the same resets as set_regions
    for step in range(3):
        a.move()
        b.move()
        assert_same_particles(a.eng, b.eng, f"step {step}")
        for what, u, v in (("flux", a.eng.flux_time, b.eng.flux_time),
                           ("collision", a.eng.collision_results(0), b.eng.collision_results(0)),
                           ("moments", a.eng.flux_moments(), b.eng.flux_moments())):
            np.testing.assert_allclose(u, v, rtol=1e-9, atol=1e-11 * np.abs(v).max(), err_msg=f"{what} {step}")
        a.eng.end_batch()
        b.eng.end_batch()
        sa, sb = a.eng.stats(), b.eng.stats()
        assert {k: sa[k] for k in sa if k != "kernel_ms"} == {k: sb[k] for k in sb if k != "kernel_ms"}
    for tally in (0, 1):
        for kind in range(3):
            v = b.eng.batch_results(tally, kind)
            np.testing.assert_allclose(a.eng.batch_results(tally, kind), v, rtol=1e-8, atol=1e-10 * np.abs(v).max())
    a.move()
    b.move()
    pa, pb = str(tmp_path / "a.vtk"), str(tmp_path / "b.vtk")
    a.eng.WriteTallyResults(pa)
    b.eng.WriteTallyResults(pb)
    ca = read_vtu_cell_data(os.path.join(pa, "pieces", "piece_0.vtu"))
    cb = read_vtu_cell_data(os.path.join(pb, "pieces", "piece_0.vtu"))
    assert list(ca) == list(cb)


def test_config_c2_ten_batches():
    """Full-size c2 (998,250 tets, 10 M particles): 10 batches with 64 slab regions against numpy, then 10 with the
    identity map against the per-element statistics, bit for bit."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    E = len(t2v)
    n = cfg["particles"]
    wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    eng = PumiTally.from_arrays(coords, t2v, n)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(3)
    s = torch.cuda.current_stream().cuda_stream
    eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)

    def batches(k, capture):
        caps = []
        for _ in range(k):
            o, d, f, w = (x.contiguous() for x in wl.next_step())
            eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
            torch.cuda.synchronize()
            if capture:
                caps.append(eng.region_results(0, 0)[0, 0, 0] / eng.source_normalization())
            eng.end_batch()
        return caps

    eng.set_regions(slab_map(coords, t2v, 64))
    vol = eng.region_volumes()
    np.testing.assert_allclose(vol.sum(), _geometry(coords, t2v)[1].sum(), rtol=1e-12)
    caps = batches(10, True)
    m, sd, rel = numpy_stats(np.array(caps))
    for kind, want in enumerate((m / vol, sd / vol, rel)):
        assert_stats(eng.region_batch_results(0, kind)[0, 0, 0], want, f"c2 slabs kind {kind}")
    eng.set_regions(np.arange(E, dtype=np.int32))
    batches(10, False)
    for kind in range(3):
        assert_bits(eng.region_batch_results(0, kind), eng.batch_results(0, kind), f"c2 identity kind {kind}")


def test_cxx_program_with_regions(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SetRegions, GetRegionVolumes, GetRegionResults and GetRegionBatchResults."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "regions_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "regions_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "REGIONS_OK" in out, out


def _two_gpu_region_worker(rank, world, port, q):
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
    eng.set_collision_estimator(True)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(3)
    eng.set_regions(slab_map(c, t, 7))
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    wl = SyntheticWorkload(box=(5.0, 5.0, 5.0), num_particles=n, mean_length=1.0, seed=200 + rank)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    rng = np.random.default_rng(rank)
    local, weights = [], []
    for _ in range(5):
        o, d, f, w = wl.next_step()
        w = w * rng.uniform(0.5, 1.5)
        _move(eng, "scored", o, d, f, w, rng.uniform(0.0, 1.0, (n, 2)))
        eng.tally_collisions(rng.uniform(0.0, 5.0, (2000, 3)), rng.uniform(0.5, 1.5, 2000),
                             rng.uniform(0.0, 1.0, (2000, 2)))
        local.append((eng.region_results(0, 0).copy(), eng.region_results(1, 0).copy()))
        weights.append(float((w * (f == 1)).sum()))
        eng.end_batch()
    results = [[eng.region_batch_results(tally, kind) for kind in range(3)] for tally in (0, 1)]
    q.put((rank, local, weights, eng.region_volumes(), results))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpus_fold_the_summed_batches():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 71) % 1000
    procs = [ctx.Process(target=_two_gpu_region_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    vol = res[0][3]
    div = np.array(res[0][2]) + np.array(res[1][2])  # mode 3: the whole batch's first-track weight
    for tally in (0, 1):
        x = np.array([(res[0][1][b][tally] + res[1][1][b][tally]) / div[b] for b in range(5)])
        m, s, rel = numpy_stats(x)
        for kind, want in enumerate((m / vol, s / vol, rel)):
            assert_stats(res[0][4][tally][kind], want, f"tally {tally} kind {kind}")
            assert_bits(res[1][4][tally][kind], res[0][4][tally][kind], f"the same on both ranks {tally} {kind}")
