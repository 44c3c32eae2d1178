"""Region currents (pumitally_set_region_currents): the face currents summed over every ordered pair of adjacent
regions on the device, and the net current of each pair, with batch statistics.  The open tally is checked against
numpy sums of pumitally_get_face_current_results over an independent numpy pair plan (region_currents_ref.py), the
pairs into the outside against the leakage, the net currents against particle balance (weight that starts in a region
minus weight that ends there), and the batch statistics against numpy statistics of the values captured before every
end_batch."""
import os
import subprocess

import numpy as np
import pytest

from helpers import ROOT, l_shaped_mesh
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from region_currents_ref import OUTSIDE, face_areas, pair_plan, pair_values, reverse
from test_gpu_batch_stats import MODES, numpy_stats
from test_gpu_face_currents import EDGES, _configure, _interior_points, _move
from test_gpu_scores import _bins, engine

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def reference(eng, region):
    """(partial, net) [ntime, nbins, P] from the engine's face currents and a numpy pair plan, and the plan"""
    adj = eng.adjacency
    frm, to, first, slots = pair_plan(adj, region)
    inc, out = eng.face_current_results(1), eng.face_current_results(0)
    T, B = inc.shape[:2]
    vals = inc.reshape(T, B, -1).copy()
    hull = adj.reshape(-1) < 0
    vals[..., hull] = out.reshape(T, B, -1)[..., hull]
    partial = pair_values(vals, first, slots)
    rev = reverse(frm, to)
    net = partial - np.where(rev >= 0, partial[..., np.maximum(rev, 0)], 0.0)
    return partial, net, (frm, to, first, slots, rev)


def assert_close(got, want, label, rtol=1e-12):
    scale = np.abs(want).max() + 1e-300
    np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-14 * scale, err_msg=label)


def check_open_tally(eng, region, label):
    partial, net, (frm, to, *_) = reference(eng, region)
    gf, gt = eng.region_current_pairs()
    np.testing.assert_array_equal(gf, frm, err_msg=label)
    np.testing.assert_array_equal(gt, to, err_msg=label)
    got_p, got_n = eng.region_current_results(0, 0), eng.region_current_results(1, 0)
    assert_close(got_p, partial, f"{label} partial")
    assert_close(got_n, net, f"{label} net")
    # the pairs into the outside add up to the leakage
    assert_close(got_p[..., to == OUTSIDE].sum(axis=-1), eng.leakage(0), f"{label} leakage")
    return got_p, got_n


def random_map(E, nregions, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(-1, nregions, E).astype(np.int32)


def slab_map(coords, t2v, nslabs, axis=2):
    cen = np.asarray(coords)[np.asarray(t2v)].mean(axis=1)[:, axis]
    lo, hi = cen.min(), cen.max()
    return np.minimum(((cen - lo) / (hi - lo) * nslabs).astype(np.int32), nslabs - 1)


def _flights(eng, rng, n, lo, hi, kind, step, nbins):
    o = eng.positions
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    d = o + u * rng.exponential(0.5 * (hi - lo).max(), n)[:, None]
    w = rng.uniform(0.25, 2.0, n)
    bins = _bins(n, nbins, step) if nbins > 1 else None
    r = np.ascontiguousarray(rng.uniform(0.0, 2.0, (n, eng.scores)))
    times = rng.uniform(EDGES[0] - 1.0, EDGES[-1] + 0.5, n)
    speeds = rng.uniform(0.3, 3.0, n)
    return o, d, np.ones(n, np.int8), w, (bins, r, times, speeds)


@pytest.mark.parametrize("mesh", ["kuhn", "lshape"])
@pytest.mark.parametrize("kind", ["plain", "binned", "timed"])
@pytest.mark.parametrize("device", [False, True])
def test_open_tally_matches_numpy(mesh, kind, device):
    coords, t2v = kuhn_box(5, 5, 4) if mesh == "kuhn" else l_shaped_mesh(6, 6, 3)
    n = 3000
    eng = engine(coords, t2v, n, -1)
    _configure(eng, kind)
    E = len(t2v)
    rng = np.random.default_rng(7)
    maps = {"random": random_map(E, 5, 3), "one": np.zeros(E, np.int32), "per_element": rng.permutation(E).astype(np.int32)}
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
    for name, region in maps.items():  # (each map resets the tally; the particles fly on from where they are)
        eng.set_regions(region, int(region.max()) + 1)
        eng.set_region_currents(True)
        assert eng.region_currents
        for step in range(2):
            o, d, f, w, extra = _flights(eng, rng, n, lo, hi, kind, step, eng.score_bins)
            _move(eng, kind, o, d, f, w, extra, device)
        check_open_tally(eng, region, f"{mesh} {kind} {name}")
        # the areas: the plan-order sum of the face areas of each pair (numpy's order here, to 1e-13)
        frm, to, first, slots = pair_plan(eng.adjacency, region)
        area = pair_values(face_areas(coords, t2v).reshape(-1), first, slots)
        np.testing.assert_allclose(eng.region_current_areas(), area, rtol=1e-13)


def _balance(eng, region, o, d, f, w):
    """sum_i w_i ([reg(o_i) == A] - [reg(d_i) == A]) for every region A in [-1, nregions), d outside: -2"""
    reg = lambda xyz: np.where((e := eng.locate(np.ascontiguousarray(xyz))) >= 0,  # noqa: E731
                               region[np.maximum(e, 0)], OUTSIDE)
    ro, rd = reg(o), reg(d)
    fly = f == 1
    ids = np.arange(-1, int(region.max()) + 1)
    return {int(a): (w[fly & (ro == a)].sum() - w[fly & (rd == a)].sum()) for a in ids}


def _check_balance(eng, net, frm, bal, wsum, label):
    for a, want in bal.items():
        got = net[..., frm == a].sum()
        assert abs(got - want) <= 1e-12 * wsum, (label, a, got, want)


def test_conservation_on_a_convex_box():
    """Sum over B of net(A -> B) is the weight that starts in A minus the weight that ends in A."""
    coords, t2v = kuhn_box(6, 5, 4)
    n = 20000
    eng = engine(coords, t2v, n, -1)
    eng.set_face_currents(True)
    E = len(t2v)
    region = random_map(E, 6, 9)
    eng.set_regions(region, 6)
    eng.set_region_currents(True)
    rng = np.random.default_rng(1)
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
    o, d, f, w, _ = _flights(eng, rng, n, lo, hi, "plain", 0, 1)
    eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
    frm, _ = eng.region_current_pairs()
    _check_balance(eng, eng.region_current_results(1, 0)[0, 0], frm, _balance(eng, region, o, d, f, w), w.sum(),
                   "box")


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_eight_batches_match_numpy(mode):
    coords, t2v = kuhn_box(5, 5, 4)
    n = 3000
    eng = engine(coords, t2v, n, -1)
    eng.set_score_bins(2)
    eng.set_face_currents(True)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(mode, MODES[mode])
    region = random_map(len(t2v), 4, mode)
    eng.set_regions(region, 4)
    eng.set_region_currents(True)
    rng = np.random.default_rng(mode)
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
    caps = {0: [], 1: []}
    for b in range(8):
        o, d, f, w, extra = _flights(eng, rng, n, lo, hi, "binned", b, 2)
        w = w * (1.0 + 0.5 * np.sin(b))
        eng.MoveToNextLocationBinned(o.reshape(-1).copy(), d.reshape(-1).copy(), f, w, extra[0])
        for which in (0, 1):
            caps[which].append(eng.region_current_results(which, 0))
        eng.end_batch()
    for which in (0, 1):
        m, s, rel = numpy_stats(np.array(caps[which]))
        scale = np.abs(np.array(caps[which])).max()
        np.testing.assert_allclose(eng.region_current_results(which, 1), m, rtol=1e-12, atol=1e-14 * scale)
        np.testing.assert_allclose(eng.region_current_results(which, 2), s, rtol=1e-9, atol=1e-12 * scale)
        np.testing.assert_allclose(eng.region_current_results(which, 3), rel, rtol=1e-8, atol=1e-12)


def test_net_error_holds_the_covariance():
    """An A | B | A slab map with flights along the slab normal: a flight through B scores A -> B and B -> A alike, so
    the net current's error is far below what independent partials would give."""
    coords, t2v = kuhn_box(4, 4, 6)
    n = 4000
    eng = engine(coords, t2v, n, -1)
    eng.set_face_currents(True)
    eng.set_batch_statistics(True)
    slab = slab_map(coords, t2v, 3)
    region = np.where(slab == 1, 1, 0).astype(np.int32)
    eng.set_regions(region, 2)
    eng.set_region_currents(True)
    frm, to = eng.region_current_pairs()
    ab = np.flatnonzero((frm == 0) & (to == 1))[0]
    ba = np.flatnonzero((frm == 1) & (to == 0))[0]
    rng = np.random.default_rng(4)
    caps = []
    eng.CopyInitialPosition(np.tile([2.0, 2.0, 1.0], n))
    for b in range(10):
        o = np.column_stack([rng.uniform(0.1, 3.9, n), rng.uniform(0.1, 3.9, n), rng.uniform(0.1, 1.9, n)])
        d = o + np.array([0.0, 0.0, 1.0]) * rng.uniform(3.0, 5.0, n)[:, None]  # about 1 in 9 ends in B
        d[:, 2] = np.minimum(d[:, 2], 5.9)
        w = rng.uniform(0.1, 3.0) * rng.uniform(0.5, 1.5, n)
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), np.ones(n, np.int8), w)
        caps.append((eng.region_current_results(0, 0)[0, 0], eng.region_current_results(1, 0)[0, 0]))
        eng.end_batch()
    part = np.array([c[0] for c in caps])
    net = np.array([c[1] for c in caps])
    _, s_net, _ = numpy_stats(net[:, ab])
    se = eng.region_current_results(1, 2)[0, 0]
    np.testing.assert_allclose(se[ab], s_net, rtol=1e-9)
    sp = eng.region_current_results(0, 2)[0, 0]
    _, s_ab, _ = numpy_stats(part[:, ab])
    _, s_ba, _ = numpy_stats(part[:, ba])
    np.testing.assert_allclose([sp[ab], sp[ba]], [s_ab, s_ba], rtol=1e-9)
    assert se[ab] < 0.25 * np.hypot(sp[ab], sp[ba]), (se[ab], sp[ab], sp[ba])


def _stats_engine(coords, t2v, n, region, rc=True):
    eng = engine(coords, t2v, n, -1)
    eng.set_face_currents(True)
    eng.set_batch_statistics(True)
    eng.set_regions(region, int(region.max()) + 1)
    if rc:
        eng.set_region_currents(True)
    return eng


def _batches(eng, coords, t2v, rng, k, capture=True):
    n = eng.num_particles
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    caps = []
    eng.CopyInitialPosition(_interior_points(rng, coords, t2v, n).reshape(-1).copy())
    for b in range(k):
        o, d, f, w, _ = _flights(eng, rng, n, lo, hi, "plain", b, 1)
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f, w * (1 + 0.3 * b))
        if capture:
            caps.append([eng.region_current_results(which, 0) for which in (0, 1)])
        eng.end_batch()
    return caps


def test_checkpoints(tmp_path, capfd):
    coords, t2v = kuhn_box(4, 4, 4)
    n = 2000
    region = random_map(len(t2v), 3, 5)
    a = _stats_engine(coords, t2v, n, region)
    caps_a = _batches(a, coords, t2v, np.random.default_rng(1), 4)
    pa = str(tmp_path / "a.ckpt")
    a.save_checkpoint(pa)
    # save and load: the statistics come back bit for bit
    c = _stats_engine(coords, t2v, n, region)
    c.load_checkpoint(pa)
    for which in (0, 1):
        for kind in (1, 2, 3):
            np.testing.assert_array_equal(bits(c.region_current_results(which, kind)),
                                          bits(a.region_current_results(which, kind)))
    # merge: Chan's update of the two runs' batches, which numpy gives as the statistics of all eight
    b = _stats_engine(coords, t2v, n, region)
    caps_b = _batches(b, coords, t2v, np.random.default_rng(2), 4)
    pb = str(tmp_path / "b.ckpt")
    b.save_checkpoint(pb)
    a.merge_checkpoint(pb)
    assert a.batches == 8
    for which in (0, 1):
        x = np.array([cap[which] for cap in caps_a + caps_b])
        m, s, rel = numpy_stats(x)
        scale = np.abs(x).max()
        np.testing.assert_allclose(a.region_current_results(which, 1), m, rtol=1e-12, atol=1e-14 * scale)
        np.testing.assert_allclose(a.region_current_results(which, 2), s, rtol=1e-9, atol=1e-12 * scale)
    # a file saved with the other setting is refused, naming region currents, and changes nothing
    off = _stats_engine(coords, t2v, n, region, rc=False)
    _batches(off, coords, t2v, np.random.default_rng(3), 2, capture=False)
    poff = str(tmp_path / "off.ckpt")
    off.save_checkpoint(poff)
    capfd.readouterr()
    with pytest.raises(RuntimeError):
        c.load_checkpoint(poff)
    assert "region currents" in capfd.readouterr().err
    assert c.batches == 4
    with pytest.raises(RuntimeError):
        c.merge_checkpoint(poff)
    assert "region currents" in capfd.readouterr().err
    with pytest.raises(RuntimeError):
        off.load_checkpoint(pa)
    assert "region currents" in capfd.readouterr().err
    assert off.batches == 2
    # with region currents off, a file is byte for byte what an engine that never had them writes
    off.set_region_currents(True)
    off.set_region_currents(False)
    off.load_checkpoint(poff)
    p2 = str(tmp_path / "off2.ckpt")
    off.save_checkpoint(p2)
    with open(poff, "rb") as f1, open(p2, "rb") as f2:
        assert f1.read() == f2.read()


def test_refusals_and_resets(capfd):
    coords, t2v = kuhn_box(3, 3, 3)
    E = len(t2v)
    eng = engine(coords, t2v, 500, -1)
    eng.set_batch_statistics(True)
    with pytest.raises(ValueError):  # no regions, no face currents
        eng.set_region_currents(True)
    eng.set_regions(random_map(E, 3, 1), 3)
    with pytest.raises(ValueError):  # face currents off
        eng.set_region_currents(True)
    assert not eng.region_currents and eng.region_current_pairs()[0].size == 0
    eng.set_face_currents(True)
    assert eng._L.pumitally_set_region_currents(eng._h, 2) != 0
    assert not eng.region_currents
    eng.set_region_currents(True)
    P = eng.region_current_pairs()[0].size
    assert eng.region_currents and P > 0
    # results: refused without batches for kinds 1-3, with a wrong which, kind or n
    with pytest.raises(RuntimeError):
        eng.region_current_results(0, 1)
    out = np.empty(P + 1)
    from pumiumtally_b200.tally import _dp
    assert eng._L.pumitally_get_region_current_results(eng._h, 0, 0, out.ctypes.data_as(_dp), P + 1) != 0
    assert eng._L.pumitally_get_region_current_results(eng._h, 2, 0, out.ctypes.data_as(_dp), P) != 0
    assert eng._L.pumitally_get_region_current_results(eng._h, 0, 4, out.ctypes.data_as(_dp), P) != 0
    # a new map keeps them on with the new map's pairs; removing the regions or the face currents switches them off
    eng.set_regions(np.zeros(E, np.int32), 1)
    assert eng.region_currents
    f, t = eng.region_current_pairs()
    assert list(zip(f, t)) == [(0, OUTSIDE)]
    eng.set_regions(None)
    assert not eng.region_currents
    with pytest.raises(RuntimeError):
        eng.region_current_results(0, 0)
    eng.set_regions(random_map(E, 3, 1), 3)
    eng.set_region_currents(True)
    eng.set_face_currents(False)
    assert not eng.region_currents
    # a refusal changes nothing: the folded batches stay
    eng.set_face_currents(True)
    eng.set_region_currents(True)
    _batches(eng, coords, t2v, np.random.default_rng(0), 2, capture=False)
    before = eng.region_current_results(1, 1)
    assert eng._L.pumitally_set_region_currents(eng._h, 7) != 0
    assert eng.batches == 2 and eng.region_currents
    np.testing.assert_array_equal(bits(eng.region_current_results(1, 1)), bits(before))


def test_refused_after_comm_init():
    import torch.distributed as dist

    if not dist.is_available():
        pytest.skip("torch.distributed unavailable")
    eng = PumiTally.from_spec("box:3,3,3", 100)
    eng.set_face_currents(True)
    eng.set_regions(np.zeros(eng.num_elements, dtype=np.int32), 1)
    try:
        eng.comm_init(0, 1, PumiTally.nccl_unique_id())
    except Exception as exc:  # no NCCL on this machine
        pytest.skip(f"comm_init unavailable: {exc}")
    with pytest.raises(ValueError):
        eng.set_region_currents(True)
    assert not eng.region_currents


def test_config_c2_ten_batches():
    """Full-size c2 (998,250 tets, 10 M particles), 64 slab regions, ten batches: in every batch the nets balance the
    particles and the partials into the outside give the leakage; the folded means are the captured means."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n = cfg["particles"]
    wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    eng = PumiTally.from_arrays(coords, t2v, n)
    eng.set_face_currents(True)
    eng.set_batch_statistics(True)
    region = slab_map(coords, t2v, 64)
    eng.set_regions(region, 64)
    eng.set_region_currents(True)
    frm, to = eng.region_current_pairs()
    s = torch.cuda.current_stream().cuda_stream
    eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
    caps = []
    for b in range(10):
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
        torch.cuda.synchronize()
        on, dn, fn, wn = (x.cpu().numpy() for x in (o, d, f, w))
        part, net = eng.region_current_results(0, 0)[0, 0], eng.region_current_results(1, 0)[0, 0]
        leak = eng.leakage(0)[0, 0]
        assert abs(part[to == OUTSIDE].sum() - leak) <= 1e-12 * leak, (b, part[to == OUTSIDE].sum(), leak)
        _check_balance(eng, net, frm, _balance(eng, region, on.reshape(-1, 3), dn.reshape(-1, 3), fn, wn),
                       wn[fn == 1].sum(), f"c2 batch {b}")
        caps.append(net)
        eng.end_batch()
    x = np.array(caps)
    m, sd, _ = numpy_stats(x)
    np.testing.assert_allclose(eng.region_current_results(1, 1)[0, 0], m, rtol=1e-12, atol=1e-14 * np.abs(x).max())
    np.testing.assert_allclose(eng.region_current_results(1, 2)[0, 0], sd, rtol=1e-8, atol=1e-12 * np.abs(x).max())


def test_cxx_program_with_region_currents(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SetRegionCurrents, GetRegionCurrentPairs, GetRegionCurrentAreas and
    GetRegionCurrentResults."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "region_currents_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "region_currents_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "REGION_CURRENTS_OK" in out, out


def _two_gpu_worker(rank, world, port, q):
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
    eng.set_face_currents(True)
    eng.set_batch_statistics(True)
    eng.set_regions(slab_map(c, t, 4), 4)
    eng.set_region_currents(True)
    eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id, device=torch.device("cuda", rank)))
    wl = SyntheticWorkload(box=(5.0, 5.0, 5.0), num_particles=n, mean_length=1.0, seed=300 + rank)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    local = []
    for _ in range(5):
        o, d, f, w = wl.next_step()
        eng.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), f.copy(), w.copy())
        local.append([eng.region_current_results(which, 0).copy() for which in (0, 1)])
        eng.end_batch()
    q.put((rank, local, [[eng.region_current_results(which, k) for k in (1, 2, 3)] for which in (0, 1)]))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpus_fold_the_summed_batches():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 113) % 1000
    procs = [ctx.Process(target=_two_gpu_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for which in (0, 1):
        x = np.array([res[0][1][b][which] + res[1][1][b][which] for b in range(5)])  # mode 0: divisor 1
        m, s, rel = numpy_stats(x)
        for k, want in enumerate((m, s, rel)):
            np.testing.assert_allclose(res[0][2][which][k], want, rtol=1e-9, atol=1e-12 * np.abs(x).max())
            np.testing.assert_array_equal(bits(res[1][2][which][k]), bits(res[0][2][which][k]))
