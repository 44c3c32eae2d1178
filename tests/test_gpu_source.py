"""Mesh source (pumitally_set_source / _sample_source): the host and device samples must equal the numpy restatement of
the contract (tests/source_ref.py) bit for bit; a sample depends on (seed, index) alone; placement puts each particle
in its sampled element without a walk, so a move from there matches the exact clip-and-walk reference even where a
relocation walk from the previous positions would stop at the hull; and set_source, sampling without placement and
every refusal leave the tally state, the particle state and the counters bit-identical."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import source_ref as sr
from helpers import ROOT, assert_flux_close
from locate_ref import MESHES, barycentric
from moments_ref import assert_m0_close, reference_moments
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_batch_stats import Batches
from test_gpu_checkpoint import assert_same, snapshot

pytestmark = pytest.mark.gpu
N = 1_000_000


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def assert_samples(got, want, label):
    for g, w, what in zip(got, want, ("xyz", "elem", "group", "weight")):
        np.testing.assert_array_equal(bits(np.asarray(g)), bits(np.asarray(w)), err_msg=f"{label}: {what}")


def case_table(mesh, groups, biased, E, seed=0):
    rng = np.random.default_rng([groups, int(biased), seed, len(mesh)])
    q = rng.lognormal(0.0, 2.0, (groups, E)) * (rng.random((groups, E)) < 0.8)
    q[0, :2] = 0.0
    q[-1, -2:] = 0.0
    b = rng.uniform(0.05, 20.0, (groups, E)) if biased else None
    return q, b


def device_samples(eng, n, seed, first=0, place=False):
    import torch

    out = eng.sample_source_device(n, seed, first, place)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


@pytest.mark.parametrize("mesh", list(MESHES))
@pytest.mark.parametrize("groups", [1, 3])
@pytest.mark.parametrize("biased", [False, True])
@pytest.mark.parametrize("per_volume", [False, True])
def test_samples_equal_the_reference(mesh, groups, biased, per_volume):
    coords, t2v = MESHES[mesh]()
    eng = PumiTally.from_arrays(coords, t2v, 16)
    E = eng.num_elements
    q, b = case_table(mesh, groups, biased, E)
    eng.set_source(q, b, per_volume)
    assert eng.source_groups == groups
    table = sr.Table(q, eng.normalized_flux()[1], b, per_volume)
    assert eng.source_strength == table.Q
    for seed, first in ((1, 0), (2 ** 64 - 3, 2 ** 32 + 5)):
        want = sr.sample(table, coords, t2v, seed, first, N)
        label = f"{mesh} G{groups} bias {biased} per_volume {per_volume} seed {seed} first {first}"
        assert_samples(eng.sample_source(N, seed, first), want, label + " host")
        assert_samples(device_samples(eng, N, seed, first), want, label + " device")


def test_chunking_and_engines_do_not_change_a_sample():
    coords, t2v = MESHES["delaunay"]()
    q, b = case_table("delaunay", 3, True, len(t2v))
    eng = PumiTally.from_arrays(coords, t2v, 16)
    eng.set_source(q, b)
    whole = eng.sample_source(300_001, 77, 2 ** 33)
    a = 123_457
    for parts in ((eng.sample_source(a, 77, 2 ** 33), eng.sample_source(300_001 - a, 77, 2 ** 33 + a)),
                  (device_samples(eng, a, 77, 2 ** 33), device_samples(eng, 300_001 - a, 77, 2 ** 33 + a))):
        assert_samples(tuple(np.concatenate([p[k] for p in parts]) for k in range(4)), whole, "two calls")
    other = [PumiTally.from_arrays(coords, t2v, 16) for _ in range(2)]
    for e in other:
        e.set_source(q, b)
        e.set_option("chunk", 4096)
    parts = other[0].sample_source(a, 77, 2 ** 33), other[1].sample_source(300_001 - a, 77, 2 ** 33 + a)
    assert_samples(tuple(np.concatenate([p[k] for p in parts]) for k in range(4)), whole, "two engines")


@pytest.mark.parametrize("mesh", list(MESHES))
def test_locate_finds_the_sampled_element(mesh):
    coords, t2v = MESHES[mesh]()
    eng = PumiTally.from_arrays(coords, t2v, 16)
    eng.set_source(np.ones(eng.num_elements), per_volume=True)
    xyz, elem, _, _ = eng.sample_source(200_000, 5)
    found = eng.locate(xyz)
    other = found != elem
    if other.any():
        assert (found[other] >= 0).all(), f"{mesh}: a sampled point located outside the mesh"
        lam = barycentric(coords, t2v, xyz[other], elem[other])
        assert (lam.min(axis=1) <= 1e-12).all(), f"{mesh}: a point away from every face located elsewhere"
        lam2 = barycentric(coords, t2v, xyz[other], found[other])
        assert (lam2.min(axis=1) >= -1e-12).all()
    print(f"{mesh}: {int(other.sum())} of {len(elem)} samples on a shared face located in the neighbour")


def test_placement_stores_the_samples_and_counts_as_initial():
    coords, t2v = MESHES["void"]()
    n = 50_000
    eng = PumiTally.from_arrays(coords, t2v, n)
    q, b = case_table("void", 2, True, len(t2v))
    eng.set_source(q, b, per_volume=True)
    launches = eng.get_option("launches")
    xyz, elem, group, w = eng.sample_source(n, 9, 0, place=True)
    np.testing.assert_array_equal(eng.elem_ids, elem)
    np.testing.assert_array_equal(bits(eng.positions), bits(xyz))
    assert eng.get_option("launches") == launches
    with pytest.raises(RuntimeError):
        eng.CopyInitialPosition(xyz.reshape(-1).copy())
    # the device placement, with another seed
    dxyz, delem, _, _ = device_samples(eng, n, 10, 0, place=True)
    np.testing.assert_array_equal(eng.elem_ids, delem)
    np.testing.assert_array_equal(bits(eng.positions), bits(dxyz))
    assert_samples(device_samples(eng, n, 10), sr.sample(sr.Table(q, eng.normalized_flux()[1], b, True), coords, t2v,
                                                         10, 0, n), "void device")


@pytest.mark.parametrize("mesh", ["l_shape", "void"])
@pytest.mark.parametrize("path", ["host", "device"])
def test_move_from_placed_particles_matches_the_reference(mesh, path):
    """Old positions in one corner; new ones sampled everywhere.  A relocation walk from the old positions stops at
    the hull for some particles (the engine relocating that way puts them elsewhere); placement needs no walk, and a
    move from the placed points to their element's centroid tallies exactly what the clip-and-walk reference does."""
    import torch

    coords, t2v = MESHES[mesh]()
    n = 20_000
    E = len(t2v)
    cen = coords[t2v].mean(1)
    # the far end of one arm of the L, or the corner of the box around the void
    corner = cen[np.argmax(cen[:, 0] - cen[:, 1])] if mesh == "l_shape" else cen[np.argmin(cen.sum(1))]
    eng = PumiTally.from_arrays(coords, t2v, n)
    eng.set_source(np.ones(E), per_volume=True)
    eng.CopyInitialPosition(np.tile(corner, n))
    reloc = PumiTally.from_arrays(coords, t2v, n)
    reloc.CopyInitialPosition(np.tile(corner, n))
    if path == "host":
        xyz, elem, _, _ = eng.sample_source(n, 21, place=True)
    else:
        xyz, elem, _, _ = device_samples(eng, n, 21, place=True)
    dest = coords[t2v[elem]].mean(1)
    w = np.random.default_rng(3).uniform(0.5, 2.0, n)
    before = eng.stats()["relocations"]
    for e in (eng, reloc):
        flying = np.ones(n, dtype=np.int8)
        if path == "host":
            e.MoveToNextLocation(xyz.reshape(-1).copy(), dest.reshape(-1).copy(), flying, w)
        else:
            T = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda()  # noqa: E731
            do, dd, df, dw = T(xyz), T(dest), T(flying), T(w)
            e.move_device(do.data_ptr(), dd.data_ptr(), df.data_ptr(), dw.data_ptr(),
                          torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
    assert eng.stats()["relocations"] == before  # the move started where the particles were placed
    m0, _, abs_sum, _ = reference_moments(coords, t2v, xyz, dest, np.ones(n, dtype=bool), w, np.ones(n))
    assert_m0_close(eng.flux, m0[0, 0], abs_sum[0, 0], f"{mesh} {path}")
    np.testing.assert_array_equal(eng.elem_ids, elem)  # the centroids are in the sampled elements
    stopped = np.abs(reloc.flux - m0[0, 0]) > 1e-9 * abs_sum[0, 0] + 1e-300
    assert stopped.any(), f"{mesh}: no relocation from the corner stopped at the hull"
    print(f"{mesh} {path}: relocating instead would have tallied {int(stopped.sum())} elements wrongly")


def full_snapshot(b):
    s = snapshot(b)
    for k in ("launches", "variant"):
        s[k] = np.int64(b.eng.get_option(k))
    s["elem"], s["pos"] = b.eng.elem_ids, b.eng.positions
    return s


def test_set_sample_and_refusals_change_nothing(capfd):
    import torch

    b = Batches("s1", mode=0, seed=7)
    b.move()
    b.eng.end_batch()
    b.move()
    eng = b.eng
    E = eng.num_elements
    before = full_snapshot(b)
    q, bias = case_table("kuhn", 2, True, E)
    eng.set_source(q, bias, per_volume=True)
    want_q = eng.source_strength
    eng.sample_source(10_000, 3)
    device_samples(eng, 10_000, 3)
    eng.sample_source(0, 3)
    torch.cuda.synchronize()
    assert_same(before, full_snapshot(b), "set_source and sampling")

    def refused(fn, why):
        capfd.readouterr()
        with pytest.raises((ValueError, RuntimeError, TypeError)):
            fn()
        err = capfd.readouterr().err
        assert why in err, err
        assert eng.source_groups == 2 and eng.source_strength == want_q
        assert_same(before, full_snapshot(b), why)

    for k, (qq, bb, why) in enumerate(((-1.0, 1.0, "a strength is negative"), (np.nan, 1.0, "a strength"),
                                       (np.inf, 1.0, "a strength"), (1.0, -1.0, "a bias is negative"),
                                       (1.0, np.nan, "a bias"), (1.0, np.inf, "a bias"),
                                       (1.0, 0.0, "a bias is 0 where the strength is > 0"))):
        q2, b2 = q.copy(), bias.copy()
        q2[k % 2, (31 * k) % E], b2[k % 2, (31 * k) % E] = qq, bb
        refused(lambda: eng.set_source(q2, b2), why)
    refused(lambda: eng.set_source(np.zeros((2, E))), "is 0 or not finite")
    L = eng._L
    dp = C.POINTER(C.c_double)
    ptr = lambda a: a.ctypes.data_as(dp)  # noqa: E731
    for args, why in (((ptr(q), None, 2 * E - 1, 2, 0), "ngroups * num_elements"),
                      ((ptr(q), None, 2 * E, 0, 0), "ngroups must be >= 1"),
                      ((None, None, 2 * E, 2, 0), "null strength array")):
        def call(a=args):
            if L.pumitally_set_source(eng._h, *a):
                raise RuntimeError("refused")
        refused(call, why)
    def sample_raw(n, first=0):
        if L.pumitally_sample_source(eng._h, 3, first, n, None, None, None, None, 0):
            raise RuntimeError("refused")

    refused(lambda: sample_raw(-1), "n must be >= 0")
    refused(lambda: eng.sample_source(10, 3, first=-5), "first must be >= 0")
    refused(lambda: eng.sample_source(10, 3, first=2 ** 63 - 5), "overflows")
    refused(lambda: eng.sample_source(b.n - 1, 3, place=True), "n must be num_particles")
    refused(lambda: eng.sample_source_device(b.n + 1, 3, place=True), "n must be num_particles")
    # removal, then every call is refused
    eng.set_source(None)
    assert eng.source_groups == 0
    capfd.readouterr()
    with pytest.raises(RuntimeError):
        eng.sample_source(10, 3)
    with pytest.raises(RuntimeError):
        eng.source_strength
    assert "no source is set" in capfd.readouterr().err
    assert_same(before, full_snapshot(b), "removal")


def test_source_survives_resets_batches_configuration_and_checkpoints(tmp_path):
    b = Batches("s1_b3_mo", mode=1, seed=9)
    q, bias = case_table("kuhn", 3, True, b.eng.num_elements)
    b.eng.set_source(q, bias)
    want = b.eng.sample_source(5000, 1)
    b.move()
    b.eng.end_batch()
    plain = str(tmp_path / "plain.ckpt")
    b.eng.set_source(None)
    b.eng.save_checkpoint(plain)
    b.eng.set_source(q, bias)
    withs = str(tmp_path / "with.ckpt")
    b.eng.save_checkpoint(withs)
    with open(plain, "rb") as f1, open(withs, "rb") as f2:
        assert f1.read() == f2.read(), "a checkpoint holds the source"

    def same(label):
        assert b.eng.source_groups == 3, label
        assert_samples(b.eng.sample_source(5000, 1), want, label)

    same("set")
    b.eng.reset_tally()
    same("reset_tally")
    b.move()
    b.eng.end_batch()
    same("end_batch")
    b.eng.load_checkpoint(withs)
    same("checkpoint load")
    for call in (lambda: b.eng.set_scores(2), lambda: b.eng.set_score_bins(2), lambda: b.eng.set_time_bins([0.0, 1.0]),
                 lambda: b.eng.set_moments(0), lambda: b.eng.set_batch_statistics(False),
                 lambda: b.eng.set_collision_estimator(False), lambda: b.eng.set_weight_windows(None)):
        call()
        same("set_*")


def test_vtk_arrays(tmp_path):
    from vtk_reader import read_vtu_cell_data

    b = Batches("s1", mode=0, seed=12)
    b.move()
    piece = lambda p: os.path.join(p, "pieces", "piece_0.vtu")  # noqa: E731
    plain = str(tmp_path / "plain.vtk")
    b.eng.WriteTallyResults(plain)
    with open(piece(plain), "rb") as f:
        plain_bytes = f.read()
    names = list(read_vtu_cell_data(piece(plain)))
    E = b.eng.num_elements
    q, _ = case_table("kuhn", 1, False, E)
    b.eng.set_source(q[0], per_volume=True)
    one = str(tmp_path / "one.vtk")
    b.eng.WriteTallyResults(one)
    cells = read_vtu_cell_data(piece(one))
    assert list(cells)[:len(names)] == names and list(cells)[len(names):] == ["source"]
    np.testing.assert_array_equal(bits(np.asarray(cells["source"]).reshape(-1)), bits(q[0]))
    q3, bias = case_table("kuhn", 3, True, E)
    b.eng.set_source(q3, bias)
    three = str(tmp_path / "three.vtk")
    b.eng.WriteTallyResults(three)
    cells = read_vtu_cell_data(piece(three))
    assert list(cells)[len(names):] == [f"source_g{g}" for g in range(3)]
    for g in range(3):
        np.testing.assert_array_equal(bits(np.asarray(cells[f"source_g{g}"]).reshape(-1)), bits(q3[g]))
    b.eng.set_source(None)
    again = str(tmp_path / "again.vtk")
    b.eng.WriteTallyResults(again)
    with open(piece(again), "rb") as f:
        assert f.read() == plain_bytes


def test_config_c2_placement_matches_localisation():
    """Full-size c2, 10 M particles: a move after placement matches a move on an engine localised by
    CopyInitialPosition at the same points -- the same parent elements, the flux to the parity tolerance."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n = cfg["particles"]
    placed, walked = PumiTally.from_arrays(coords, t2v, n), PumiTally.from_arrays(coords, t2v, n)
    rng = np.random.default_rng(8)
    placed.set_source(rng.uniform(0.0, 1.0, (4, placed.num_elements)), per_volume=True)
    s = torch.cuda.current_stream().cuda_stream
    xyz, elem, group, w = placed.sample_source_device(n, 1234, 0, place=True)
    walked.copy_initial_position_device(xyz.data_ptr(), s)
    torch.cuda.synchronize()
    e_placed, e_walked = placed.elem_ids, walked.elem_ids
    np.testing.assert_array_equal(e_placed, elem.cpu().numpy())
    differ = e_placed != e_walked
    print(f"c2: {int(differ.sum())} of {n} samples on a shared face localised in the neighbour")
    assert differ.sum() <= n * 1e-4
    wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    d = (xyz + (wl.initial_positions() - xyz) * 0.05).contiguous()  # short flights from the sampled points
    f = torch.ones(n, dtype=torch.int8, device="cuda")
    for e in (placed, walked):
        e.move_device(xyz.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(placed.elem_ids, walked.elem_ids)
    assert_flux_close(placed.flux, walked.flux, "c2 placed vs localised")


def test_cxx_program_with_a_source(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SetSource, GetSourceGroups, GetSourceStrength and SampleSource."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "source_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "source_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "SOURCE_OK" in out, out
