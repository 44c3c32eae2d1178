"""Checkpoints (pumitally_save_checkpoint / load_checkpoint / merge_checkpoint): the tally state and the batch statistics
written to a file, restored into a fresh engine and merged across independent runs.  A loaded engine must answer every
accessor with the saving engine's bits; merged statistics must match numpy statistics of all the batches; every refusal
must leave every accessor bit-identical."""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from helpers import ROOT
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload
from test_gpu_batch_stats import MODES, Batches, assert_stats, numpy_stats
from test_gpu_moments import _move
from test_gpu_regions import slab_map
from test_gpu_tally_collisions import CASES

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _try(fn):
    try:
        return fn()
    except (RuntimeError, ValueError):
        return "refused"


def snapshot(b):
    """Every accessor of the engine's tally state, as arrays (a refused accessor as the string "refused")."""
    e = b.eng
    s = {"flux": e.flux_time, "norm": _try(lambda: e.normalized_flux_time()[0]), "coll0": e.collision_results(0),
         "coll1": _try(lambda: e.collision_results(1)), "divisor": np.float64(e.source_normalization())}
    if b.moments:
        s.update(mom=e.flux_moments(), grad=_try(e.flux_gradient), coll2=e.collision_results(2),
                 coll3=_try(lambda: e.collision_results(3)))
    st = e.stats()
    for k in ("segments", "tracks", "relocations", "lost", "moves"):
        s[k] = np.int64(st[k])
    for k in ("collisions", "collisions_outside", "collisions_rejected", "batches"):
        s[k] = np.int64(e.get_option(k))
    B = e.batches
    for t in (0, 1):
        for kind in range(4):
            s[f"batch{t}{kind}"] = _try(lambda: e.batch_results(t, kind))
        s[f"mre{t}"] = _try(lambda: np.array(e.batch_max_rel_err(t, 0), dtype=np.float64))
        if e.regions:
            for kind in range(2):
                s[f"reg{t}{kind}"] = _try(lambda: e.region_results(t, kind))
            for kind in range(3):
                s[f"regb{t}{kind}"] = _try(lambda: e.region_batch_results(t, kind))
    assert B == e.batches
    return s


def as_bits(v):
    v = np.atleast_1d(np.asarray(v))
    return v.view(np.uint64) if v.dtype == np.float64 else v


def assert_same(a, b, label, only=None):
    """a and b (snapshots) hold the same bits; only: the keys compared (default: all, and the same keys)"""
    if only is None:
        assert sorted(a) == sorted(b), label
    for k in sorted(a) if only is None else only:
        if isinstance(a[k], str) or isinstance(b[k], str):
            assert isinstance(a[k], str) and isinstance(b[k], str), f"{label} {k}: refused by one engine only"
        else:
            np.testing.assert_array_equal(as_bits(a[k]), as_bits(b[k]), err_msg=f"{label} {k}")


def stats_only(s):
    return [k for k in s if k.startswith(("batch", "mre", "regb"))]


def engine(case, mode=0, path="host", seed=5, regions=True, stats=True):
    b = Batches(case, mode=mode, path=path, seed=seed, stats=stats)
    if regions:
        b.eng.set_regions(slab_map(b.c, b.t, 5))
    return b


def run(b, batches, mid=False):
    for _ in range(batches):
        b.move()
        b.eng.end_batch()
    if mid:
        b.move()


def file_digest(p):
    import hashlib

    h = hashlib.sha256()
    with open(p, "rb") as f:
        for block in iter(lambda: f.read(1 << 24), b""):
            h.update(block)
    return h.hexdigest()


def read_bytes(p):
    with open(p, "rb") as f:
        return f.read()


@pytest.mark.parametrize("when", ["batch_end", "mid_batch"])
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("case", list(CASES))
def test_round_trip(case, mode, path, when, tmp_path):
    a = engine(case, mode, path, seed=3)
    c = engine(case, mode, path, seed=3)  # never saves
    for x in (a, c):
        run(x, 3, mid=when == "mid_batch")
    before = snapshot(a)
    f1 = str(tmp_path / "a.ckpt")
    a.eng.save_checkpoint(f1)
    assert not os.path.exists(f1 + ".tmp")
    assert_same(before, snapshot(a), "the save changed A")
    b = engine(case, mode, path, seed=3)
    b.eng.load_checkpoint(f1)
    assert_same(before, snapshot(b), "B after load")
    f2 = str(tmp_path / "b.ckpt")
    b.eng.save_checkpoint(f2)
    assert read_bytes(f1) == read_bytes(f2)
    # A after one more batch, against the engine that never saved (moves: atomics, so to rounding)
    for x in (a, c):
        if when == "batch_end":
            x.move()
        x.eng.end_batch()
    sa, sc = snapshot(a), snapshot(c)
    for k in sa:
        if k in ("segments", "tracks", "relocations", "lost", "moves", "collisions", "batches"):
            assert sa[k] == sc[k], k
        elif not isinstance(sa[k], str) and k.startswith(("batch", "regb")):
            np.testing.assert_allclose(sa[k], sc[k], rtol=1e-9, atol=1e-11 * np.nanmax(np.abs(sc[k])), err_msg=k)


def collision_batch(b, rng):
    """One collision event per element, at its centroid: no two events reduce into one address, so the batch has the
    same bits in every engine."""
    cen = np.asarray(b.c)[np.asarray(b.t)].mean(axis=1)
    E = len(cen)
    bins = rng.integers(0, b.nbins, E).astype(np.int32)
    times = None if b.edges is None else rng.uniform(0.0, 4.0, E)
    b.eng.tally_collisions(cen, rng.uniform(0.1, 2.0, E), rng.uniform(0.0, 2.0, (E, b.nscores)), bins, times)
    b.eng.end_batch()


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("case", list(CASES))
def test_exact_continuation(case, mode, tmp_path):
    a = engine(case, mode, seed=8)
    run(a, 4)
    f = str(tmp_path / "four.ckpt")
    a.eng.save_checkpoint(f)
    b = engine(case, mode, seed=8)
    b.eng.load_checkpoint(f)
    for x in (a, b):
        rng = np.random.default_rng(77)
        for _ in range(4):
            collision_batch(x, rng)
    sa, sb = snapshot(a), snapshot(b)
    assert sa["batches"] == 8
    assert_same(sa, sb, f"{case} mode {mode}", only=stats_only(sa))


def captures(b):
    out = b.capture()[:2]
    d = b.eng.source_normalization()
    out += [b.eng.region_results(t, 0) / d for t in (0, 1)]
    return out


@pytest.mark.parametrize("mode", list(MODES))
def test_statistical_continuation_with_moves(mode, tmp_path):
    a = engine("s3_b3_t", mode, seed=21)
    caps = []
    for _ in range(3):
        a.move()
        caps.append(captures(a))
        a.eng.end_batch()
    f = str(tmp_path / "k.ckpt")
    a.eng.save_checkpoint(f)
    b = engine("s3_b3_t", mode, seed=21)
    b.eng.load_checkpoint(f)
    b.wl, b.rng = a.wl, a.rng  # the run continues where A stopped
    for _ in range(4):
        b.move()
        caps.append(captures(b))
        b.eng.end_batch()
    assert b.eng.batches == 7
    vol_r = b.eng.region_volumes()
    for t in (0, 1):
        m, s, rel = numpy_stats(np.array([c[t] for c in caps]))
        for kind, want in enumerate((m, s, rel)):
            assert_stats(b.eng.batch_results(t, kind), want, f"tally {t} kind {kind}")
        m, s, rel = numpy_stats(np.array([c[2 + t] for c in caps]))
        for kind, want in enumerate((m / vol_r, s / vol_r, rel)):
            assert_stats(b.eng.region_batch_results(t, kind), want, f"region tally {t} kind {kind}")


def test_merge_of_three_and_five_batches(tmp_path):
    a = engine("s3_b3_t_mo", 3, seed=31)
    r = engine("s3_b3_t_mo", 3, seed=32)
    caps = []
    for x, k in ((a, 3), (r, 5)):
        for _ in range(k):
            x.move()
            caps.append(captures(x))
            x.eng.end_batch()
    f = str(tmp_path / "r.ckpt")
    r.eng.save_checkpoint(f)
    a.move()  # an open batch in A survives the merge
    open_before = snapshot(a)
    a.eng.merge_checkpoint(f)
    assert a.eng.batches == 8
    after = snapshot(a)
    open_keys = ["flux", "coll0", "mom", "coll2", "segments", "tracks", "relocations", "lost", "moves", "collisions",
                 "reg00", "reg10"]
    assert_same(open_before, after, "the open batch", only=open_keys)
    vol_r = a.eng.region_volumes()
    for t in (0, 1):
        m, s, rel = numpy_stats(np.array([c[t] for c in caps]))
        for kind, want in enumerate((m, s, rel)):
            assert_stats(a.eng.batch_results(t, kind), want, f"tally {t} kind {kind}")
        m, s, rel = numpy_stats(np.array([c[2 + t] for c in caps]))
        for kind, want in enumerate((m / vol_r, s / vol_r, rel)):
            assert_stats(a.eng.region_batch_results(t, kind), want, f"region tally {t} kind {kind}")
    # merged into a fresh engine: the same bits as a load
    fresh, loaded = engine("s3_b3_t_mo", 3, seed=33), engine("s3_b3_t_mo", 3, seed=33)
    fresh.eng.merge_checkpoint(f)
    loaded.eng.load_checkpoint(f)
    sf, sl = snapshot(fresh), snapshot(loaded)
    assert sf["batches"] == 5
    assert_same(sf, sl, "merge into a fresh engine vs load", only=stats_only(sl))
    # a checkpoint of no batches changes nothing
    z = engine("s3_b3_t_mo", 3, seed=34)
    z.eng.reset_tally()
    fz = str(tmp_path / "z.ckpt")
    z.eng.save_checkpoint(fz)
    a.eng.merge_checkpoint(fz)
    assert_same(after, snapshot(a), "merging 0 batches")


def patched(data, off, new):
    """data with bytes [off, off + len(new)) replaced and the header CRC recomputed"""
    d = bytearray(data)
    d[off:off + len(new)] = new
    ne = struct.unpack_from("<I", d, 152)[0]
    end = 156 + 8 * ne
    d[end:end + 4] = struct.pack("<I", zlib.crc32(bytes(d[:end])))
    return bytes(d)


# fingerprint field -> (offset in the file, bytes that differ from what the refusal engine writes)
def field_patches(data):
    u64 = lambda off: struct.unpack_from("<Q", data, off)[0]  # noqa: E731
    i32 = lambda off: struct.unpack_from("<i", data, off)[0]  # noqa: E731
    p = {
        "number of elements": (56, struct.pack("<Q", u64(56) + 1)),
        "number of vertices": (64, struct.pack("<Q", u64(64) + 1)),
        "mesh": (72, struct.pack("<Q", u64(72) ^ 1)),
        "internal element order": (80, struct.pack("<Q", u64(80) ^ 1)),
        "score bins": (88, struct.pack("<i", i32(88) + 1)),
        "scores": (92, struct.pack("<i", i32(92) + 1)),
        "record stride": (96, struct.pack("<i", i32(96) + 1)),
        "moment order": (100, struct.pack("<i", 1 - i32(100))),
        "collision estimator": (104, struct.pack("<i", 1 - i32(104))),
        "batch statistics": (108, struct.pack("<i", 1 - i32(108))),
        "number of regions": (112, struct.pack("<i", i32(112) + 1)),
        "source-normalisation mode": (116, struct.pack("<i", 3 - i32(116))),
        "region map": (120, struct.pack("<Q", u64(120) ^ 1)),
        "source-normalisation value": (128, struct.pack("<d", 38.0)),
        "rank": (136, struct.pack("<i", 1)),
        "number of ranks": (140, struct.pack("<i", 2)),
        "rank share": (144, struct.pack("<Q", 7)),
        "time-bin edges": (156 + 8, struct.pack("<d", np.nextafter(struct.unpack_from("<d", data, 164)[0], 9.0))),
    }
    return p


def test_refusals_change_nothing(tmp_path, capfd):
    a = engine("s3_b3_t_mo", 2, seed=41)  # mode 2: the normalisation value is in the fingerprint
    run(a, 3, mid=True)
    good = str(tmp_path / "good.ckpt")
    a.eng.save_checkpoint(good)
    other = engine("s3_b3_t_mo", 2, seed=42)
    run(other, 2)
    end = str(tmp_path / "end.ckpt")
    other.eng.save_checkpoint(end)
    ref = snapshot(a)
    data = read_bytes(good)

    def refused(fn, why, label):
        capfd.readouterr()
        with pytest.raises(RuntimeError):
            fn()
        err = capfd.readouterr().err
        assert why in err, f"{label}: {err!r}"
        assert_same(ref, snapshot(a), label)

    for field, (off, new) in field_patches(data).items():
        p = str(tmp_path / "f.ckpt")
        with open(p, "wb") as f:
            f.write(patched(data, off, new))
        for fn in (a.eng.load_checkpoint, a.eng.merge_checkpoint):
            if fn == a.eng.merge_checkpoint and field == "source-normalisation value":
                continue  # merge ignores it (below)
            refused(lambda: fn(p), field, f"{field} via {fn.__name__}")
    # merge accepts another mode-2 value (the folded values are per source); load refuses it
    p = str(tmp_path / "v.ckpt")
    with open(p, "wb") as f:
        f.write(patched(read_bytes(end), 128, struct.pack("<d", 38.0)))
    refused(lambda: a.eng.load_checkpoint(p), "source-normalisation value", "load with another value")
    # a real configuration difference, from an engine set up differently
    d = engine("s3_b3_t", 2, seed=43)
    dp = str(tmp_path / "d.ckpt")
    d.eng.save_checkpoint(dp)
    refused(lambda: a.eng.load_checkpoint(dp), "record stride", "another configuration")  # (no moment slots)
    # missing, corrupt and truncated files
    refused(lambda: a.eng.load_checkpoint(str(tmp_path / "missing")), "No such file", "missing")
    for cut in (len(data) - 1, len(data) // 2, 100):
        p = str(tmp_path / "t.ckpt")
        with open(p, "wb") as f:
            f.write(data[:cut])
        refused(lambda: a.eng.load_checkpoint(p), "", f"truncated at {cut}")
    for where in (len(data) - 8, len(data) // 2, 300):
        bad = bytearray(data)
        bad[where] ^= 0x40
        p = str(tmp_path / "c.ckpt")
        with open(p, "wb") as f:
            f.write(bytes(bad))
        refused(lambda: a.eng.load_checkpoint(p), "", f"corrupt at {where}")
    # merges: of an open batch, and into an engine with statistics off
    refused(lambda: a.eng.merge_checkpoint(good), "open batch", "merge of an open batch")
    off = engine("s3_b3_t_mo", 2, seed=44, stats=False)
    ref_off = snapshot(off)
    capfd.readouterr()
    with pytest.raises(RuntimeError):
        off.eng.merge_checkpoint(end)
    assert "statistics are off" in capfd.readouterr().err
    assert_same(ref_off, snapshot(off), "merge with statistics off")
    # a multi-rank checkpoint into a one-rank engine
    p = str(tmp_path / "r.ckpt")
    with open(p, "wb") as f:
        f.write(patched(data, 140, struct.pack("<i", 2)))
    refused(lambda: a.eng.load_checkpoint(p), "number of ranks", "two ranks")
    # saves that fail leave an existing file untouched
    refused(lambda: a.eng.save_checkpoint(str(tmp_path / "no_such_dir" / "x.ckpt")), "cannot create",
            "missing directory")
    os.mkdir(good + ".tmp")  # the temporary file cannot be created
    refused(lambda: a.eng.save_checkpoint(good), "cannot create", "blocked temporary")
    assert read_bytes(good) == data
    # and after all of that, the good file still loads into A, bit for bit
    a.eng.load_checkpoint(good)
    assert_same(ref, snapshot(a), "reload")


def test_config_c2_round_trip(tmp_path):
    """Full-size c2: 8 scores, 16 time bins, the collision estimator and 64 slab regions, round trip at a batch end."""
    import torch

    cfg = CONFIGS["c2"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n = cfg["particles"]
    edges = np.linspace(0.0, 8.0, 17)
    regions = slab_map(coords, t2v, 64)

    def make():
        e = PumiTally.from_arrays(coords, t2v, n)
        e.set_collision_estimator(True)
        e.set_batch_statistics(True)
        e.set_scores(8)
        e.set_time_bins(edges)
        e.set_source_normalization(3)
        e.set_regions(regions)
        return e

    a = make()
    wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    a.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
    g = torch.Generator(device="cuda").manual_seed(5)
    for _ in range(2):
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        r = torch.rand((n, 8), device="cuda", dtype=torch.float64, generator=g)
        t = torch.rand(n, device="cuda", dtype=torch.float64, generator=g) * 6.0
        v = torch.rand(n, device="cuda", dtype=torch.float64, generator=g) + 0.5
        a.move_device_timed(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), t.data_ptr(), v.data_ptr(),
                            r.data_ptr(), None, s)
        torch.cuda.synchronize()
        a.tally_collisions_at_particles_device((f != 0).to(torch.int8), w.to(torch.float64), r, None, t)
        torch.cuda.synchronize()
        a.end_batch()
    p = str(tmp_path / "c2.ckpt")
    a.save_checkpoint(p)
    L = 2 * len(t2v) * 16 * 8
    assert os.path.getsize(p) > 2 * 8 * L
    digest = file_digest(p)
    b = make()
    b.load_checkpoint(p)
    os.remove(p)  # (4 GB: one file at a time)
    assert b.batches == 2
    for tally in (0, 1):
        for kind in range(3):
            np.testing.assert_array_equal(bits(a.batch_results(tally, kind)), bits(b.batch_results(tally, kind)))
            np.testing.assert_array_equal(bits(a.region_batch_results(tally, kind)),
                                          bits(b.region_batch_results(tally, kind)))
    b.save_checkpoint(p)
    assert file_digest(p) == digest


def test_cxx_program_with_checkpoints(tmp_path):
    """A C++ caller of PumiTallyExtras.h: SaveCheckpoint, LoadCheckpoint and MergeCheckpoint."""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    exe = str(tmp_path / "checkpoint_demo")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "checkpoint_demo.cpp"), "-o", exe,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    out = subprocess.check_output([exe], cwd=str(tmp_path), text=True)
    assert "CHECKPOINT_OK" in out, out


def _two_gpu_checkpoint_worker(rank, world, port, directory, q):
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

    def make():
        eng = PumiTally.from_arrays(c, t, n, device=rank)
        eng.set_scores(2)
        eng.set_collision_estimator(True)
        eng.set_batch_statistics(True)
        eng.set_source_normalization(3)
        eng.set_regions(slab_map(c, t, 7))
        eng.comm_init(rank, world, broadcast_unique_id(dist, PumiTally.nccl_unique_id,
                                                       device=torch.device("cuda", rank)))
        return eng

    eng = make()
    wl = SyntheticWorkload(box=(5.0, 5.0, 5.0), num_particles=n, mean_length=1.0, seed=300 + rank)
    eng.CopyInitialPosition(wl.initial_positions().reshape(-1).copy())
    rng = np.random.default_rng(rank)
    for _ in range(4):
        o, d, f, w = wl.next_step()
        _move(eng, "scored", o, d, f, w, rng.uniform(0.0, 1.0, (n, 2)))
        eng.tally_collisions(rng.uniform(0.0, 5.0, (2000, 3)), rng.uniform(0.5, 1.5, 2000),
                             rng.uniform(0.0, 1.0, (2000, 2)))
        eng.end_batch()
    path = os.path.join(directory, f"rank{rank}.ckpt")
    eng.save_checkpoint(path)
    want = [[eng.batch_results(tally, kind) for kind in range(3)] for tally in (0, 1)]
    fresh = make()
    fresh.load_checkpoint(path)
    got = [[fresh.batch_results(tally, kind) for kind in range(3)] for tally in (0, 1)]
    regions = [[fresh.region_batch_results(tally, kind) for kind in range(3)] for tally in (0, 1)]
    q.put((rank, want, got, regions))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpus_per_rank_checkpoints(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() + 113) % 1000
    procs = [ctx.Process(target=_two_gpu_checkpoint_worker, args=(r, 2, port, str(tmp_path), q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank in range(2):
        for tally in (0, 1):
            for kind in range(3):
                np.testing.assert_array_equal(bits(res[rank][1][tally][kind]), bits(res[rank][2][tally][kind]))
                np.testing.assert_array_equal(bits(res[rank][3][tally][kind]), bits(res[0][3][tally][kind]))
