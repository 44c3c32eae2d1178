"""The mesh source (source_sample.cuh: source_build, source_mix, source_uniform, source_entry, source_sample) compiled
for the host by g++ with -ffp-contract=off as a TEST-ONLY build (tests/host_emul/emul_source.cpp), against the numpy
restatement of the contract (tests/source_ref.py) bit for bit, on the Kuhn, Delaunay, L-shaped and carved-void meshes.
Then the statistics of the reference at fixed seeds, and the kernel's register budget."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
from scipy import stats

import source_ref as sr
from helpers import HERE, ROOT
from locate_ref import MESHES, barycentric
from pumiumtally_b200 import build as pbuild
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.workload import _NumpyOps

_LIB = []
INF, NAN = float("inf"), float("nan")
_d = C.c_void_p


def src_lib():
    if not _LIB:
        so = os.path.join(HERE, "host_emul", "libptb_source.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        src = os.path.join(HERE, "host_emul", "emul_source.cpp")
        deps = [src] + [os.path.join(csrc, h) for h in ("source_sample.cuh", "walk_core.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off",
                                   "-I", csrc, src, "-o", so])
        L = C.CDLL(so)
        L.ptb_src_mix.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64]
        L.ptb_src_mix.restype = C.c_uint64
        L.ptb_src_uniform.argtypes = [C.c_uint64]
        L.ptb_src_uniform.restype = C.c_double
        L.ptb_src_entry.argtypes = [_d, C.c_int64, C.c_int64, C.c_double]
        L.ptb_src_entry.restype = C.c_int64
        L.ptb_src_build.argtypes = [_d, _d, _d, C.c_int64, C.c_int32, C.c_int32, _d, _d, _d]
        L.ptb_src_build.restype = C.c_char_p
        L.ptb_src_sample.argtypes = [_d, _d, _d, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_uint64,
                                     C.c_uint64, C.c_int64, _d, _d, _d, _d]
        L.ptb_src_sample.restype = None
        _LIB.append(L)
    return _LIB[0]


def build(q, volume, bias=None, per_volume=False):
    """The host build's table: (why, cdf, T, Q, klast)"""
    q = np.ascontiguousarray(q, dtype=np.float64).ravel()
    volume = np.ascontiguousarray(volume, dtype=np.float64)
    b = None if bias is None else np.ascontiguousarray(bias, dtype=np.float64).ravel()
    E = len(volume)
    cdf, tq, kk = np.empty(q.size), np.empty(2), np.empty(2, dtype=np.int64)
    why = src_lib().ptb_src_build(q.ctypes.data, None if b is None else b.ctypes.data, volume.ctypes.data, E,
                                  q.size // E, int(per_volume), cdf.ctypes.data, tq.ctypes.data, kk.ctypes.data)
    return why, cdf, tq[0], tq[1], int(kk[0])


def host_sample(table, bias, coords, t2v, seed, first, n):
    verts = np.ascontiguousarray(np.asarray(coords, dtype=np.float64)[np.asarray(t2v)].reshape(-1, 12))
    C_ = np.ascontiguousarray(table.C)
    b = None if bias is None else np.ascontiguousarray(bias, dtype=np.float64).ravel()
    xyz, w = np.empty((n, 3)), np.empty(n)
    elem, group = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
    src_lib().ptb_src_sample(C_.ctypes.data, None if b is None else b.ctypes.data, verts.ctypes.data, len(C_),
                             table.E, table.klast, table.T, table.Q, seed & sr.MASK, first, n, xyz.ctypes.data,
                             elem.ctypes.data, group.ctypes.data, w.ctypes.data)
    return xyz, elem, group, w


def assert_bits(got, want, label=""):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, label
    np.testing.assert_array_equal(got.view(np.uint8), want.view(np.uint8), err_msg=label)


def strengths(rng, G, E):
    """lognormal strengths with interior, leading and trailing zeros"""
    q = rng.lognormal(0.0, 2.0, (G, E)) * (rng.random((G, E)) < 0.8)
    q[0, :3] = 0.0
    q[-1, -3:] = 0.0
    return q


# ---- random numbers ----------------------------------------------------------------------------------------------
def test_mix_is_the_workload_generator():
    ops = _NumpyOps()
    for seed in (0, 1, 12345, 2 ** 63 + 7, 2 ** 64 - 1):
        ids = np.array([0, 1, 2, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 3, 2 ** 63, 2 ** 64 - 1], dtype=np.uint64)
        for k in range(4):
            z = sr.mix(seed, ids, k)
            assert_bits((z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53, ops.uniform(ids, seed, 0, k))
            assert [src_lib().ptb_src_mix(seed, int(i), k) for i in ids] == [int(x) for x in z]
            assert_bits(np.array([src_lib().ptb_src_uniform(int(x)) for x in z]), sr.uniform(z))


def test_uniform_stays_inside_the_open_interval():
    L = src_lib()
    top, bottom = L.ptb_src_uniform(2 ** 64 - 1), L.ptb_src_uniform(0)
    assert top == 1.0 - 2.0 ** -53 and top < 1.0 and float(sr.uniform(2 ** 64 - 1)) == top
    assert bottom == 2.0 ** -53 and float(sr.uniform(0)) == bottom
    # the mapping the contract rules out rounds the largest z to 1
    assert ((2 ** 53 - 1) + 0.5) * 2.0 ** -53 == 1.0


# ---- the table ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_volume", [False, True])
@pytest.mark.parametrize("biased", [False, True])
def test_table_is_the_sequential_sum(per_volume, biased):
    rng = np.random.default_rng(5)
    G, E = 3, 997
    q, vol = strengths(rng, G, E), rng.uniform(1e-3, 2.0, E)
    b = rng.uniform(0.1, 10.0, (G, E)) if biased else None
    why, cdf, T, Q, klast = build(q, vol, b, per_volume)
    ref = sr.Table(q, vol, b, per_volume)
    assert why is None
    assert_bits(cdf, ref.C)
    assert_bits(np.array([T, Q]), np.array([ref.T, ref.Q]))
    assert klast == ref.klast == G * E - 4


@pytest.mark.parametrize("q_bad, b_bad, msg", [
    (-1.0, None, b"a strength is negative"), (NAN, None, b"a strength"), (INF, None, b"a strength"),
    (-0.0, -1.0, b"a bias is negative"), (1.0, NAN, b"a bias is negative or not finite"), (1.0, INF, b"a bias"),
    (2.0, 0.0, b"a bias is 0 where the strength is > 0")])
def test_bad_entries_are_refused(q_bad, b_bad, msg):
    E = 10
    q, b, vol = np.ones((2, E)), np.ones((2, E)), np.ones(E)
    q[1, 7] = q_bad
    if b_bad is not None:
        b[1, 7] = b_bad
    why = build(q, vol, b if b_bad is not None else None)[0]
    assert why is not None and why.startswith(msg), why


def test_zero_bias_with_zero_strength_and_signed_zero_are_accepted():
    q, b = np.array([0.0, -0.0, 1.0, 0.0]), np.array([0.0, 0.0, 2.0, 5.0])
    why, cdf, T, Q, klast = build(q, np.ones(4), b)
    assert why is None and T == 2.0 and Q == 1.0 and klast == 2


def test_totals_that_are_zero_or_overflow_are_refused():
    vol = np.array([1.0, 2.0])
    assert build(np.zeros(2), vol)[0].startswith(b"the total (biased) strength is 0")
    assert build(np.array([1e308, 1e308]), vol)[0].startswith(b"the total (biased) strength")
    assert build(np.array([1.0, 1e308]), vol, per_volume=True)[0].startswith(b"the total (biased) strength")
    # the biased total overflows, or only the unbiased one does
    assert build(np.array([1e300, 1.0]), vol, np.array([1e10, 1.0]))[0].startswith(b"the total (biased)")
    assert build(np.array([1e308, 1e308]), vol, np.array([0.25, 0.25]))[0].startswith(b"the total strength")


# ---- the entry search --------------------------------------------------------------------------------------------
def entries(table, xs):
    C_ = np.ascontiguousarray(table.C)
    return np.array([src_lib().ptb_src_entry(C_.ctypes.data, len(C_), table.klast, float(x)) for x in xs])


def probe_points(table):
    """every C[k], its neighbours, 0, the smallest positive double, T and the doubles just below it"""
    xs = [0.0, 5e-324, table.T, np.nextafter(table.T, 0.0), np.nextafter(np.nextafter(table.T, 0.0), 0.0)]
    for c in table.C:
        xs += [c, np.nextafter(c, 0.0), np.nextafter(c, INF)]
    return np.array([x for x in xs if 0.0 <= x <= table.T])


@pytest.mark.parametrize("p", [
    [0.0, 0.0, 1.0, 2.0, 0.0, 3.0, 0.0, 0.0],      # leading, interior and trailing zeros
    [1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0],      # one entry first
    [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0],      # one entry last
    [1e-300, 1e300, 1e-300, 0.0, 1e300, 1e-300],   # dynamic range: the small entries are absorbed
    [1e-300, 2e-300, 0.0, 3e-300],
    [3.0, 1e-17, 1e-17, 5.0],                      # entries too small to move the sum are never chosen
])
def test_entry_is_the_first_above_x_and_never_a_zero_entry(p):
    table = sr.Table(np.array(p), np.ones(len(p)))
    xs = probe_points(table)
    got = entries(table, xs)
    np.testing.assert_array_equal(got, table.entry(xs))
    chosen = set(got.tolist())
    assert all(table.p[k] > 0 for k in chosen)
    # x == C[k] takes the next entry up (C[k] > x is strict); x == T takes the last entry with p > 0
    assert entries(table, [table.T])[0] == table.klast
    np.testing.assert_array_equal(got, [min(np.searchsorted(table.C, x, "right"), len(p) - 1)
                                        if np.searchsorted(table.C, x, "right") < len(p) else table.klast for x in xs])


def test_x_rounds_up_to_the_total():
    """u_0 < 1 always, and u_0 T < T for every normal T; a subnormal total has a fixed spacing, so u_0 T rounds up to T
    for u_0 near 1.  Then the last entry with p > 0 is taken, not one past the end."""
    tiny = 5e-324
    table = sr.Table(np.array([0.0, tiny, 2 * tiny, 0.0, 0.0]), np.ones(5))
    assert table.T == 3 * tiny and table.klast == 2
    for u in (1.0 - 2.0 ** -53, float(sr.uniform(2 ** 64 - 1)), 0.9):
        x = u * table.T
        assert x == table.T
        assert entries(table, [x])[0] == 2 == table.entry(np.array([x]))[0]
    # a normal total never rounds up
    for T in (1.0, 3.0, 1.5e300, np.nextafter(2.0, 0.0), 1e-300):
        assert (1.0 - 2.0 ** -53) * T < T


# ---- whole samples -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mesh", list(MESHES))
@pytest.mark.parametrize("groups", [1, 3])
@pytest.mark.parametrize("biased", [False, True])
@pytest.mark.parametrize("per_volume", [False, True])
def test_samples_bit_for_bit(mesh, groups, biased, per_volume):
    coords, t2v = MESHES[mesh]()
    E = len(t2v)
    rng = np.random.default_rng(hash((mesh, groups, biased, per_volume)) % 2 ** 32)
    q = strengths(rng, groups, E)
    b = rng.uniform(0.05, 20.0, (groups, E)) * (rng.random((groups, E)) < 0.95) + (q > 0) * 1e-3 if biased else None
    vol = sr.volumes(coords, t2v)
    table = sr.Table(q, vol, b, per_volume)
    why, cdf, T, Q, klast = build(q, vol, b, per_volume)
    assert why is None
    assert_bits(cdf, table.C)
    for seed, first in ((0, 0), (987654321, 2 ** 32 + 11), (2 ** 64 - 5, 2 ** 40)):
        got = host_sample(table, b, coords, t2v, seed, first, 20_000)
        want = sr.sample(table, coords, t2v, seed, first, 20_000)
        for g, w, what in zip(got, want, ("xyz", "elem", "group", "weight")):
            assert_bits(g, w, f"{mesh} seed {seed} first {first}: {what}")
        assert (q.reshape(groups, E)[got[2], got[1]] > 0).all()
        lam = barycentric(coords, t2v, got[0], got[1])
        assert (lam >= -1e-12).all(), f"{mesh}: a point outside its element"


def test_a_sample_depends_only_on_seed_and_index():
    coords, t2v = MESHES["kuhn"]()
    table = sr.Table(np.ones(len(t2v)), sr.volumes(coords, t2v))
    whole = host_sample(table, None, coords, t2v, 42, 2 ** 33, 3000)
    parts = [host_sample(table, None, coords, t2v, 42, 2 ** 33 + a, b - a) for a, b in ((0, 1000), (1000, 2999),
                                                                                       (2999, 3000))]
    for k in range(4):
        assert_bits(np.concatenate([p[k] for p in parts]), whole[k])


# ---- statistics of the reference (fixed seeds) -------------------------------------------------------------------
def test_counts_follow_the_strengths():
    coords, t2v = kuhn_box(6, 6, 5)
    assert len(t2v) == 1080
    rng = np.random.default_rng(17)
    q = rng.uniform(0.5, 3.0, (2, 1080))
    vol = sr.volumes(coords, t2v)
    table = sr.Table(q, vol, per_volume=True)
    n = 4_000_000
    _, e, g, _ = sr.sample(table, coords, t2v, 2024, 0, n)
    counts = np.bincount(g.astype(np.int64) * 1080 + e, minlength=2160)
    expect = table.p / table.T * n
    chi = stats.chisquare(counts, expect)
    assert chi.pvalue > 1e-3, chi


def test_points_are_uniform_in_the_element():
    coords, t2v = kuhn_box(6, 6, 5)
    table = sr.Table(np.ones(1080), sr.volumes(coords, t2v))
    xyz, e, _, _ = sr.sample(table, coords, t2v, 99, 0, 400_000)
    lam = barycentric(coords, t2v, xyz, e)
    assert (lam >= -1e-12).all()
    for c in range(4):
        ks = stats.kstest(np.clip(lam[:, c], 0.0, 1.0), stats.beta(1, 3).cdf)
        assert ks.pvalue > 1e-3, (c, ks)


def test_biased_weights_are_unbiased():
    coords, t2v = kuhn_box(4, 4, 4)
    E = len(t2v)
    rng = np.random.default_rng(23)
    q = rng.uniform(0.0, 2.0, E) * (rng.random(E) < 0.9)
    b = rng.lognormal(0.0, 1.5, E)
    table = sr.Table(q, sr.volumes(coords, t2v), b)
    n = 2_000_000
    _, e, _, w = sr.sample(table, coords, t2v, 7, 0, n)
    assert abs(w.mean() - 1.0) < 0.01
    mean = np.bincount(e, weights=w, minlength=E) / n
    want = q / table.Q
    ex2 = np.where(q > 0, q * table.T / (table.Q ** 2 * b), 0.0)
    sigma = np.sqrt(np.maximum(ex2 - want ** 2, 0.0) / n)
    assert (np.abs(mean - want) <= 5 * sigma + 1e-15).all()
    assert (mean[q == 0] == 0).all()


# ---- the kernel --------------------------------------------------------------------------------------------------
def test_kernel_does_not_spill(tmp_path):
    cmd = [pbuild._nvcc(), *pbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(pbuild.CSRC, "source_kernels.cu"),
           "-o", str(tmp_path / "source_kernels.o")]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True)
    text = log.stdout + log.stderr
    found = {}
    for block in re.split(r"Compiling entry function '", text)[1:]:
        name = re.search(r"\d(source_[a-z_]+_kernel)E", block.split("'", 1)[0]).group(1)
        s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        found[name] = tuple(int(x) for x in s.groups())
    assert sorted(found) == ["source_sample_kernel"]
    for name, (stack, stores, loads) in found.items():
        assert stack == 0 and stores == 0 and loads == 0, (name, stack, stores, loads)
