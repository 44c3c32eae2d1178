"""The batch-statistics kernels (stats_kernels.cu) and the weight-window generation (ww_kernels.cu) called directly,
through a test-only C wrapper of their launchers (tests/gpu_harness/stats_harness.cpp), at the lengths, offsets and
rank shares that the engine only reaches on several GPUs: odd lengths, shares that start at an odd double (the scalar
fold and merge), shares that start inside a score record or hold only padding, region plans of several levels, and
weight-window groups up to the engine's limit; and the leakage sums over hull lists of up to 100 003 slots.  Every
result must equal an exactly rounded host reference bit for bit (the leakage: one in the documented order), and every
device buffer carries canaries on both sides that must come back untouched."""
import ctypes as C
import functools
import json
import math
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

from helpers import HERE, ROOT

gpu = pytest.mark.gpu
PAD = 64  # canary entries on each side of every device array
NB_LIST = (1, 2, 37)


# ---------------------------------------------------------------------------------------------------------------------
# Exactly rounded reference.
#
# batch_stats.cuh builds every output from IEEE-rounded operations only.  cuobjdump -sass of stats_kernels.cu.o
# (nvcc -O3, sm_90a, default flags) shows, for welford_fold in both batch_fold_kernel<true> and <false>:
#   d = x - mean                  DADD
#   mean += d / nb                division (MUFU.RCP64H + Newton DFMAs, with the slow-path call: correctly rounded),
#                                 then DADD -- not fused
#   m2 += d * (x - mean)          DADD for x - mean, then ONE DFMA m2 + d * (x - mean)
# and x / *divisor is a correctly rounded division.  The readout and max-relative-error kernels contract nothing:
# nb * (nb - 1) is a DADD then a DMUL, sqrt and the divisions are correctly rounded.  So the only fused operation is
# the m2 update, and numpy's float64 arithmetic (which never contracts) reproduces everything else exactly.
# ---------------------------------------------------------------------------------------------------------------------
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a  # 2^27 + 1
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def fma_exact(a, b, c):
    """round(a * b + c) with one rounding, vectorised: the exact product and sum as error-free pairs, the low part
    rounded to odd, then one round to nearest (Boldo and Melquiond's emulated FMA; no overflow or underflow in the
    data used here).  test_exact_fma_matches_fractions checks it against fractions.Fraction."""
    a, b, c = (np.asarray(v, dtype=np.float64) for v in (a, b, c))
    ph, pl = _two_prod(a, b)
    th, tl = _two_sum(c, ph)
    v, err = _two_sum(tl, pl)
    fix = (err != 0) & ((v.view(np.int64) & 1) == 0)  # inexact and even: the odd neighbour towards the exact value
    v = np.where(fix, np.nextafter(v, np.where(err > 0, np.inf, -np.inf)), v)
    return th + v


def fma_fraction(a, b, c):
    """The definition: the exact rational a * b + c, rounded once to the nearest double by float()."""
    return np.array([float(Fraction(x) * Fraction(y) + Fraction(z)) for x, y, z in zip(a, b, c)])


def fold_ref(x, mean, m2, div, nb):
    """welford_fold(x / div, nb, mean, m2) as the device rounds it."""
    v = x / div
    d = v - mean
    mean = mean + d / nb
    return mean, fma_exact(d, v - mean, m2)


def merge_ref(mean_b, m2_b, na, nb, mean, m2):
    """welford_merge(mean_b, m2_b, na, nb, mean, m2) as the device rounds it (the merge section below)."""
    if nb == 0.0:
        return mean.copy(), m2.copy()
    if na == 0.0:
        return mean_b.copy(), m2_b.copy()
    n = na + nb
    kb, kab = nb / n, (na * nb) / n
    d = mean_b - mean
    return fma_exact(d, kb, mean), fma_exact(d * d, kab, m2 + m2_b)


def merge_unfused(mean_b, m2_b, na, nb, mean, m2):
    """the same update with every product rounded before its sum: what the data must tell apart from merge_ref"""
    n = na + nb
    d = mean_b - mean
    return mean + d * (nb / n), (m2 + m2_b) + (d * d) * ((na * nb) / n)


def std_err_ref(m2, nb):
    return np.sqrt(m2 / (nb * (nb - 1.0)))


def rel_ref(mean, s):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(mean != 0.0, s / np.abs(mean), 0.0)


def readout_ref(mean, m2, vol, orig, E, R, nscores, stride, nb, kind):
    """out[(r * nscores + k) * E + orig[e]] of batch_readout(mean[(r E + e) stride + k], ...)"""
    m = mean.reshape(R, E, stride)[:, :, :nscores].transpose(0, 2, 1) / vol
    if kind == 0:
        val = m
    else:
        with np.errstate(divide="ignore", invalid="ignore"):
            s = std_err_ref(m2.reshape(R, E, stride)[:, :, :nscores].transpose(0, 2, 1), nb) / vol
        val = s if kind == 1 else rel_ref(m, s)
    out = np.empty((R, nscores, E))
    out[:, :, orig] = val
    return out.reshape(-1)


def max_rel_err_ref(mean, m2, base, length, stride, score, nb):
    """(largest relative error, count) over the global m0 slots of `score` in [base, base + length) with a nonzero
    mean"""
    g = np.arange(base + score, base + length, stride)
    g = g[mean[g] != 0.0]
    if not len(g):
        return 0.0, 0
    return float(rel_ref(mean[g], std_err_ref(m2[g], nb)).max()), len(g)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def assert_bits(got, want, label):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.shape == want.shape, label
    if not np.array_equal(bits(got), bits(want)):
        bad = np.flatnonzero(got.view(np.int64) != want.view(np.int64))
        raise AssertionError(f"{label}: {len(bad)} of {got.size} differ, first at {bad[0]}: "
                             f"{got[bad[0]]!r} != {want[bad[0]]!r}")


# ---------------------------------------------------------------------------------------------------------------------
# Harness
# ---------------------------------------------------------------------------------------------------------------------
def build_harness(tmp_path_factory, name):
    """tests/gpu_harness/<name>.cpp compiled against libpumitally.so; returns the path of the shared library"""
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    cuda = os.path.dirname(os.path.dirname(pbuild._nvcc()))
    so = str(tmp_path_factory.mktemp(name) / f"lib{name}.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-fPIC", "-shared",
                           "-I", os.path.join(ROOT, "pumiumtally_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(cuda, "include"), os.path.join(HERE, "gpu_harness", f"{name}.cpp"),
                           "-o", so, "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib),
                           "-L", os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + os.path.join(cuda, "lib64")])
    return so


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return _load_harness(build_harness(tmp_path_factory, "stats_harness"))


def _load_harness(so):
    L = C.CDLL(so)
    p, i64, i32, f64 = C.c_void_p, C.c_int64, C.c_int32, C.c_double
    L.ptb_test_batch_fold.argtypes = [p, p, p, i64, p, f64, p]
    L.ptb_test_batch_readout.argtypes = [p, p, p, p, p, i64, i32, i32, i32, f64, C.c_int, p]
    L.ptb_test_batch_max_rel_err.argtypes = [p, p, i64, i64, i64, i64, i32, i32, f64, p, p]
    L.ptb_test_batch_merge.argtypes = [p, p, p, p, i64, f64, f64, p]
    L.ptb_test_region_sums.argtypes = [p, i64, i32, i32, i32, i64, i64, p, p, C.POINTER(C.c_int), p]
    L.ptb_test_ww_generate.argtypes = [p, p, p, i64, i32, i64, i32, f64, f64, f64, f64, p, p, p]
    L.ptb_test_leakage.argtypes = [p, i64, i32, p, i64, p, p]
    return L


def _stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def run_in_fresh_process(module, func, *args):
    """module.func(*args) (str arguments) run in a new Python process; returns the JSON it printed last.

    The tests that check which kernel a launcher chose use torch.profiler, and in a process that has been running for
    more than about a minute it stops reporting kernels (torch 2.11 on an H100: the runtime API calls are still
    recorded, the kernel launches they made are not).  So such a check cannot run inside a long test session; it runs
    in a process of its own."""
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c",
           f"import sys; sys.path[:0] = {[ROOT, HERE]!r}; import {module}; {module}.{func}(*sys.argv[1:])",
           *map(str, args)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def kernels_launched(fn, pattern):
    """names of the kernels containing `pattern` that fn() launched (in this process: see run_in_fresh_process)"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if pattern in e.name]


class Guarded:
    """A device array of the given values starting `off` entries past a 16-byte boundary, between PAD canary
    entries of random bits on each side."""

    def __init__(self, values, off=0, seed=0):
        import torch

        values = np.ascontiguousarray(values)
        self.n, self.lo, self.dtype = len(values), PAD + off, values.dtype
        size = self.lo + self.n + PAD
        raw = np.frombuffer(np.random.default_rng(seed).bytes(size * values.itemsize), dtype=values.dtype).copy()
        raw[self.lo:self.lo + self.n] = values
        self.host = raw
        self.t = torch.from_numpy(raw.copy()).cuda()
        assert self.t.data_ptr() % 16 == 0

    def ptr(self, k=0):
        return self.t.data_ptr() + (self.lo + k) * self.dtype.itemsize

    def get(self):
        import torch

        torch.cuda.synchronize()
        return self.t.cpu().numpy()

    def values(self, a=0, b=None):
        b = self.n if b is None else b
        return self.get()[self.lo + a:self.lo + b]

    def assert_unchanged_outside(self, a, b, label):
        """Nothing outside entries [a, b) was written: canaries and the rest of the array bit-identical."""
        h = self.get()
        assert np.array_equal(bits(h[:self.lo + a]), bits(self.host[:self.lo + a])), f"{label}: written before {a}"
        assert np.array_equal(bits(h[self.lo + b:]), bits(self.host[self.lo + b:])), f"{label}: written after {b}"


# ---------------------------------------------------------------------------------------------------------------------
# The reference itself
# ---------------------------------------------------------------------------------------------------------------------
def test_exact_fma_matches_fractions():
    rng = np.random.default_rng(3)
    n = 20000
    cases = [
        (rng.normal(0, 1, n), rng.normal(0, 1, n), rng.uniform(0, 5, n)),
        (rng.normal(0, 1e-9, n), rng.normal(0, 1e-9, n), rng.uniform(0, 1e-17, n)),  # Welford on 1e8 (1 + 1e-9 u)
        (rng.normal(0, 1, n), rng.normal(0, 1, n), np.zeros(n)),
    ]
    # products whose low half decides a tie of the sum: c + a b with a b = ulp(c) / 2 (1 +- tiny)
    a = 1.0 + np.ldexp(rng.integers(1, 2**20, n).astype(np.float64), -52)
    c = np.ones(n) + np.ldexp(rng.integers(0, 2, n).astype(np.float64), -52)
    b = np.ldexp(1.0 / a, -53) * np.where(rng.random(n) < 0.5, 1.0, -1.0)
    cases.append((a, b, c))
    for k, (a, b, c) in enumerate(cases):
        assert_bits(fma_exact(a, b, c), fma_fraction(a, b, c), f"case {k}")
    # a fold of ill-conditioned batches takes the fused rounding where it differs from two roundings
    x = 1e8 * (1.0 + 1e-9 * rng.uniform(-1, 1, (12, 2000)))
    mean, m2 = np.zeros(2000), np.zeros(2000)
    differs = 0
    for b in range(12):
        v = x[b] / 1.0
        d = v - mean
        nm = mean + d / (b + 1.0)
        want = fma_fraction(d, v - nm, m2)
        mean, m2 = fold_ref(x[b], mean, m2, 1.0, b + 1.0)
        assert_bits(mean, nm, f"batch {b} mean")
        assert_bits(m2, want, f"batch {b} m2")
        differs += int((want != m2 + d * (v - nm)).sum())
    assert differs > 0


# ---------------------------------------------------------------------------------------------------------------------
# Fold
# ---------------------------------------------------------------------------------------------------------------------
FOLD_N = [0, 1, 2, 3, 255, 256, 257, 4097, "vec-1", "vec", "vec+1", "scalar-1", "scalar", "scalar+1"]
FOLD_DATA = ["random", "negative", "zeros", "ill"]
OFFSETS = [(ox, om, oq) for ox in (0, 1) for om in (0, 1) for oq in (0, 1)]
B_FOLD = 12


def _fold_len(n):
    """Lengths around the grid-stride wrap: the vector path covers 2 x SMs x 8 x 256 doubles per step, the scalar path
    SMs x 8 x 256."""
    if isinstance(n, int):
        return n
    path, _, delta = n.partition("+") if "+" in n else n.partition("-")
    wrap = _sms() * 8 * 256 * (2 if path == "vec" else 1)
    return wrap + (int(delta) if "+" in n else -int(delta) if delta else 0)


CHECKED = (0, 1, B_FOLD - 1)  # batches after which the state is compared


@functools.lru_cache(maxsize=2)  # the offsets vary fastest: eight tests share one reference
def _fold_case(n, data):
    """(x [B, n], divisors [B], {batch b in CHECKED: (mean, m2) after it})"""
    rng = np.random.default_rng([n, FOLD_DATA.index(data)])
    if data == "random":
        x = rng.lognormal(0.0, 1.0, (B_FOLD, n)) * rng.uniform(0.5, 2.0, n)
        x[:, ::7] = rng.normal(0.0, 1.0, (B_FOLD, len(x[0, ::7])))
        x[:, 3::11] = 0.0
    elif data == "negative":
        x = -rng.lognormal(0.0, 2.0, (B_FOLD, n))
    elif data == "zeros":
        x = np.zeros((B_FOLD, n))
    else:  # the spread is 1e-9 of the mean: sum and sum of squares lose every digit
        x = 1e8 * (1.0 + 1e-9 * rng.uniform(-1.0, 1.0, (B_FOLD, n)))
    div = rng.uniform(0.3, 3.0, B_FOLD)
    mean, m2, states = np.zeros(n), np.zeros(n), {}
    for b in range(B_FOLD):
        mean, m2 = fold_ref(x[b], mean, m2, div[b], float(b + 1))
        if b in CHECKED:
            states[b] = (mean, m2)
    return x, div, states


@gpu
@pytest.mark.parametrize("offs", OFFSETS, ids=[f"x{a}m{b}q{c}" for a, b, c in OFFSETS])
@pytest.mark.parametrize("data", FOLD_DATA)
@pytest.mark.parametrize("n", FOLD_N, ids=str)
def test_fold_is_exact(harness, n, data, offs):
    n = _fold_len(n)
    x, div, states = _fold_case(n, data)
    ox, om, oq = offs
    xs = [Guarded(x[b], ox, seed=10 + b) for b in range(B_FOLD)]
    dv = Guarded(div, 1, seed=1)
    mean, m2 = Guarded(np.zeros(n), om, seed=2), Guarded(np.zeros(n), oq, seed=3)
    for b in range(B_FOLD):
        assert harness.ptb_test_batch_fold(xs[b].ptr(), mean.ptr(), m2.ptr(), n, dv.ptr(b), float(b + 1),
                                           _stream()) == 0
        if b in CHECKED:
            label = f"n {n} offsets {offs} {data} batch {b + 1}"
            assert_bits(mean.values(), states[b][0], label + " mean")
            assert_bits(m2.values(), states[b][1], label + " m2")
    for g, what in ((mean, "mean"), (m2, "m2")):
        g.assert_unchanged_outside(0, n, what)
    for g in xs + [dv]:
        g.assert_unchanged_outside(0, 0, "read-only input")
    if data == "zeros":
        assert not mean.values().any() and not m2.values().any()

def _fold_path_case(offs):
    n = 257
    x, div, states = _fold_case(n, "random")
    ox, om, oq = offs
    xg, dv = Guarded(x[0], ox), Guarded(div)
    mean, m2 = Guarded(np.zeros(n), om), Guarded(np.zeros(n), oq)
    return lambda L: L.ptb_test_batch_fold(xg.ptr(), mean.ptr(), m2.ptr(), n, dv.ptr(), 1.0, _stream()), mean, \
        states[0][0]


@gpu
@pytest.mark.parametrize("offs", OFFSETS, ids=[f"x{a}m{b}q{c}" for a, b, c in OFFSETS])
def test_fold_path_follows_alignment(harness, offs):
    """The double2 kernel runs only when x, mean and m2 all start on a 16-byte boundary; otherwise the scalar one."""
    names = _path_kernels(harness._name)["fold"][str(offs)]
    want = "batch_fold_kernel<true>" if offs == (0, 0, 0) else "batch_fold_kernel<false>"
    assert len(names) == 1 and want in names[0], names
    launch, mean, want_mean = _fold_path_case(offs)
    assert launch(harness) == 0
    assert_bits(mean.values(), want_mean, "mean")


# ---------------------------------------------------------------------------------------------------------------------
# Merge (merge_checkpoint: Chan's parallel update of two runs' statistics, in place)
#
# cuobjdump -sass of stats_kernels.cu.o (nvcc -O3, sm_90a, default flags), welford_merge in batch_merge_kernel<false>,
# and in <true> both in its double2 loop and in its odd tail:
#   n = na + nb, then nb / n and (na * nb) / n    DADD; correctly rounded divisions (MUFU.RCP64H + Newton DFMAs with
#                                                 the slow-path call), na * nb a DMUL; hoisted out of the loop
#   s = m2 + m2_b                                 DADD
#   d = mean_b - mean                             DADD
#   mean' = fma(d, nb / n, mean)                  DFMA
#   m2' = fma(d * d, (na * nb) / n, s)            DMUL for d * d, then DFMA
# The nb == 0 and na == 0 selects are FSELs in the tail; in the loops they are branches, hoisted out, to a loop that
# keeps the arrays or copies mean_b and m2_b.  So merge_ref rounds the two updates once each.
# ---------------------------------------------------------------------------------------------------------------------
MERGE_DATA = ["random", "negative", "zeros", "opposite", "ill"]
MERGE_COUNTS = [(0.0, 5.0), (5.0, 0.0), (1.0, 1.0), (3.0, 5.0), (1e6, 1.0), (2.0 ** 40, 3.0)]
OFFSETS4 = [(a, b, c, d) for a in (0, 1) for b in (0, 1) for c in (0, 1) for d in (0, 1)]
FULL_OFFSETS = (257, "scalar")  # every alignment of the four arrays; other lengths: all aligned, or all not
MERGE_CASES = [(n, offs) for n in FOLD_N for offs in (OFFSETS4 if n in FULL_OFFSETS else [(0,) * 4, (1,) * 4])]


@functools.lru_cache(maxsize=2)
def _merge_data(n, data):
    """(mean_b, m2_b, mean, m2): the statistics of the merged run and of the run it is merged into"""
    rng = np.random.default_rng([n, MERGE_DATA.index(data)])
    ln = lambda s: rng.lognormal(0.0, s, n)  # noqa: E731
    if data == "random":
        mean = rng.normal(0.0, 1.0, n) * ln(2.0)
        mean_b = mean * rng.uniform(0.5, 1.5, n) + rng.normal(0.0, 1.0, n)
        m2, m2_b = ln(2.0), ln(2.0)
        mean[::13], m2_b[5::17] = 0.0, 0.0
    elif data == "negative":
        mean, mean_b, m2, m2_b = -ln(2.0), -ln(2.0), ln(2.0), ln(2.0)
    elif data == "zeros":
        mean, mean_b, m2, m2_b = (np.zeros(n) for _ in range(4))
    elif data == "opposite":  # means of opposite sign: d is larger than either
        mean, mean_b, m2, m2_b = ln(1.0), -ln(1.0), ln(2.0), ln(2.0)
    else:  # the spread is 1e-9 of the mean, as in the fold
        mean, mean_b = (1e8 * (1.0 + 1e-9 * rng.uniform(-1.0, 1.0, n)) for _ in range(2))
        m2, m2_b = (0.1 * rng.uniform(0.0, 1.0, n) for _ in range(2))
    return mean_b, m2_b, mean, m2


def test_exact_fma_matches_fractions_on_merges():
    """merge_ref's two fused operations on every kind of merge data, against the exact rational result; and the data
    has elements where one rounding differs from two, so a merge that rounds the product first cannot pass."""
    for data in MERGE_DATA:
        mean_b, m2_b, mean, m2 = _merge_data(4097, data)
        dm = dq = 0
        for na, nb in MERGE_COUNTS:
            if not na or not nb:
                continue
            n = na + nb
            d = mean_b - mean
            args_m, args_q = (d, np.full_like(d, nb / n), mean), (d * d, np.full_like(d, na * nb / n), m2 + m2_b)
            assert_bits(fma_exact(*args_m), fma_fraction(*args_m), f"{data} ({na}, {nb}) mean")
            assert_bits(fma_exact(*args_q), fma_fraction(*args_q), f"{data} ({na}, {nb}) m2")
            got, un = merge_ref(mean_b, m2_b, na, nb, mean, m2), merge_unfused(mean_b, m2_b, na, nb, mean, m2)
            dm += int((got[0] != un[0]).sum())
            dq += int((got[1] != un[1]).sum())
        if data != "zeros":
            assert dq > 0, data
            assert dm > 0 or data == "ill", data  # mean ~ 1e8 against d nb / n ~ 1e-1: the product's rounding is lost


@gpu
@pytest.mark.parametrize("n, offs", MERGE_CASES, ids=[f"{n}-b{a}{b}a{c}{d}" for n, (a, b, c, d) in MERGE_CASES])
@pytest.mark.parametrize("data", MERGE_DATA)  # the offsets of one length vary fastest and share one _merge_data
def test_merge_is_exact(harness, n, offs, data):
    n = _fold_len(n)
    mean_b, m2_b, mean, m2 = _merge_data(n, data)
    ob, qb, om, oq = offs
    gmb, gqb = Guarded(mean_b, ob, seed=1), Guarded(m2_b, qb, seed=2)
    dm = dq = 0
    for na, nb in MERGE_COUNTS:
        label = f"n {n} offsets {offs} {data} (na, nb) = ({na}, {nb})"
        gm, gq = Guarded(mean, om, seed=3), Guarded(m2, oq, seed=4)
        assert harness.ptb_test_batch_merge(gmb.ptr(), gqb.ptr(), gm.ptr(), gq.ptr(), n, na, nb, _stream()) == 0
        want = merge_ref(mean_b, m2_b, na, nb, mean, m2)
        assert_bits(gm.values(), want[0], label + " mean")
        assert_bits(gq.values(), want[1], label + " m2")
        if nb == 0.0:  # a file of no batches: the arrays keep their bits
            assert_bits(gm.values(), mean, label + " kept mean")
            assert_bits(gq.values(), m2, label + " kept m2")
        elif na == 0.0:  # merged into no batches: the file's bits
            assert_bits(gm.values(), mean_b, label + " copied mean")
            assert_bits(gq.values(), m2_b, label + " copied m2")
        else:
            un = merge_unfused(mean_b, m2_b, na, nb, mean, m2)
            dm += int((want[0] != un[0]).sum())
            dq += int((want[1] != un[1]).sum())
        gm.assert_unchanged_outside(0, n, label + " mean")
        gq.assert_unchanged_outside(0, n, label + " m2")
    for g in (gmb, gqb):
        g.assert_unchanged_outside(0, 0, "read-only input")
    if n >= 255 and data != "zeros":  # the data tells the fused update from the twice-rounded one
        assert dq > 0 and (dm > 0 or data == "ill"), (dm, dq)


def _merge_path_case(offs):
    n = 257
    mean_b, m2_b, mean, m2 = _merge_data(n, "random")
    ob, qb, om, oq = offs
    gmb, gqb, gm, gq = Guarded(mean_b, ob), Guarded(m2_b, qb), Guarded(mean, om), Guarded(m2, oq)
    return lambda L: L.ptb_test_batch_merge(gmb.ptr(), gqb.ptr(), gm.ptr(), gq.ptr(), n, 3.0, 5.0, _stream()), gq, \
        merge_ref(mean_b, m2_b, 3.0, 5.0, mean, m2)[1]


PATH_CASES = {"fold": (_fold_path_case, OFFSETS), "merge": (_merge_path_case, OFFSETS4)}


def print_path_kernels(so):
    """(run by run_in_fresh_process) {fold / merge: {offsets: the kernels one launch at those offsets ran}}"""
    L = _load_harness(so)
    res = {}
    for which, (case, offsets) in PATH_CASES.items():
        res[which] = {}
        for offs in offsets:
            launch, _, _ = case(offs)
            res[which][str(offs)] = kernels_launched(lambda: launch(L), f"batch_{which}_kernel")
    print(json.dumps(res))


@functools.lru_cache(maxsize=1)
def _path_kernels(so):
    return run_in_fresh_process("test_gpu_stats_kernels", "print_path_kernels", so)


@gpu
@pytest.mark.parametrize("offs", OFFSETS4, ids=[f"b{a}{b}a{c}{d}" for a, b, c, d in OFFSETS4])
def test_merge_path_follows_alignment(harness, offs):
    """The double2 kernel runs only when mean_b, m2_b, mean and m2 all start on a 16-byte boundary; otherwise the
    scalar one."""
    names = _path_kernels(harness._name)["merge"][str(offs)]
    want = "batch_merge_kernel<true>" if offs == (0, 0, 0, 0) else "batch_merge_kernel<false>"
    assert len(names) == 1 and want in names[0], names
    launch, m2, want_m2 = _merge_path_case(offs)
    assert launch(harness) == 0
    assert_bits(m2.values(), want_m2, "m2")


# ---------------------------------------------------------------------------------------------------------------------
# Readout
# ---------------------------------------------------------------------------------------------------------------------
def score_stride(nscores):
    return 1 if nscores <= 1 else 2 if nscores <= 2 else 4 if nscores <= 4 else 8


READOUT_STRIDES = {  # the record stride of nscores results
    "m0": score_stride,  # the tally's padded records
    "moments": lambda s: 4 * score_stride(s),  # with the three moment slots of each score
    "unpadded": lambda s: s,  # the region statistics: nscores results per record, no padding
}
# (unpadded only where it differs from m0)
READOUT_CASES = [(s, lay) for s in range(1, 9) for lay in READOUT_STRIDES if lay != "unpadded" or score_stride(s) != s]


@gpu
@pytest.mark.parametrize("nscores, layout", READOUT_CASES, ids=[f"{s}-{lay}" for s, lay in READOUT_CASES])
@pytest.mark.parametrize("R", [1, 3, 6])
@pytest.mark.parametrize("E", [1, 7, 719, 100_003])
def test_readout_is_exact(harness, E, R, nscores, layout):
    stride = READOUT_STRIDES[layout](nscores)
    rng = np.random.default_rng([E, R, nscores, list(READOUT_STRIDES).index(layout)])
    size = R * E * stride
    mean = np.full(size, np.nan)  # padding and moment slots: NaN, so reading one shows
    m2 = np.full(size, np.nan)
    slots = (np.arange(size) % stride) < nscores
    k = int(slots.sum())
    mean[slots] = rng.normal(0.0, 1.0, k) * rng.lognormal(0.0, 3.0, k)
    mean[slots] = np.where(rng.random(k) < 0.15, 0.0, mean[slots])  # zero means: relative error 0
    mean[0] = 0.0
    m2[slots] = rng.lognormal(0.0, 3.0, k) * (rng.random(k) > 0.05)
    vol = rng.uniform(0.05, 3.0, E)
    orig = rng.permutation(E).astype(np.int32)
    gm, gq = Guarded(mean, 1, seed=1), Guarded(m2, 1, seed=2)
    gnan = Guarded(np.full(size, np.nan), 1, seed=3)  # kind 0 must not read m2
    gv, go = Guarded(vol, 1, seed=4), Guarded(orig, 1, seed=5)
    for kind in range(3):
        for nb in NB_LIST:
            if nb == 1 and kind:
                continue
            out = Guarded(np.zeros(R * nscores * E), 0, seed=6)
            assert harness.ptb_test_batch_readout(gm.ptr(), (gnan if kind == 0 else gq).ptr(), gv.ptr(), go.ptr(),
                                                  out.ptr(), E, R, nscores, stride, float(nb), kind, _stream()) == 0
            want = readout_ref(mean, m2, vol, orig, E, R, nscores, stride, float(nb), kind)
            assert_bits(out.values(), want, f"kind {kind} nb {nb}")
            out.assert_unchanged_outside(0, out.n, f"out kind {kind} nb {nb}")
            if kind == 2:  # a zero mean has relative error 0, not NaN
                zero = readout_ref(mean, m2, vol, orig, E, R, nscores, stride, float(nb), 0) == 0.0
                assert zero.any() and (out.values()[zero] == 0.0).all()
    for g in (gm, gq, gnan, gv, go):
        g.assert_unchanged_outside(0, 0, "read-only input")


# ---------------------------------------------------------------------------------------------------------------------
# Max relative error, sharded as the engine shards it
# ---------------------------------------------------------------------------------------------------------------------
NRANKS = [1, 2, 3, 4, 5, 7, 8]


def _tally_layout(E, nscores, ntime=1, nbins=1, moments=False):
    """The engine's d_flux_ with the collision estimator: [tally][time][bin][element][stride], tally 1 starting at
    flux_len.  Returns (stride, flux_len, L)."""
    stride = score_stride(nscores) * (4 if moments else 1)
    flux_len = ntime * nbins * E * stride
    return stride, flux_len, 2 * flux_len


def _global_stats(rng, L, stride, nscores):
    """mean / m2 with zero means, means of both signs and zero m2 in the score slots, garbage in the padding and
    moment slots"""
    mean = rng.normal(0.0, 1.0, L) * rng.lognormal(0.0, 2.0, L)
    m2 = rng.lognormal(0.0, 2.0, L)
    m0 = (np.arange(L) % stride) < nscores
    mean[m0 & (rng.random(L) < 0.2)] = 0.0
    m2[m0 & (rng.random(L) < 0.05)] = 0.0
    return mean, m2


def _shares(L, nranks):
    """(lo, n) of every rank: share_ = ceil(L / nranks) entries from lo = rank * share_, n = min(share_, L - lo) or 0"""
    share = -(-L // nranks)
    return share, [(r * share, min(share, L - r * share) if r * share < L else 0) for r in range(nranks)]


def _red_value(red):
    return float(red[0:1].view(np.float64)[0]), int(red[1])


LAYOUTS = {  # E, nscores, ntime, nbins, moments
    "s1": (1001, 1, 1, 1, False),
    "s3_b2": (719, 3, 1, 2, False),
    "s2_mo": (333, 2, 1, 1, True),
    "s5_t3_mo": (97, 5, 3, 1, True),
    "s7_b3": (129, 7, 1, 3, False),
    "wrap": (None, 5, 1, 1, False),  # E > SMs x 8 x 256 m0 slots per tally: the grid-stride loop wraps
}


@gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_max_rel_err_over_rank_shares(harness, layout):
    E, nscores, ntime, nbins, moments = LAYOUTS[layout]
    if E is None:
        E = _sms() * 8 * 256 + 3
    stride, flux_len, L = _tally_layout(E, nscores, ntime, nbins, moments)
    rng = np.random.default_rng(len(layout))
    mean, m2 = _global_stats(rng, L, stride, nscores)
    nb = 7.0
    want = {(t, k): max_rel_err_ref(mean, m2, t * flux_len, flux_len, stride, k, nb)
            for t in (0, 1) for k in range(nscores)}
    assert all(c > 0 for _, c in want.values())
    first = None
    for nranks in NRANKS:
        share, ranks = _shares(L, nranks)
        got = {key: (0.0, 0) for key in want}
        for lo, n in ranks:
            loc_m, loc_q = np.zeros(share), np.zeros(share)  # alloc_stats zeroes; the fold fills [0, n)
            loc_m[:n], loc_q[:n] = mean[lo:lo + n], m2[lo:lo + n]
            gm, gq = Guarded(loc_m, lo % 2), Guarded(loc_q, lo % 2, seed=1)
            red = Guarded(np.zeros(2 * len(want), dtype=np.int64), seed=2)
            for j, (t, k) in enumerate(want):
                assert harness.ptb_test_batch_max_rel_err(gm.ptr(), gq.ptr(), n, lo, t * flux_len, flux_len, stride,
                                                          k, nb, red.ptr(2 * j), _stream()) == 0
            r = red.values()
            red.assert_unchanged_outside(0, red.n, "red")
            for j, key in enumerate(want):
                mx, cnt = _red_value(r[2 * j:2 * j + 2])
                got[key] = (max(got[key][0], mx), got[key][1] + cnt)  # the engine's all-gather: max and sum
            for g in (gm, gq):
                g.assert_unchanged_outside(0, 0, "read-only input")
        for key in want:
            assert got[key][1] == want[key][1], (nranks, key)
            assert_bits(np.array([got[key][0]]), np.array([want[key][0]]), f"{nranks} ranks, (tally, score) {key}")
        first = first or got
        assert got == first


GRID = {1: 99, 2: 25, 4: 11, 8: 5, 16: 2, 32: 1}  # stride -> elements per tally; L = 2 E stride <= 200


@gpu
@pytest.mark.parametrize("stride", list(GRID))
def test_max_rel_err_every_window(harness, stride):
    """Every window [goff, goff + n) of a two-tally array, every score slot of the stride: windows that start inside
    a record, end before the collision tally's base, start past the track-length tally's end, or are empty.  Besides
    the two tallies, a third region [3, L - 2) whose records start at an entry that is not a multiple of the stride:
    the engine's bases always are, so only this region tells (g - base) % stride from g % stride."""
    E = GRID[stride]
    flux_len = E * stride
    L = 2 * flux_len
    assert L <= 200
    regions = [(0, flux_len), (flux_len, flux_len), (3, L - 5)]  # (base, len)
    rng = np.random.default_rng(stride)
    mean, m2 = _global_stats(rng, L, stride, stride)
    nb = 3.0
    gm, gq = Guarded(mean, 1, seed=1), Guarded(m2, 0, seed=2)
    windows = [(goff, n) for goff in range(L + 1) for n in range(L - goff + 1)]
    calls = [(base, ln, k, goff, n) for base, ln in regions for k in range(stride) for goff, n in windows]
    red = Guarded(np.zeros(2 * len(calls), dtype=np.int64), seed=3)
    s = _stream()
    for j, (base, ln, k, goff, n) in enumerate(calls):
        assert harness.ptb_test_batch_max_rel_err(gm.ptr(goff), gq.ptr(goff), n, goff, base, ln, stride, k, nb,
                                                  red.ptr(2 * j), s) == 0
    got = red.values()
    red.assert_unchanged_outside(0, red.n, "red")
    gm.assert_unchanged_outside(0, 0, "mean")
    gq.assert_unchanged_outside(0, 0, "m2")
    got_max = got[0::2].view(np.float64)
    got_cnt = got[1::2]
    # reference: per (region, score) and window start, running max and count over the window's end
    want_max, want_cnt = np.empty(len(calls)), np.empty(len(calls), dtype=np.int64)
    rel = rel_ref(mean, std_err_ref(m2, nb))
    g = np.arange(L)
    j = 0
    for base, ln in regions:
        for k in range(stride):
            elig = (g >= base) & (g < base + ln) & ((g - base) % stride == k) & (mean != 0)
            r = np.where(elig, rel, 0.0)
            for goff in range(L + 1):
                cm = np.concatenate([[0.0], np.maximum.accumulate(r[goff:])])
                cc = np.concatenate([[0], np.cumsum(elig[goff:])])
                want_max[j:j + len(cm)], want_cnt[j:j + len(cc)] = cm, cc
                j += len(cm)
    assert j == len(calls)
    bad = np.flatnonzero((got_cnt != want_cnt) | (got_max.view(np.int64) != want_max.view(np.int64)))
    assert not len(bad), [(calls[i], (got_max[i], got_cnt[i]), (want_max[i], want_cnt[i])) for i in bad[:5]]
    assert (want_cnt > 0).any() and (want_max > 0).any()


# ---------------------------------------------------------------------------------------------------------------------
# Sharded fold and readout
# ---------------------------------------------------------------------------------------------------------------------
SHARD_LAYOUTS = {  # E, nscores, ntime, nbins, moments
    "s3_b2": (719, 3, 1, 2, False),
    "s1_t3_mo": (363, 1, 3, 1, True),
    "s6": (1001, 6, 1, 1, False),
}


@gpu
@pytest.mark.parametrize("layout", list(SHARD_LAYOUTS))
def test_sharded_fold_and_readout_equal_unsharded(harness, layout):
    E, nscores, ntime, nbins, moments = SHARD_LAYOUTS[layout]
    stride, flux_len, L = _tally_layout(E, nscores, ntime, nbins, moments)
    R = ntime * nbins
    rng = np.random.default_rng(E)
    B = 5
    x = rng.normal(1.0, 0.5, (B, L)) * rng.lognormal(0.0, 1.0, L)
    x[:, rng.random(L) < 0.1] = 0.0
    div = rng.uniform(0.5, 2.0, B)
    vol = rng.uniform(0.1, 2.0, E)
    orig = rng.permutation(E).astype(np.int32)
    xs = [Guarded(x[b], 0, seed=b) for b in range(B)]
    dv, gv, go = Guarded(div), Guarded(vol, 1), Guarded(orig, 1)
    s = _stream()

    def readouts(gm, gq):
        res = []
        for t in (0, 1):
            for kind, nb in ((0, B), (1, B), (2, B)):
                out = Guarded(np.zeros(R * nscores * E), seed=9)
                assert harness.ptb_test_batch_readout(gm.ptr(t * flux_len), gq.ptr(t * flux_len), gv.ptr(), go.ptr(),
                                                      out.ptr(), E, R, nscores, stride, float(nb), kind, s) == 0
                out.assert_unchanged_outside(0, out.n, "out")
                res.append(out.values())
        return res

    um, uq = Guarded(np.zeros(L)), Guarded(np.zeros(L), seed=1)
    want_m, want_q = np.zeros(L), np.zeros(L)
    for b in range(B):
        assert harness.ptb_test_batch_fold(xs[b].ptr(), um.ptr(), uq.ptr(), L, dv.ptr(b), float(b + 1), s) == 0
        want_m, want_q = fold_ref(x[b], want_m, want_q, div[b], float(b + 1))
    assert_bits(um.values(), want_m, "unsharded mean")
    assert_bits(uq.values(), want_q, "unsharded m2")
    unsharded = readouts(um, uq)
    for t in (0, 1):
        for j, kind in enumerate(range(3)):
            sl = slice(t * flux_len, (t + 1) * flux_len)
            assert_bits(unsharded[3 * t + j],
                        readout_ref(want_m[sl], want_q[sl], vol, orig, E, R, nscores, stride, float(B), kind),
                        f"unsharded tally {t} kind {kind}")
    for nranks in NRANKS[1:]:
        share, ranks = _shares(L, nranks)
        shards = []
        for lo, n in ranks:  # end_batch: fold this rank's share of the summed batch at d_flux_global_ + lo
            gm, gq = Guarded(np.zeros(share), seed=3), Guarded(np.zeros(share), seed=4)
            for b in range(B):
                assert harness.ptb_test_batch_fold(xs[b].ptr(lo), gm.ptr(), gq.ptr(), n, dv.ptr(b), float(b + 1),
                                                   s) == 0
            gm.assert_unchanged_outside(0, n, f"{nranks} ranks, share at {lo}: mean")
            gq.assert_unchanged_outside(0, n, f"{nranks} ranks, share at {lo}: m2")
            shards.append((gm.values(0, n), gq.values(0, n)))
        cm = np.concatenate([m for m, _ in shards])
        cq = np.concatenate([q for _, q in shards])
        assert_bits(cm, want_m, f"{nranks} ranks: mean")
        assert_bits(cq, want_q, f"{nranks} ranks: m2")
        got = readouts(Guarded(cm, 1, seed=5), Guarded(cq, 1, seed=6))
        for j in range(len(got)):
            assert_bits(got[j], unsharded[j], f"{nranks} ranks: readout {j}")
    for g in xs + [dv, gv, go]:
        g.assert_unchanged_outside(0, 0, "read-only input")


# ---------------------------------------------------------------------------------------------------------------------
# Region sums (batch_stats.cuh, the documented order; launch_region_sums through the product's build_region_plan)
# ---------------------------------------------------------------------------------------------------------------------
CHUNK = 32  # kRegionChunk
U = 2.0 ** -53


def region_sums_ref(region, nregions, values, reverse=False):
    """values [E, K] summed over the regions of region[E] in the documented order: a region's elements in ascending
    internal id, cut into chunks of CHUNK consecutive inputs, each chunk summed left to right (reverse: right to
    left), level after level until one value per region is left.  Returns ([nregions, K], levels)."""
    values = np.asarray(values, dtype=np.float64).reshape(len(region), -1)
    ids = np.flatnonzero(region >= 0)
    ids = ids[np.argsort(region[ids], kind="stable")]  # ascending region, then ascending id
    x, n = values[ids], np.bincount(region[ids], minlength=nregions)
    levels = 0
    while True:
        levels += 1
        c = np.where(n > CHUNK, -(-n // CHUNK), 1)
        g = np.repeat(np.arange(nregions), c)  # region of every chunk
        j = np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c)  # its index within the region
        lo = (np.cumsum(n) - n)[g] + CHUNK * j
        ln = np.clip(n[g] - CHUNK * j, 0, CHUNK)
        acc = np.zeros((len(g), x.shape[1]))
        acc[ln > 0] = x[lo[ln > 0] + (ln[ln > 0] - 1 if reverse else 0)]
        for i in range(1, CHUNK):
            t = ln > i
            acc[t] = acc[t] + x[lo[t] + (ln[t] - 1 - i if reverse else i)]
        x, n = acc, c
        if (c == 1).all():
            return x, levels


def _shuffled_map(rng, sizes, unassigned):
    """region of every internal id: sizes[g] elements in region g and `unassigned` in none (-1), shuffled"""
    region = np.concatenate([np.repeat(np.arange(len(sizes), dtype=np.int32), sizes),
                             np.full(unassigned, -1, dtype=np.int32)])
    return rng.permutation(region), len(sizes)


REGION_SIZES = [0, 1, 31, 32, 33, 1023, 1024, 1025, 32769]  # 32769 takes four levels


@functools.lru_cache(maxsize=1)
def _region_map(name):
    """(region of every internal id, nregions, levels)"""
    rng = np.random.default_rng(len(name))
    if name == "sizes":
        region, nreg = _shuffled_map(rng, REGION_SIZES, 501)
        return region, nreg, 4
    if name == "singletons":
        return rng.permutation(4099).astype(np.int32), 4099, 1
    return np.zeros(33 * 1024 + 7, dtype=np.int32), 1, 4  # one region of every element


def _cancelling(rng, shape):
    """O(1) terms with +-1e16 among them: the order of a sum decides which of them survive"""
    v = rng.normal(0.0, 1.0, shape) * rng.lognormal(0.0, 1.0, shape)
    big = rng.random(shape) < 0.03
    v[big] = np.where(rng.random(int(big.sum())) < 0.5, 1e16, -1e16)
    return v


def test_region_reference_within_the_fsum_bound():
    """region_sums_ref against math.fsum: each level adds at most CHUNK terms left to right, so the error is at most
    h u / (1 - h u) * sum |x| with h = levels * (CHUNK - 1); and the order is not fsum's, nor the reversed one."""
    rng = np.random.default_rng(11)
    for name in ("sizes", "singletons", "one"):
        region, nreg, levels = _region_map(name)
        x = _cancelling(rng, len(region))
        got, lv = region_sums_ref(region, nreg, x)
        rev, _ = region_sums_ref(region, nreg, x, reverse=True)
        assert lv == levels, name
        h = levels * (CHUNK - 1)
        apart = 0
        for g in range(nreg):
            xs = x[region == g]
            want = math.fsum(xs)
            assert abs(got[g, 0] - want) <= h * U / (1 - h * U) * math.fsum(np.abs(xs)), (name, g)
            apart += got[g, 0] != want and got[g, 0] != rev[g, 0]
        assert apart > 0 or name != "sizes", name  # (one region may happen to agree with one of them)
    # one region of 33 elements in two chunks: ((x0 + ... + x31) + x32), summed left to right within the first
    x = np.array([1e16, 1.0, -1e16] + [0.5] * 29 + [3.0])
    got, lv = region_sums_ref(np.zeros(33, dtype=np.int32), 1, x)
    assert lv == 2 and got[0, 0] == ((1e16 + 1.0) - 1e16 + 0.5 * 29) + 3.0


@gpu
@pytest.mark.parametrize("gap", [False, True], ids=["packed", "gap"])
@pytest.mark.parametrize("narrays", [1, 3, 6])
@pytest.mark.parametrize("nscores", range(1, 9))
@pytest.mark.parametrize("name", ["sizes", "singletons", "one"])
def test_region_sums_are_exact(harness, name, nscores, narrays, gap):
    region, nreg, levels = _region_map(name)
    E = len(region)
    stride = score_stride(nscores)
    pitch = E * stride + (5 if gap else 0)
    rng = np.random.default_rng([levels, nscores, narrays, int(gap)])
    vals = _cancelling(rng, (narrays, E, nscores))
    vals[:, region < 0] = np.nan  # elements in no region must not reach a sum
    if name == "sizes":  # the one-element region is its value, -0.0 included
        vals[0, np.flatnonzero(region == 1)[0], 0] = -0.0
    src = np.full(narrays * pitch, np.nan)  # padding slots and the gap: NaN
    for a in range(narrays):
        src[a * pitch:a * pitch + E * stride].reshape(E, stride)[:, :nscores] = vals[a]
    gs = Guarded(src, 1, seed=1)
    out = Guarded(np.full(narrays * nreg * nscores, np.nan), seed=2)
    nlevels = C.c_int(-1)
    assert harness.ptb_test_region_sums(region.ctypes.data, E, nreg, nscores, stride, narrays, pitch, gs.ptr(),
                                        out.ptr(), C.byref(nlevels), _stream()) == 0, "scratch canary"
    assert nlevels.value == levels
    want, lv = region_sums_ref(region, nreg, vals.transpose(1, 0, 2))  # [nregions, narrays * nscores]
    assert lv == levels
    want = want.reshape(nreg, narrays, nscores).transpose(1, 0, 2).reshape(-1)
    got = out.values()
    assert_bits(got, want, f"{name} nscores {nscores} narrays {narrays} gap {gap}")
    out.assert_unchanged_outside(0, out.n, "out")
    gs.assert_unchanged_outside(0, 0, "read-only input")
    assert not np.isnan(got).any()
    got = got.reshape(narrays, nreg, nscores)
    if name == "sizes":
        assert np.signbit(got[0, 1, 0]) and got[0, 1, 0] == 0.0
        empty = got[:, 0, :]  # region 0 holds no element: +0.0
        assert (empty.view(np.int64) == 0).all()
        rev, _ = region_sums_ref(region, nreg, vals.transpose(1, 0, 2), reverse=True)
        rev = rev.reshape(nreg, narrays, nscores).transpose(1, 0, 2)
        fs = np.array([[[math.fsum(vals[a, region == g, k]) for k in range(nscores)] for g in range(nreg)]
                       for a in range(narrays)])
        assert ((got != rev) & (got != fs)).any()  # the order is checked, not just a sum
    if name == "singletons":
        assert_bits(got, vals[:, np.argsort(region), :], "every element its own region")


# ---------------------------------------------------------------------------------------------------------------------
# Weight windows (weight_windows.cuh, ww_kernels.cu): the MAGIC step over raw mean, m2 and volume
# ---------------------------------------------------------------------------------------------------------------------
def ww_ref(mean, m2, vol, nb, max_rel_err, ratio):
    """(phimax [G], lower [G, E], upper [G, E]) of the m0 values mean, m2 [G, E]: phi and r are batch_readout kinds
    0 and 2, eligible where phi is finite and > 0 and r <= max_rel_err; lower = (phi / phimax) * c, upper =
    lower * ratio with c = 2 / (ratio + 1); (-1, -1) where not eligible, phimax 0 for a group with no eligible
    element."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        phi = mean / vol
        r = rel_ref(phi, std_err_ref(m2, nb) / vol)
        ok = (phi > 0.0) & (phi <= np.finfo(np.float64).max) & (r <= max_rel_err)
        pm = np.where(ok, phi, 0.0).max(axis=1)
        lo = (phi / pm[:, None]) * (2.0 / (ratio + 1.0))
        hi = lo * ratio
    return pm, np.where(ok, lo, -1.0), np.where(ok, hi, -1.0)


WW_GROUPS = [1, 3, 16, 4096]
WW_E = [1, 5, 31, 257, 100_003]
WW_CASES = [(G, E) for G in WW_GROUPS for E in WW_E if (G, E) != (4096, 100_003)]  # 4096 x 100003 x 16 B: 6.5 GB
WW_CALLS = [(5.0, float("inf")), (2.0, 0.3), (1.0 + 2.0 ** -40, 0.05), (1e6, 1.0)]  # (ratio, max_rel_err)
NB_WW = 6.0


def _peak(g, E):
    """where group g's largest phi lies.  Group 0: the last element, in the last grid-stride step when one block
    strides over the mesh.  Group g > 0: the last element at thread 255 - 33 ((g - 1) % 8) of a 256-thread block,
    so that the maxima of groups 1 to 8 lie in warps 7 down to 0."""
    o = 255 - 33 * ((g - 1) % 8)
    if g == 0 or E - 1 < o:
        return (E - 1) if g == 0 else (g - 1) % E
    return (E - 1) - ((E - 1 - o) % 256)


def _ww_case(rng, G, E, stride, score, gap, base):
    """(mean array, m2 array, volumes, mean [G, E], m2 [G, E], pitch): mean and m2 of group b and element e at
    base + b * pitch + e * stride + score, NaN in every other slot.  phi spans 6 decades across groups.  A tenth of
    the elements have a phi of 0, -0.0, -1, NaN or +-inf, a tenth a relative error of 10; the others up to 0.25.
    Each group's largest phi is at _peak, with a relative error of 0.01: eligible under every limit of WW_CALLS."""
    pitch = E * stride + gap
    vol = rng.uniform(0.05, 3.0, E)
    phi = rng.uniform(0.5, 1.0, (G, E)) * 10.0 ** rng.integers(-3, 3, (G, 1))
    rel = rng.uniform(0.0, 0.25, (G, E))
    special, high_r = rng.random((G, E)) < 0.1, rng.random((G, E)) < 0.1
    for g in range(G):
        p = _peak(g, E)
        phi[g, p], rel[g, p], special[g, p], high_r[g, p] = 1.5 * phi[g].max(), 0.01, False, False
    rel[high_r] = 10.0
    mean = phi * vol
    m2 = (rel * mean) ** 2 * NB_WW * (NB_WW - 1.0)
    mean[special] = rng.choice(np.array([0.0, -0.0, -1.0, np.nan, np.inf, -np.inf]), int(special.sum()))
    arr, arr2 = np.full(base + G * pitch, np.nan), np.full(base + G * pitch, np.nan)
    idx = base + np.arange(G)[:, None] * pitch + np.arange(E)[None, :] * stride + score
    arr[idx], arr2[idx] = mean, m2
    return arr, arr2, vol, mean, m2, pitch


def _ww_run(harness, gm, gq, gv, base, score, E, G, pitch, stride, mean, m2, vol, mre, ratio, label):
    """one launch_ww_generate on the m0 values at gm / gq + base + score, checked bit for bit against ww_ref, with
    canaries on red and the table; returns ww_ref's (phimax, lower, upper)"""
    red = Guarded(np.random.default_rng(G).integers(0, 2 ** 63, G).astype(np.uint64), seed=7)  # zeroed first
    table = Guarded(np.full(2 * G * E, np.nan), seed=8)
    assert harness.ptb_test_ww_generate(gm.ptr(base + score), gq.ptr(base + score), gv.ptr(), E, G, pitch, stride,
                                        NB_WW, mre, 2.0 / (ratio + 1.0), ratio, red.ptr(), table.ptr(),
                                        _stream()) == 0
    pm, lo, hi = ww_ref(mean, m2, vol, NB_WW, mre, ratio)
    assert_bits(red.values().view(np.float64), pm, label + " group maxima")
    got = table.values().reshape(G, E, 2)
    assert_bits(got[:, :, 0], lo, label + " lower")
    assert_bits(got[:, :, 1], hi, label + " upper")
    red.assert_unchanged_outside(0, G, label + " red")
    table.assert_unchanged_outside(0, table.n, label + " table")
    return pm, lo, hi


@gpu
@pytest.mark.parametrize("stride", [1, 2, 4, 8])
@pytest.mark.parametrize("G, E", WW_CASES, ids=[f"g{G}-e{E}" for G, E in WW_CASES])
def test_ww_generate_is_exact(harness, G, E, stride):
    rng = np.random.default_rng([G, E, stride])
    score = (G + E) % stride
    gap = 3 if stride % 2 else 0  # a pitch with a gap, or E * stride
    base = 2 * E * stride + 1  # a time bin's base, taken by pointer: odd, so the arrays start at an odd double
    arr, arr2, vol, mean, m2, pitch = _ww_case(rng, G, E, stride, score, gap, base)
    gm, gq, gv = Guarded(arr, 0, seed=1), Guarded(arr2, 1, seed=2), Guarded(vol, 1, seed=3)
    for ratio, mre in WW_CALLS:
        label = f"G {G} E {E} stride {stride} ratio {ratio} max_rel_err {mre}"
        pm, lo, _ = _ww_run(harness, gm, gq, gv, base, score, E, G, pitch, stride, mean, m2, vol, mre, ratio, label)
        peaks = [_peak(g, E) for g in range(G)]
        assert (pm == mean[range(G), peaks] / vol[peaks]).all(), label
        assert (lo[range(G), peaks] == 2.0 / (ratio + 1.0)).all(), label
    for g in (gm, gq, gv):
        g.assert_unchanged_outside(0, 0, "read-only input")


@gpu
@pytest.mark.parametrize("E", [1, 5, 257, 100_003])
def test_ww_generate_edges(harness, E):
    """r at the limit and one ulp below it; an infinite limit with an infinite r; phi of 0, -0.0, negative, NaN and
    +-inf; a group whose only eligible element is the last; a group with none; tied maxima."""
    G = 5
    rng = np.random.default_rng(E)
    vol = rng.uniform(0.5, 2.0, E)
    vol[-1] = vol[0]  # the tie of group 3: equal means in equal volumes
    mean = rng.uniform(0.1, 1.0, (G, E)) * vol
    specials = np.array([0.0, -0.0, -2.0, np.nan, np.inf, -np.inf])
    for g in (1, 2):  # group 1: every element ineligible but the last; group 2: none eligible
        mean[g] = specials[np.arange(E) % len(specials)]
    mean[1, -1] = 0.25 * vol[-1]
    mean[3, 0] = mean[3, -1] = 4.0 * vol[0]  # group 3: the largest phi twice, at the first and the last element
    # group 4: the largest phi has an infinite relative error (m2 = inf), the next largest is element k, whose relative
    # error of 0.1 is the largest of all the others (0.01)
    k = E // 2
    mean[4, -1], mean[4, k] = 8.0 * vol[-1], 6.0 * vol[k]
    with np.errstate(invalid="ignore", over="ignore"):
        m2 = (0.01 * mean) ** 2 * NB_WW * (NB_WW - 1.0)
    m2[4, k] = (0.1 * mean[4, k]) ** 2 * NB_WW * (NB_WW - 1.0)
    m2[4, -1] = np.inf
    phi_k = mean[4, k] / vol[k]
    r_k = float(rel_ref(np.array([phi_k]), std_err_ref(np.array([m2[4, k]]), NB_WW) / vol[k])[0])
    gm, gq, gv = Guarded(mean.reshape(-1), 1, seed=1), Guarded(m2.reshape(-1), 0, seed=2), Guarded(vol, 0, seed=3)
    seen = []
    for mre in (float("inf"), r_k, np.nextafter(r_k, 0.0)):
        label = f"E {E} max_rel_err {mre!r}"
        pm, lo, hi = _ww_run(harness, gm, gq, gv, 0, 0, E, G, E, 1, mean, m2, vol, mre, 3.0, label)
        assert pm[1] == 0.25 and (lo[1, :-1] == -1.0).all() and lo[1, -1] == 0.5, label
        assert pm[2] == 0.0 and (lo[2] == -1.0).all() and (hi[2] == -1.0).all(), label
        if E > 1:
            assert pm[3] == 4.0 and lo[3, 0] == lo[3, -1] == 0.5, label
        seen.append(pm[4])
    if E > 1:  # inf: the infinite r counts; r_k: the element at the limit does; one ulp below r_k: it does not
        assert seen[0] == 8.0 and seen[1] == phi_k and seen[2] < phi_k, seen


# ---------------------------------------------------------------------------------------------------------------------
# Leakage (stats_kernels.cu, leakage_kernel): the documented order of the hull sums
# ---------------------------------------------------------------------------------------------------------------------
LEAK_BLOCK = 256  # kLeakBlock
LEAK_NHULL = [0, 1, 255, 256, 257, 511, 1027, 100_003]
LEAK_CASES = [(E, nh) for E in (1, 1000, 300_007) for nh in LEAK_NHULL if nh <= 4 * E]
CANARY = np.array([0x7ff5a5a5c3c3e1e1], dtype=np.uint64).view(np.float64)[0]  # a signalling NaN


def leakage_ref(cur, hull, threads=LEAK_BLOCK):
    """out[r] of launch_leakage over cur [R, 4E] in the documented order: thread k of array r's block adds
    cur[r, hull[k + threads j]] for j = 0, 1, ... left to right, starting from +0.0; then part[t] += part[t + h] for
    h = threads / 2, ..., 1."""
    J = -(-len(hull) // threads)
    idx = np.zeros(J * threads, dtype=np.int64)
    idx[:len(hull)] = hull
    with np.errstate(invalid="ignore"):
        vals = np.where(np.arange(J * threads) < len(hull), cur[:, idx], 0.0)  # +0.0 + x is x (and never -0.0)
        part = np.zeros((len(cur), threads))
        for j in range(J):
            part = part + vals[:, j * threads:(j + 1) * threads]
        h = threads // 2
        while h:
            part[:, :h] = part[:, :h] + part[:, h:2 * h]
            h //= 2
    return part[:, 0]


def kuhn_hull_slots(n):
    """the hull slots 4 e + f, ascending, of kuhn_box(n, n, n) as ensure_face_maps lists them: face f of a tet is the
    one opposite its vertex f, and a face no other tet shares lies on the hull"""
    from pumiumtally_b200.mesh import kuhn_box

    _, t2v = kuhn_box(n, n, n)
    faces = np.sort(np.stack([np.delete(t2v, f, axis=1) for f in range(4)], axis=1).reshape(-1, 3), axis=1)
    _, inv, cnt = np.unique(faces, axis=0, return_inverse=True, return_counts=True)
    return len(t2v), np.flatnonzero(cnt[inv.reshape(-1)] == 1).astype(np.uint32)


def _leak_case(E, R, nhull, order, seed=0):
    """(cur [R, 4E] with signalling-NaN canaries in every slot that is not a hull slot, hull): data of mixed magnitudes
    (1e-8 to 1e8) and signs; with R > 3, arrays 1, 2 and 3 hold a NaN, +inf with -inf, and only -0.0"""
    rng = np.random.default_rng([E, R, nhull, order == "shuffled", seed])
    if order == "kuhn":
        E, hull = kuhn_hull_slots(E)
        nhull = len(hull)
    else:
        hull = np.sort(rng.choice(4 * E, nhull, replace=False)).astype(np.uint32)
        if order == "shuffled":
            hull = rng.permutation(hull)
    cur = np.full((R, 4 * E), CANARY)
    cur[:, hull] = np.where(rng.random((R, nhull)) < 0.5, -1.0, 1.0) * 10.0 ** rng.uniform(-8, 8, (R, nhull))
    if R > 3 and nhull >= 2:
        cur[1, hull[rng.integers(nhull)]] = np.nan
        a, b = rng.choice(nhull, 2, replace=False)
        cur[2, hull[a]], cur[2, hull[b]] = np.inf, -np.inf
        cur[3, hull] = -0.0
    return E, cur, hull


def assert_leak(got, want, label):
    """bit for bit, except that a NaN is only a NaN (the device's NaN of inf - inf is not the host's)"""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{label}: NaN at {np.flatnonzero(np.isnan(got))}, want {nan}"
    assert_bits(got[~nan], want[~nan], label)


def test_leakage_reference_tells_the_order_apart():
    """The documented order differs, on many arrays, from numpy's pairwise sum, from a sequential sum and from the
    same scheme with 128 threads; on the special arrays it gives NaN, NaN and +0.0."""
    E, cur, hull = _leak_case(300_007, 40, 100_003, "shuffled")
    want = leakage_ref(cur, hull)
    normal = np.r_[0, 4:40]
    vals = cur[normal][:, hull]
    others = {"np.sum": vals.sum(axis=1), "sequential": np.cumsum(vals, axis=1)[:, -1],
              "128 threads": leakage_ref(cur, hull, threads=128)[normal]}
    for name, o in others.items():
        assert (o != want[normal]).sum() >= len(normal) // 2, name
    assert np.isnan(want[1]) and np.isnan(want[2]) and want[3] == 0.0 and not np.signbit(want[3])
    exact = [math.fsum(v) for v in vals]  # and it is a sum: each term goes through at most J + 8 additions
    h = -(-len(hull) // LEAK_BLOCK) + 8
    bound = h * U / (1 - h * U) * np.abs(vals).sum(axis=1)
    assert (np.abs(want[normal] - exact) <= bound).all()


@gpu
@pytest.mark.parametrize("order", ["ascending", "shuffled"])
@pytest.mark.parametrize("R", [1, 3, 40])
@pytest.mark.parametrize("E, nhull", LEAK_CASES, ids=[f"e{E}-h{nh}" for E, nh in LEAK_CASES])
def test_leakage_is_exact(harness, E, nhull, R, order):
    _leakage_run(harness, E, R, nhull, order)


@gpu
@pytest.mark.parametrize("R", [1, 3, 40])
def test_leakage_of_a_kuhn_box_hull(harness, R):
    _leakage_run(harness, 20, R, 0, "kuhn")


def _leakage_run(harness, E, R, nhull, order):
    E, cur, hull = _leak_case(E, R, nhull, order)
    label = f"E {E} R {R} nhull {len(hull)} {order}"
    gc, gh = Guarded(cur.reshape(-1), 1, seed=1), Guarded(hull, 1, seed=2)
    out = Guarded(np.full(R, np.nan), seed=3)
    assert harness.ptb_test_leakage(gc.ptr(), E, R, gh.ptr(), len(hull), out.ptr(), _stream()) == 0
    want = leakage_ref(cur, hull)
    assert_leak(out.values(), want, label)
    out.assert_unchanged_outside(0, R, label + " out")
    for g in (gc, gh):
        g.assert_unchanged_outside(0, 0, label + " read-only input")
    if not len(hull):
        assert (out.values().view(np.int64) == 0).all(), label  # nothing to add: +0.0
    if R > 3 and len(hull) >= 2:
        got = out.values()
        assert np.isnan(got[1]) and np.isnan(got[2]) and got[3] == 0.0 and not np.signbit(got[3]), label
