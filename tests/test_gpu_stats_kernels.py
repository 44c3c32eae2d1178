"""The batch-statistics kernels (stats_kernels.cu) called directly, through a test-only C wrapper of their launchers
(tests/gpu_harness/stats_harness.cpp), at the lengths, offsets and rank shares that the engine only reaches on several
GPUs: odd lengths, shares that start at an odd double (the scalar fold), shares that start inside a score record or
hold only padding.  Every result must equal an exactly rounded host reference bit for bit, and every device buffer
carries canaries on both sides that must come back untouched."""
import ctypes as C
import functools
import os
import subprocess
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
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    from pumiumtally_b200 import build as pbuild

    lib = pbuild.build_library()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(pbuild._nvcc())), "include")
    so = str(tmp_path_factory.mktemp("stats_harness") / "libstats_harness.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-fPIC", "-shared",
                           "-I", os.path.join(ROOT, "pumiumtally_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                           "-I", cuda_inc, os.path.join(HERE, "gpu_harness", "stats_harness.cpp"), "-o", so,
                           "-L", os.path.dirname(lib), "-lpumitally", "-Wl,-rpath," + os.path.dirname(lib)])
    L = C.CDLL(so)
    p, i64, i32, f64 = C.c_void_p, C.c_int64, C.c_int32, C.c_double
    L.ptb_test_batch_fold.argtypes = [p, p, p, i64, p, f64, p]
    L.ptb_test_batch_readout.argtypes = [p, p, p, p, p, i64, i32, i32, i32, f64, C.c_int, p]
    L.ptb_test_batch_max_rel_err.argtypes = [p, p, i64, i64, i64, i64, i32, i32, f64, p, p]
    return L


def _stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


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


@gpu
@pytest.mark.parametrize("offs", OFFSETS, ids=[f"x{a}m{b}q{c}" for a, b, c in OFFSETS])
def test_fold_path_follows_alignment(harness, offs):
    """The double2 kernel runs only when x, mean and m2 all start on a 16-byte boundary; otherwise the scalar one."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    n = 257
    x, div, states = _fold_case(n, "random")
    ox, om, oq = offs
    xg, dv = Guarded(x[0], ox), Guarded(div)
    mean, m2 = Guarded(np.zeros(n), om), Guarded(np.zeros(n), oq)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert harness.ptb_test_batch_fold(xg.ptr(), mean.ptr(), m2.ptr(), n, dv.ptr(), 1.0, _stream()) == 0
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "batch_fold_kernel" in e.name]
    want = "batch_fold_kernel<true>" if offs == (0, 0, 0) else "batch_fold_kernel<false>"
    assert len(names) == 1 and want in names[0], names
    assert_bits(mean.values(), states[0][0], "mean")


# ---------------------------------------------------------------------------------------------------------------------
# Readout
# ---------------------------------------------------------------------------------------------------------------------
def score_stride(nscores):
    return 1 if nscores <= 1 else 2 if nscores <= 2 else 4 if nscores <= 4 else 8


@gpu
@pytest.mark.parametrize("moments", [False, True], ids=["m0", "moments"])
@pytest.mark.parametrize("nscores", range(1, 9))
@pytest.mark.parametrize("R", [1, 3, 6])
@pytest.mark.parametrize("E", [1, 7, 719, 100_003])
def test_readout_is_exact(harness, E, R, nscores, moments):
    stride = score_stride(nscores) * (4 if moments else 1)
    rng = np.random.default_rng([E, R, nscores, int(moments)])
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
