"""The batch-statistics arithmetic (batch_stats.cuh: welford_fold, batch_readout) compiled for the host by g++ as a
TEST-ONLY build (tests/host_emul/emul_batch_stats.cpp), against numpy's mean and std(ddof=1) / sqrt(B)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT

_LIB = []


def stats_lib():
    if not _LIB:
        so = os.path.join(HERE, "host_emul", "libptb_batch_stats.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        src = os.path.join(HERE, "host_emul", "emul_batch_stats.cpp")
        deps = [src] + [os.path.join(csrc, h) for h in ("batch_stats.cuh", "walk_core.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off",
                                   "-I", csrc, src, "-o", so])
        L = C.CDLL(so)
        L.ptb_fold_batches.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
        L.ptb_readout.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_int32, C.c_void_p]
        _LIB.append(L)
    return _LIB[0]


def fold(x):
    """x [B, n] -> (mean [n], m2 [n]) by the host build of the fold"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    B, n = x.shape
    mean, m2 = np.empty(n), np.empty(n)
    stats_lib().ptb_fold_batches(x.ctypes.data, B, n, mean.ctypes.data, m2.ctypes.data)
    return mean, m2


def readout(mean, m2, volume, nb, kind):
    out = np.empty(len(mean))
    stats_lib().ptb_readout(mean.ctypes.data, m2.ctypes.data, np.ascontiguousarray(volume).ctypes.data, len(mean),
                            float(nb), kind, out.ctypes.data)
    return out


def numpy_stats(x, volume):
    """mean / volume, std(ddof=1) / sqrt(B) / volume and their ratio (0 where the mean is 0), two-pass"""
    B = x.shape[0]
    m = x.mean(axis=0) / volume
    s = x.std(axis=0, ddof=1) / np.sqrt(B) / volume
    rel = np.divide(s, np.abs(m), out=np.zeros_like(s), where=m != 0)
    return m, s, rel


@pytest.mark.parametrize("B", [2, 3, 8, 50])
def test_random_batches_match_numpy(B):
    rng = np.random.default_rng(B)
    n = 4000
    x = rng.lognormal(0.0, 1.0, (B, n)) * rng.uniform(0.5, 2.0, n)
    x[:, :50] = 0.0                       # never scored: mean 0, relative error 0
    x[:, 50:100] = rng.normal(0.0, 1.0, (B, 50))  # of both signs
    x[:, 100:120] = 3.25                  # the same every batch: error exactly 0
    vol = rng.uniform(0.1, 3.0, n)
    mean, m2 = fold(x)
    want = numpy_stats(x, vol)
    for kind in range(3):
        got = readout(mean, m2, vol, B, kind)
        np.testing.assert_allclose(got, want[kind], rtol=1e-12, atol=1e-14 * np.abs(want[kind]).max(),
                                   err_msg=f"kind {kind}")
    assert (readout(mean, m2, vol, B, 2)[:50] == 0).all()
    assert (m2[100:120] == 0).all() and (readout(mean, m2, vol, B, 1)[100:120] == 0).all()


def test_one_batch_mean_is_the_batch_value():
    x = np.random.default_rng(1).uniform(-1.0, 5.0, (1, 1000))
    mean, m2 = fold(x)
    np.testing.assert_array_equal(mean, x[0])
    assert not m2.any()


def test_ill_conditioned_batches_keep_their_digits():
    """Values 1e8 (1 + 1e-9 u_b): the spread is 1e-9 of the mean.  Sum and sum of squares lose every digit of the
    variance (S2 - S1^2 / B cancels at 1e16 / 1e-2 ~ 1e18 times the rounding of S2); the fold matches the two-pass
    result to 1e-6 relative."""
    rng = np.random.default_rng(7)
    B, n = 20, 500
    u = rng.uniform(-1.0, 1.0, (B, n))
    x = 1e8 * (1.0 + 1e-9 * u)
    vol = np.ones(n)
    mean, m2 = fold(x)
    _, want_s, want_rel = numpy_stats(x, vol)
    s = readout(mean, m2, vol, B, 1)
    np.testing.assert_allclose(s, want_s, rtol=1e-6, atol=0)
    np.testing.assert_allclose(readout(mean, m2, vol, B, 2), want_rel, rtol=1e-6, atol=0)
    s1, s2 = x.sum(axis=0), (x * x).sum(axis=0)
    naive = np.sqrt(np.maximum(s2 - s1 * s1 / B, 0.0) / (B * (B - 1)))
    assert np.median(np.abs(naive - want_s) / want_s) > 0.1  # the naive formula has no correct digit left
