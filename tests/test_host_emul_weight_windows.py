"""The weight-window arithmetic (weight_windows.cuh: ww_entry, ww_max_candidate, ww_generate, ww_slot) compiled for the
host by g++ with -ffp-contract=off as a TEST-ONLY build (tests/host_emul/emul_weight_windows.cpp), against numpy bit
for bit: the MAGIC windows are phi / phimax * 2 / (ratio + 1) and that times ratio, in that order of operations, where
phi and its relative error are what pumitally_get_batch_results returns.  The same file compiles ww_kernels.cu with
-Xptxas -v: its kernels must not spill."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT
from pumiumtally_b200 import build as pbuild

_LIB = []
INF, NAN = float("inf"), float("nan")


def ww_lib():
    if not _LIB:
        so = os.path.join(HERE, "host_emul", "libptb_weight_windows.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        src = os.path.join(HERE, "host_emul", "emul_weight_windows.cpp")
        deps = [src] + [os.path.join(csrc, h) for h in ("weight_windows.cuh", "batch_stats.cuh", "walk_core.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off",
                                   "-I", csrc, src, "-o", so])
        L = C.CDLL(so)
        L.ptb_ww_generate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_double, C.c_double,
                                      C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ptb_ww_generate.restype = None
        L.ptb_ww_entry.argtypes = [C.c_double, C.c_double]
        L.ptb_ww_entry.restype = C.c_int32
        L.ptb_ww_slot.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int64]
        L.ptb_ww_slot.restype = C.c_int64
        L.ptb_ww_no_window.restype = C.c_double
        _LIB.append(L)
    return _LIB[0]


def generate(mean, m2, volume, nb, max_rel_err, ratio):
    """The host build's windows of mean, m2 [ngroups, E]: (lower, upper, phimax)"""
    mean, m2 = (np.ascontiguousarray(a, dtype=np.float64) for a in (mean, m2))
    volume = np.ascontiguousarray(volume, dtype=np.float64)
    G, E = mean.shape
    lo, hi, pm = np.empty((G, E)), np.empty((G, E)), np.empty(G)
    ww_lib().ptb_ww_generate(mean.ctypes.data, m2.ctypes.data, volume.ctypes.data, E, G, nb, max_rel_err, ratio,
                             lo.ctypes.data, hi.ctypes.data, pm.ctypes.data)
    return lo, hi, pm


def readout(mean, m2, volume, nb):
    """phi and r as batch_readout kinds 0 and 2 form them"""
    with np.errstate(divide="ignore", invalid="ignore"):
        phi = mean / volume
        s = np.sqrt(m2 / (nb * (nb - 1.0))) / volume
        r = np.where(phi != 0.0, s / np.abs(phi), 0.0)
    return phi, r


def numpy_windows(mean, m2, volume, nb, max_rel_err, ratio):
    phi, r = readout(mean, m2, volume, nb)
    ok = (phi > 0) & np.isfinite(phi) & (r <= max_rel_err)
    pm = np.where(ok, phi, 0.0).max(axis=1)
    c = 2.0 / (ratio + 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        lo = (phi / pm[:, None]) * c
    hi = lo * ratio
    return np.where(ok, lo, -1.0), np.where(ok, hi, -1.0), pm


def assert_bits(got, want, label=""):
    np.testing.assert_array_equal(np.asarray(got).view(np.uint64), np.asarray(want).view(np.uint64), err_msg=label)


def check(mean, m2, volume, nb, max_rel_err, ratio, label=""):
    got = generate(mean, m2, volume, nb, max_rel_err, ratio)
    want = numpy_windows(mean, m2, volume, nb, max_rel_err, ratio)
    for g, w, what in zip(got, want, ("lower", "upper", "phimax")):
        assert_bits(g, w, f"{label} {what}")
    return got


def random_stats(rng, G, E, nb):
    mean = rng.lognormal(0.0, 3.0, (G, E)) * (rng.random((G, E)) < 0.9)
    m2 = mean ** 2 * rng.uniform(0.0, 2.0, (G, E)) * nb
    return mean, m2, rng.uniform(0.1, 3.0, E)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("ratio", [5.0, 1.0 + 2.0 ** -52, 1.5, 1e12])
def test_random_statistics_bit_for_bit(seed, ratio):
    rng = np.random.default_rng(seed)
    nb = float(rng.integers(2, 50))
    mean, m2, vol = random_stats(rng, 3, 1001, nb)
    for mre in (INF, 0.5, 0.05):
        lo, hi, pm = check(mean, m2, vol, nb, mre, ratio, f"seed {seed} mre {mre}")
        ok = lo > 0
        assert (hi[ok] >= lo[ok]).all() and (lo[~ok] == -1).all() and (hi[~ok] == -1).all()


def test_the_element_with_the_most_flux_is_centred_on_one():
    rng = np.random.default_rng(7)
    mean, m2, vol = random_stats(rng, 2, 500, 10.0)
    for ratio in (2.0, 5.0, 10.0):
        lo, hi, pm = check(mean, m2, vol, 10.0, INF, ratio)
        phi, _ = readout(mean, m2, vol, 10.0)
        for g in range(2):
            top = np.argmax(np.where(phi[g] > 0, phi[g], 0.0))
            assert lo[g, top] == 2.0 / (ratio + 1.0)
            assert hi[g, top] == lo[g, top] * ratio


def test_phi_zero_negative_nan_and_infinite_get_no_window():
    mean = np.array([[0.0, -0.0, -3.0, NAN, INF, -INF, 2.0, 4.0]])
    m2 = np.full_like(mean, 0.01)
    vol = np.full(mean.shape[1], 2.0)
    lo, hi, pm = check(mean, m2, vol, 5.0, INF, 5.0)
    assert (lo[0, :6] == -1).all() and (hi[0, :6] == -1).all()
    assert pm[0] == 2.0 and lo[0, 7] == 2.0 / 6.0 and lo[0, 6] == 0.5 * (2.0 / 6.0)
    # an infinite or NaN error never passes a finite limit; +inf passes every finite error
    m2[0, 6] = INF
    lo, _, _ = check(mean, m2, vol, 5.0, 1e300, 5.0)
    assert lo[0, 6] == -1 and lo[0, 7] > 0
    lo, _, _ = check(mean, m2, vol, 5.0, INF, 5.0)
    assert lo[0, 6] > 0  # (r = inf <= inf)
    m2[0, 6] = NAN
    lo, _, _ = check(mean, m2, vol, 5.0, INF, 5.0)
    assert lo[0, 6] == -1


def test_relative_error_just_below_at_and_above_the_limit():
    mean = np.array([[3.0, 1.0, 2.0]])
    m2 = np.array([[0.7, 0.3, 0.1]])
    vol = np.array([1.3, 0.7, 1.1])
    nb = 7.0
    _, r = readout(mean, m2, vol, nb)
    x = r[0, 1]
    for mre, eligible in ((np.nextafter(x, 0.0), False), (x, True), (np.nextafter(x, INF), True)):
        lo, _, _ = check(mean, m2, vol, nb, mre, 5.0, f"limit {mre!r}")
        assert (lo[0, 1] > 0) == eligible
    # with element 0 over the limit too, phimax comes from the remaining eligible elements
    lo, _, pm = check(mean, m2, vol, nb, min(r[0, 1], r[0, 2]) * 1.0000001, 5.0)
    phi, _ = readout(mean, m2, vol, nb)
    assert pm[0] == max(phi[0, k] for k in range(3) if r[0, k] <= min(r[0, 1], r[0, 2]) * 1.0000001)


def test_group_without_an_eligible_element():
    rng = np.random.default_rng(3)
    mean, m2, vol = random_stats(rng, 3, 200, 4.0)
    mean[1] = 0.0                      # no flux at all
    mean[2] = -np.abs(mean[2])         # negative only
    lo, hi, pm = check(mean, m2, vol, 4.0, INF, 5.0)
    assert pm[1] == 0.0 and pm[2] == 0.0 and pm[0] > 0
    assert (lo[1:] == -1).all() and (hi[1:] == -1).all()
    assert (lo[0][mean[0] > 0] > 0).all()


def test_ratio_near_one_and_large():
    rng = np.random.default_rng(11)
    mean, m2, vol = random_stats(rng, 1, 300, 3.0)
    for ratio in (np.nextafter(1.0, 2.0), 1.0 + 1e-9, 1e15, 1e300):
        lo, hi, _ = check(mean, m2, vol, 3.0, INF, ratio, f"ratio {ratio!r}")
        ok = lo > 0
        assert (hi[ok] >= lo[ok]).all()


def test_entries_of_set():
    E = ww_lib().ptb_ww_entry
    assert ww_lib().ptb_ww_no_window() == -1.0
    for lo, hi in ((0.0, 5.0), (-0.0, NAN), (-1.0, -2.0), (-INF, INF), (-2.0, NAN)):
        assert E(lo, hi) == 0, (lo, hi)            # lower <= 0: no window, upper unread
    for lo, hi in ((0.5, 2.0), (1e-300, 2e-300), (1.0, np.nextafter(1.0, 2.0)), (1.0, 1.7976931348623157e308)):
        assert E(lo, hi) == 1, (lo, hi)
    for lo, hi in ((NAN, 1.0), (1.0, NAN), (INF, INF), (1.0, INF), (2.0, 2.0), (2.0, 1.0), (1.0, -INF)):
        assert E(lo, hi) == -1, (lo, hi)


def test_groups_and_elements_out_of_range():
    S = ww_lib().ptb_ww_slot
    assert S(0, 3, 0, 10) == 0 and S(2, 3, 9, 10) == 29 and S(1, 3, 4, 10) == 14
    for g, e in ((-1, 0), (3, 0), (2 ** 31 - 1, 0), (-2 ** 31, 5), (0, -1), (1, -5)):
        assert S(g, 3, e, 10) == -1, (g, e)
    assert S(0, 0, 0, 10) == -1  # no windows: every group is out of range
    assert S(5, 6, 2 ** 31 - 1, 2 ** 31) == 5 * 2 ** 31 + 2 ** 31 - 1  # 64-bit index


def test_kernels_do_not_spill(tmp_path):
    cmd = [pbuild._nvcc(), *pbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(pbuild.CSRC, "ww_kernels.cu"),
           "-o", str(tmp_path / "ww_kernels.o")]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True)
    text = log.stdout + log.stderr
    found = {}
    for block in re.split(r"Compiling entry function '", text)[1:]:
        name = re.search(r"\d(ww_[a-z_]+_kernel)E", block.split("'", 1)[0]).group(1)
        s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        found[name] = tuple(int(x) for x in s.groups())
    assert sorted(found) == ["ww_generate_kernel", "ww_group_max_kernel", "ww_particles_kernel", "ww_points_kernel"]
    for name, (stack, stores, loads) in found.items():
        assert stack == 0 and stores == 0 and loads == 0, (name, stack, stores, loads)
