"""The checkpoint format (checkpoint.cpp) and the merge update (batch_stats.cuh, welford_merge) compiled for the host by
g++ as a TEST-ONLY build (tests/host_emul/emul_checkpoint.cpp).  merge_checkpoint's kernel runs the same welford_merge,
and the engine writes and reads files through the same chunked callbacks, fed from pinned buffers instead of memory."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT

_LIB = []
_dp = C.POINTER(C.c_double)


def lib():
    if not _LIB:
        so = os.path.join(HERE, "host_emul", "libptb_checkpoint.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        src = os.path.join(HERE, "host_emul", "emul_checkpoint.cpp")
        deps = [src] + [os.path.join(csrc, h) for h in ("batch_stats.cuh", "walk_core.cuh", "checkpoint.hpp",
                                                         "checkpoint.cpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off",
                                   "-I", csrc, src, os.path.join(csrc, "checkpoint.cpp"), "-lz", "-o", so])
        L = C.CDLL(so)
        L.ptb_welford_merge.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p,
                                        C.c_int64]
        L.ptb_welford_fold_all.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_void_p]
        L.ptb_hash64.argtypes = [C.c_void_p, C.c_int64, C.c_uint64]
        L.ptb_hash64.restype = C.c_uint64
        L.ptb_ckpt_write.argtypes = [C.c_void_p] * 7 + [C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int64,
                                                        C.c_void_p, C.c_int64]
        L.ptb_ckpt_write.restype = C.c_int64
        L.ptb_ckpt_read.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int64,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_char_p, C.c_int64]
        L.ptb_ckpt_read.restype = C.c_int32
        _LIB.append(L)
    return _LIB[0]


# ---------------------------------------------------------------- welford_merge

def fold(x, nb0=0, mean=None, m2=None):
    """x [B, n] folded in order by welford_fold"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    mean = np.zeros(x.shape[1]) if mean is None else mean.copy()
    m2 = np.zeros(x.shape[1]) if m2 is None else m2.copy()
    lib().ptb_welford_fold_all(x.ctypes.data, x.shape[0], x.shape[1], float(nb0), mean.ctypes.data, m2.ctypes.data)
    return mean, m2


def merge(a, b, na, nb):
    mean, m2 = a[0].copy(), a[1].copy()
    mb, qb = np.ascontiguousarray(b[0]), np.ascontiguousarray(b[1])
    lib().ptb_welford_merge(mb.ctypes.data, qb.ctypes.data, float(na), float(nb), mean.ctypes.data, m2.ctypes.data,
                            len(mean))
    return mean, m2


def two_pass(x):
    m = x.mean(axis=0)
    return m, ((x - m) ** 2).sum(axis=0)


@pytest.mark.parametrize("seed", range(6))
def test_merge_matches_two_pass_statistics_of_the_union(seed):
    rng = np.random.default_rng(seed)
    B, n = int(rng.integers(2, 40)), 257
    x = rng.normal(rng.uniform(-5, 5, n), rng.uniform(0.01, 3, n), (B, n))
    for split in sorted(set(rng.integers(1, B, 4).tolist())):
        got = merge(fold(x[:split]), fold(x[split:]), split, B - split)
        want = two_pass(x)
        np.testing.assert_allclose(got[0], want[0], rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(got[1], want[1], rtol=1e-11, atol=1e-11 * want[1].max())


def test_merge_with_an_empty_side_is_exact():
    rng = np.random.default_rng(7)
    a = (rng.normal(size=1000), rng.uniform(0, 5, 1000))
    b = (rng.normal(size=1000), rng.uniform(0, 5, 1000))
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 5e-324, 1.7e308, -1e-300])
    a = tuple(np.concatenate([v, specials]) for v in a)
    b = tuple(np.concatenate([v, specials[::-1]]) for v in b)
    bits = lambda v: v.view(np.uint64)  # noqa: E731
    for na in (0, 0.0):
        got = merge(a, b, na, 13)  # na == 0: b's bits, whatever a holds
        np.testing.assert_array_equal(bits(got[0]), bits(b[0]))
        np.testing.assert_array_equal(bits(got[1]), bits(b[1]))
    got = merge(a, b, 13, 0)  # nb == 0: a unchanged
    np.testing.assert_array_equal(bits(got[0]), bits(a[0]))
    np.testing.assert_array_equal(bits(got[1]), bits(a[1]))


def test_many_small_runs_against_one_sequential_fold():
    rng = np.random.default_rng(11)
    n = 513
    runs = [rng.normal(3.0, 0.5, (int(k), n)) for k in rng.integers(1, 6, 40)]
    acc, na = (np.zeros(n), np.zeros(n)), 0
    for r in runs:
        acc = merge(acc, fold(r), na, len(r))
        na += len(r)
    want = fold(np.concatenate(runs))
    np.testing.assert_allclose(acc[0], want[0], rtol=1e-14)
    np.testing.assert_allclose(acc[1], want[1], rtol=1e-10)


def test_ill_conditioned_merge():
    """The fold tests' 1e8 (1 + 1e-9 u) set: a relative spread of 1e-9 around 1e8, split and merged."""
    rng = np.random.default_rng(13)
    B, n = 64, 301
    x = 1e8 * (1.0 + 1e-9 * rng.uniform(-1, 1, (B, n)))
    want_s = x.astype(np.longdouble).std(axis=0, ddof=1).astype(np.float64)
    for split in (1, 17, 32, 63):
        m, q = merge(fold(x[:split]), fold(x[split:]), split, B - split)
        np.testing.assert_allclose(m, x.mean(axis=0), rtol=1e-15)
        np.testing.assert_allclose(np.sqrt(q / (B - 1)), want_s, rtol=1e-6)


# ---------------------------------------------------------------- the file format

EDGES = np.array([0.0, 0.5, 1.25, 4.0])
E, S = 11, 3


class Ckpt:
    """One checkpoint's arrays and its file (written through 4 KiB chunks)."""

    def __init__(self, open_batch=True, stats=True, regions=True, seed=1, chunk=4096):
        rng = np.random.default_rng(seed)
        self.hdr = np.array([5 if stats else 0, int(open_batch), 1237 if open_batch else 0, 1003 if stats else 0,
                             18 if (stats and regions) else 0], dtype=np.int64)
        self.open = rng.normal(size=max(self.hdr[2], 1))
        self.scalars = rng.integers(0, 2 ** 40, 13, dtype=np.uint64)
        self.scalars[1] = 1
        self.scalars[0] = np.float64(3.25).view(np.uint64)
        self.scalars[12] = 0
        self.mean, self.m2 = (rng.normal(size=max(self.hdr[3], 1)) for _ in range(2))
        self.rmean, self.rm2 = (rng.normal(size=max(self.hdr[4], 1)) for _ in range(2))
        self.chunk = chunk
        self.data = self.write()

    def write(self):
        cap = 1 << 20
        out = np.zeros(cap, dtype=np.uint8)
        n = lib().ptb_ckpt_write(self.hdr.ctypes.data, self.open.ctypes.data, self.scalars.ctypes.data,
                                 self.mean.ctypes.data, self.m2.ctypes.data, self.rmean.ctypes.data,
                                 self.rm2.ctypes.data, E, S, EDGES.ctypes.data, len(EDGES), self.chunk,
                                 out.ctypes.data, cap)
        assert n > 0
        return out[:n].tobytes()

    def sections(self):
        """(start, end) of every section, header included, after the fixed part"""
        pos = 16 + 40 + 100 + 8 * len(EDGES) + 4
        out = []
        for nbytes in self.section_bytes():
            out.append((pos, pos + 16 + nbytes))
            pos += 16 + nbytes
        assert pos == len(self.data)
        return out

    def section_bytes(self):
        h = self.hdr
        s = []
        if h[1]:
            s += [8 * h[2], 8 * 13]
        if h[3]:
            s += [8 * h[3]] * 2
        if h[4]:
            s += [8 * h[4]] * 2
        return [int(v) for v in s]


def read(data, chunk=4096, nscores=S, edges=EDGES):
    buf = np.frombuffer(bytes(data), dtype=np.uint8).copy()
    hdr = np.zeros(5, dtype=np.int64)
    arrays = [np.zeros(4096) for _ in range(5)]
    scalars = np.zeros(13, dtype=np.uint64)
    maxreq = C.c_int64(0)
    err = C.create_string_buffer(512)
    rc = lib().ptb_ckpt_read(buf.ctypes.data, len(buf), E, nscores, edges.ctypes.data, len(edges), chunk,
                             hdr.ctypes.data, arrays[0].ctypes.data, scalars.ctypes.data, arrays[1].ctypes.data,
                             arrays[2].ctypes.data, arrays[3].ctypes.data, arrays[4].ctypes.data, C.byref(maxreq),
                             err, 512)
    return rc, hdr, arrays, scalars, maxreq.value, err.value.decode()


@pytest.mark.parametrize("open_batch,stats,regions", [(True, True, True), (False, True, True), (True, False, False),
                                                      (False, True, False)])
@pytest.mark.parametrize("chunk", [8, 4096, 1 << 16])
def test_round_trip_is_byte_exact(open_batch, stats, regions, chunk):
    c = Ckpt(open_batch, stats, regions, chunk=chunk)
    rc, hdr, a, sc, _, err = read(c.data, chunk=chunk)
    assert rc == 0, err
    np.testing.assert_array_equal(hdr, c.hdr)
    for got, want, n in ((a[0], c.open, c.hdr[2]), (a[1], c.mean, c.hdr[3]), (a[2], c.m2, c.hdr[3]),
                         (a[3], c.rmean, c.hdr[4]), (a[4], c.rm2, c.hdr[4])):
        np.testing.assert_array_equal(got[:n].view(np.uint64), want[:n].view(np.uint64))
    if open_batch:
        np.testing.assert_array_equal(sc[:12], c.scalars[:12])
    # written again from what was read: the same bytes (no timestamps, no chunk-size dependence)
    c2 = Ckpt(open_batch, stats, regions, chunk=4096)
    assert c2.data == c.data
    assert len(c.sections()) == len(c.section_bytes())


def test_fingerprint_mismatch_is_named():
    c = Ckpt()
    rc, *_, err = read(c.data, nscores=S + 1)
    assert rc == 2 and "scores" in err
    e2 = EDGES.copy()
    e2[2] = np.nextafter(e2[2], 9.0)  # one ulp
    rc, *_, err = read(c.data, edges=e2)
    assert rc == 2 and "time-bin edges" in err


def test_a_flipped_byte_anywhere_is_refused():
    c = Ckpt()
    d = bytearray(c.data)
    secs = c.sections()
    fixed_end = secs[0][0]
    # every byte of the prefix, header and fingerprint, and a spread of bytes in every section (its head and payload)
    positions = list(range(fixed_end))
    for lo, hi in secs:
        positions += list(range(lo, lo + 16)) + sorted({lo + 16, (lo + hi) // 2, hi - 1})
    for p in positions:
        bad = bytearray(d)
        bad[p] ^= 0x10
        rc, *_, err = read(bad)
        assert rc != 0, f"byte {p} flipped was accepted"
        assert (rc == 2) == (p < fixed_end), (p, rc, err)


def test_truncation_is_refused_before_any_section():
    c = Ckpt()
    secs = c.sections()
    cuts = {0, 1, 8, 15, 16, 100, secs[0][0] - 1, secs[0][0]}
    for lo, hi in secs:
        cuts |= {lo, lo + 1, lo + 16, (lo + hi) // 2, hi - 1, hi}
    cuts.discard(len(c.data))
    for n in sorted(cuts):
        rc, *_, maxreq, err = read(c.data[:n])
        assert rc == 2, (n, rc, err)  # the declared lengths no longer add up to the file size
    # extra bytes at the end are refused the same way
    rc, *_, err = read(c.data + b"\0")
    assert rc == 2 and "file size" in err


def test_wrong_magic_version_and_endianness():
    c = Ckpt()
    d = bytearray(c.data)
    bad = bytearray(d)
    bad[0:8] = b"PTBCKPX\0"
    rc, *_, err = read(bad)
    assert rc == 2 and "magic" in err
    bad = bytearray(d)
    bad[8:12] = struct.pack("<I", 2)
    rc, *_, err = read(bad)
    assert rc == 2 and "version" in err
    bad = bytearray(d)
    bad[12:16] = struct.pack(">I", 0x01020304)
    rc, *_, err = read(bad)
    assert rc == 2 and "endianness" in err


def test_a_declared_length_larger_than_the_file_is_refused_before_reading_it():
    """stats_len patched to 2^40 doubles, with the header CRC recomputed: the reader refuses from the header alone and
    never asks for more than the fixed part."""
    import zlib

    c = Ckpt()
    d = bytearray(c.data)
    fixed = c.sections()[0][0]
    d[16 + 24:16 + 32] = struct.pack("<Q", 1 << 40)
    d[fixed - 4:fixed] = struct.pack("<I", zlib.crc32(bytes(d[:fixed - 4])))
    rc, *_, maxreq, err = read(d)
    assert rc == 2 and "file size" in err, err
    assert maxreq < 4096


def test_hash64_is_deterministic_and_sensitive():
    a = np.arange(1001, dtype=np.int32)
    h = lib().ptb_hash64(a.ctypes.data, a.nbytes, 0)
    assert h == lib().ptb_hash64(a.ctypes.data, a.nbytes, 0)
    hs = {h}
    for i in (0, 500, 1000):
        b = a.copy()
        b[i] ^= 1
        hs.add(lib().ptb_hash64(b.ctypes.data, b.nbytes, 0))
    hs.add(lib().ptb_hash64(a.ctypes.data, a.nbytes - 1, 0))
    hs.add(lib().ptb_hash64(a.ctypes.data, a.nbytes, 1))
    assert len(hs) == 6
