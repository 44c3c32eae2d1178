"""Checkpoint format version 3 (point detectors), through a TEST-ONLY host build of checkpoint.cpp
(tests/host_emul/emul_checkpoint_detectors.cpp): the version is 3 exactly when the fingerprint holds detectors, the
detector sections round-trip, and a file of other detector positions, radii or cross-section table is refused with a
message that names them."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT

_LIB = []


def lib():
    if not _LIB:
        so = os.path.join(HERE, "host_emul", "libptb_ckpt_det.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        srcs = [os.path.join(HERE, "host_emul", "emul_checkpoint_detectors.cpp"), os.path.join(csrc, "checkpoint.cpp")]
        deps = srcs + [os.path.join(csrc, "checkpoint.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-I", csrc, *srcs, "-o", so,
                                   "-lz"])
        L = C.CDLL(so)
        L.ptb_ckpt_det_write.restype = C.c_int64
        L.ptb_ckpt_det_write.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int64, C.c_int32,
                                         C.c_void_p, C.c_int64]
        L.ptb_ckpt_det_read.restype = C.c_int32
        L.ptb_ckpt_det_read.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int64]
        _LIB.append(L)
    return _LIB[0]


XYZ = np.array([[1.0, 2.0, 3.0], [0.5, 0.25, 0.125]])
R0 = np.array([0.0, 0.3])


def write(xyz=XYZ, r0=R0, crc=1234, det_len=6, nmu=0):
    out = np.zeros(1 << 16, dtype=np.uint8)
    n = lib().ptb_ckpt_det_write(len(r0), np.ascontiguousarray(xyz).ctypes.data, np.ascontiguousarray(r0).ctypes.data,
                                 crc, det_len, nmu, out.ctypes.data, out.size)
    assert n > 0
    return out[:n].copy()


def read(data, xyz=XYZ, r0=R0, crc=1234, nmu=0):
    det_len = C.c_int64(-1)
    ids = np.zeros(16, dtype=np.uint32)
    nids = C.c_int32(0)
    err = C.create_string_buffer(256)
    rc = lib().ptb_ckpt_det_read(data.ctypes.data, data.size, len(r0), np.ascontiguousarray(xyz).ctypes.data,
                                 np.ascontiguousarray(r0).ctypes.data, crc, nmu, C.byref(det_len), ids.ctypes.data,
                                 C.byref(nids), err, 256)
    return rc, err.value.decode(), det_len.value, list(ids[:nids.value])


def version(data):
    return int(np.frombuffer(data[8:12].tobytes(), dtype="<u4")[0])


@pytest.mark.parametrize("nmu", [0, 4])
def test_version_3_only_with_detectors_and_the_round_trip(nmu):
    with_det = write(nmu=nmu)
    without = write(xyz=np.zeros((0, 3)), r0=np.zeros(0), crc=0, nmu=nmu)
    assert version(with_det) == 3
    assert version(without) == (2 if nmu else 1)
    rc, err, det_len, ids = read(with_det, nmu=nmu)
    assert rc == 0, err
    assert det_len == 6 and ids == [1, 2, 3, 4, 7, 8, 9, 10]
    rc, err, det_len, ids = read(without, xyz=np.zeros((0, 3)), r0=np.zeros(0), crc=0, nmu=nmu)
    assert rc == 0 and det_len == 0 and ids == [1, 2, 3, 4]


def test_other_detectors_or_table_are_named():
    data = write()
    assert "cross-section table" in read(data, crc=1235)[1]
    r0 = R0.copy()
    r0[1] = np.nextafter(r0[1], 1.0)
    assert "exclusion radii" in read(data, r0=r0)[1]
    xyz = XYZ.copy()
    xyz[1, 2] = -xyz[1, 2]
    assert "positions" in read(data, xyz=xyz)[1]
    assert "number of point detectors" in read(data, xyz=XYZ[:1], r0=R0[:1])[1]
    assert "number of point detectors" in read(data, xyz=np.zeros((0, 3)), r0=np.zeros(0))[1]


def test_a_flipped_byte_in_the_detector_fingerprint_is_refused():
    data = write()
    for at in range(140, len(data) - 16 * 4, 37):
        bad = data.copy()
        bad[at] ^= 0x10
        assert read(bad)[0] != 0, at
