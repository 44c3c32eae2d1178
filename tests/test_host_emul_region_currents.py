"""The region-current pair plan (batch_stats.cuh: build_region_current_plan, face_area) compiled for the host by g++
as a TEST-ONLY build (tests/host_emul/emul_region_currents.cpp), against an independent numpy construction from the
face adjacency and the region map (region_currents_ref.py).  The same file compiles stats_kernels.cu with -Xptxas -v:
region_net_kernel must not spill or use a stack frame."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import HERE, ROOT, l_shaped_mesh
from pumiumtally_b200 import build as pbuild
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.partition import face_adjacency
from region_currents_ref import OUTSIDE, face_areas, pair_plan, plan_sum, reverse

_LIB = []


def rc_lib():
    if not _LIB:
        so = os.path.join(HERE, "host_emul", "libptb_region_currents.so")
        csrc = os.path.join(ROOT, "pumiumtally_b200", "csrc")
        src = os.path.join(HERE, "host_emul", "emul_region_currents.cpp")
        deps = [src] + [os.path.join(csrc, h) for h in ("batch_stats.cuh", "walk_core.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off",
                                   "-I", csrc, src, "-o", so])
        L = C.CDLL(so)
        L.ptb_rc_build.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.ptb_rc_build.restype = C.c_int64
        L.ptb_rc_nslots.restype = C.c_int64
        L.ptb_rc_levels.restype = C.c_int32
        L.ptb_rc_get.argtypes = [C.c_void_p] * 6
        L.ptb_rc_get.restype = None
        L.ptb_face_areas.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.ptb_face_areas.restype = None
        _LIB.append(L)
    return _LIB[0]


def host_plan(region, adj, slot_area):
    region = np.ascontiguousarray(region, dtype=np.int32)
    adj = np.ascontiguousarray(adj, dtype=np.int32)
    slot_area = np.ascontiguousarray(slot_area, dtype=np.float64)
    L = rc_lib()
    P = L.ptb_rc_build(region.ctypes.data, adj.ctypes.data, len(region), slot_area.ctypes.data)
    frm, to, rev = (np.empty(P, dtype=np.int32) for _ in range(3))
    area, first = np.empty(P), np.empty(P + 1, dtype=np.int64)
    slots = np.empty(L.ptb_rc_nslots(), dtype=np.int32)
    L.ptb_rc_get(*(a.ctypes.data for a in (frm, to, rev, area, first, slots)))
    return frm, to, rev, area, first, slots


def host_face_areas(coords, t2v):
    coords = np.ascontiguousarray(coords, dtype=np.float64)
    t2v = np.ascontiguousarray(t2v, dtype=np.int32)
    out = np.empty((len(t2v), 4))
    rc_lib().ptb_face_areas(coords.ctypes.data, t2v.ctypes.data, len(t2v), out.ctypes.data)
    return out


def meshes():
    yield "kuhn3", kuhn_box(3, 3, 3)
    yield "kuhn_6_5_4", kuhn_box(6, 5, 4, 1.5, 2.0, 0.7)
    yield "lshape", l_shaped_mesh(6, 6, 3)


def maps(E, seed):
    rng = np.random.default_rng(seed)
    yield "random", rng.integers(-1, 5, E).astype(np.int32)
    yield "random_sparse", np.where(rng.random(E) < 0.3, -1, rng.integers(0, 40, E)).astype(np.int32)
    yield "one", np.zeros(E, dtype=np.int32)
    yield "per_element", rng.permutation(E).astype(np.int32)


CASES = [(m, r) for m in ("kuhn3", "kuhn_6_5_4", "lshape") for r in ("random", "random_sparse", "one", "per_element")]


@pytest.mark.parametrize("mesh_name,map_name", CASES)
def test_pair_plan_matches_numpy(mesh_name, map_name):
    coords, t2v = dict(meshes())[mesh_name]
    E = len(t2v)
    region = dict(maps(E, 11))[map_name]
    adj = face_adjacency(t2v, len(coords)).astype(np.int32)
    area4 = face_areas(coords, t2v)
    got = host_plan(region, adj, area4.ravel())
    frm, to, rev, area, first, slots = got
    wf, wt, wfirst, wslots = pair_plan(adj, region)
    # the pair list, and every pair's slots, ascending
    np.testing.assert_array_equal(frm, wf)
    np.testing.assert_array_equal(to, wt)
    np.testing.assert_array_equal(first, wfirst)
    np.testing.assert_array_equal(slots, wslots)
    assert (np.lexsort((to, frm)) == np.arange(len(frm))).all()
    np.testing.assert_array_equal(rev, reverse(frm, to))
    # every slot in at most one pair
    assert len(np.unique(slots)) == len(slots)
    # the slots in no pair are exactly the interior faces inside one region
    e = np.repeat(np.arange(E), 4)
    nb = adj.ravel()
    interior_same = (nb >= 0) & (region[e] == region[np.maximum(nb, 0)])
    unused = np.ones(4 * E, dtype=bool)
    unused[slots] = False
    # an interior slot 4 n + b is "the face" of both sides; the unused slots are those of faces with A == B
    np.testing.assert_array_equal(unused, interior_same)
    # every hull slot lies in a pair into OUTSIDE, and those pairs hold nothing else
    pair_of = np.full(4 * E, -1)
    for p in range(len(frm)):
        pair_of[slots[first[p]:first[p + 1]]] = p
    hull = nb < 0
    assert (to[pair_of[hull]] == OUTSIDE).all()
    assert hull[slots[np.isin(pair_of[slots], np.flatnonzero(to == OUTSIDE))]].all()
    assert (rev[to == OUTSIDE] == -1).all()
    # the from region of a pair is the region of the element the weight leaves, the to region where it enters
    for p in range(len(frm)):
        s = slots[first[p]:first[p + 1]]
        if to[p] == OUTSIDE:
            assert (region[s // 4] == frm[p]).all()
        else:
            assert (region[s // 4] == to[p]).all()
            assert (region[adj.ravel()[s]] == frm[p]).all()
    # areas: the plan-order sum bit for bit, and math.fsum to 1e-14
    flat = area4.ravel()
    for p in range(len(frm)):
        x = flat[slots[first[p]:first[p + 1]]]
        assert area[p] == plan_sum(x), (p, area[p], plan_sum(x))
        want = math.fsum(x)
        assert abs(area[p] - want) <= 1e-14 * want, (p, area[p], want)
    if map_name == "one":
        assert list(zip(frm, to)) == [(0, OUTSIDE)]
    if map_name == "per_element":  # every face is in a pair: P is about 4E / 2 + hull faces
        assert len(slots) == 4 * E


@pytest.mark.parametrize("mesh_name", ["kuhn3", "kuhn_6_5_4", "lshape"])
def test_face_area_matches_numpy_bit_for_bit(mesh_name):
    coords, t2v = dict(meshes())[mesh_name]
    got = host_face_areas(coords, t2v)
    want = face_areas(coords, t2v)
    np.testing.assert_array_equal(got.view(np.uint64), want.view(np.uint64))
    # the two sides of an interior face give its area to within rounding, and the areas of the hull of a box add up
    # to its surface
    if mesh_name == "kuhn_6_5_4":
        adj = face_adjacency(t2v, len(coords))
        hull = adj < 0
        assert math.isclose(math.fsum(got[hull]), 2 * (1.5 * 2.0 + 1.5 * 0.7 + 2.0 * 0.7), rel_tol=1e-13)


def test_net_kernel_does_not_spill(tmp_path):
    cmd = [pbuild._nvcc(), *pbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(pbuild.CSRC, "stats_kernels.cu"),
           "-o", str(tmp_path / "stats_kernels.o")]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True)
    text = log.stdout + log.stderr
    found = {}
    for block in re.split(r"Compiling entry function '", text)[1:]:
        m = re.search(r"\d(region_net_kernel)E", block.split("'", 1)[0])
        if m:
            s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
            found[m.group(1)] = tuple(int(x) for x in s.groups())
    assert found == {"region_net_kernel": (0, 0, 0)}, found
