"""The per-move counting sort (bin_kernels.cu: bin_count_kernel, the three-kernel scan scan_block_kernel,
scan_sums_kernel and scan_add_kernel, then bin_scatter_kernel or bin_pack_kernel) and the initial-weight sum
(walk_kernels.cu: sum_flying_weights_kernel), called directly through a test-only C wrapper of their launchers
(tests/gpu_harness/bin_harness.cpp).  The grids run from 1 cell to the two largest choose_seed_grid builds (257^3 and
1024 x 1024 x 17 cells), through every block and tile boundary of the scan; the keys include cell boundaries, points
outside the box, non-finite coordinates and midpoints.  Every output must equal a host reference exactly, and every
device buffer carries canaries that must come back untouched.

cuobjdump -sass of bin_kernels.cu (nvcc -O3, sm_90a, default flags), bin_count_kernel:
  0.5 * (x + mx)          DADD, then DMUL by 0.5
  f = (x - x0) * inv_h    DADD, then DMUL: not fused with the midpoint's product or with each other
  (int)f                  F2I.F64.TRUNC (saturating), taken only where f > 0 (DSETP.GT)
  all_finite(mx, my, mz)  DMUL 0 * my, then DFMA 0 * mx + _, DFMA 0 * mz + _: the kernel's only DFMAs.  Each product
                          is +-0 or NaN, so fused or not the sum is +-0 exactly when all three are finite.
So numpy's float64 arithmetic, which never contracts, gives every key exactly.  test_kernel_sass_bin.py checks the
SASS for this."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

from test_gpu_stats_kernels import Guarded, _sms, _stream, assert_bits, build_harness

gpu = pytest.mark.gpu
SCAN_BLOCK = 1024  # kScanBlock: counts per scan block
TILE = SCAN_BLOCK * 1024  # cells whose block sums scan_sums_kernel scans in one pass of its tile loop
ID_MASK = 0x3fffffff  # kIdMask


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    L = C.CDLL(build_harness(tmp_path_factory, "bin_harness"))
    p, i32, f64 = C.c_void_p, C.c_int32, C.c_double
    grid = [f64] * 5 + [i32] * 3
    L.ptb_test_bin_particles.argtypes = grid + [p, p, p, p, p, i32, i32, p, p, p, p, p, p]
    L.ptb_test_bin_pack_particles.argtypes = grid + [p, p, p, p, p, p, i32, i32, p, p, p, p, p, C.c_int, p]
    L.ptb_test_sum_flying_weights.argtypes = [p, p, i32, i32, p, p]
    return L


# ---------------------------------------------------------------------------------------------------------------------
# Reference
# ---------------------------------------------------------------------------------------------------------------------
class Grid:
    def __init__(self, dims, lo=(-2.3, -0.7, -1.1), h=0.25):
        self.dims = np.array(dims, dtype=np.int64)
        self.lo = np.array(lo, dtype=np.float64)
        self.h, self.inv_h = h, 1.0 / h  # as choose_seed_grid sets them
        self.ncell = int(np.prod(self.dims))

    def args(self):
        return (*map(float, self.lo), self.h, self.inv_h, *map(int, self.dims))


def cell_ref(g, xyz):
    """cell_of without ranks: f = (x - x0) * inv_h rounded twice; 0 unless f > 0, else int(min(f, n - 1)) (clamped
    before the conversion, which saturates on the device)"""
    with np.errstate(invalid="ignore", over="ignore"):
        f = (xyz - g.lo) * g.inv_h
        c = np.where(f > 0.0, np.minimum(f, g.dims - 1), 0.0).astype(np.int64)
    nx, ny, _ = g.dims
    return (c[:, 2] * ny + c[:, 1]) * nx + c[:, 0]


def key_position(start, mid):
    """the binning key's position: the start, or with a midpoint 0.5 * (x + mx) per axis where all three mid
    components are finite"""
    if mid is None:
        return start
    with np.errstate(invalid="ignore", over="ignore"):
        m = 0.5 * (start + mid)
    return np.where(np.isfinite(mid).all(axis=1)[:, None], m, start)


def morton_rank(dims):
    """morton_cell_ranks (seed_grid.hpp): the cells sorted by (bit interleave of (cx, cy, cz), cell)"""
    nx, ny, nz = map(int, dims)

    def spread(v):
        v = v.astype(np.uint64) & np.uint64(0x1fffff)
        for sh, m in ((32, 0x1f00000000ffff), (16, 0x1f0000ff0000ff), (8, 0x100f00f00f00f00f),
                      (4, 0x10c30c30c30c30c3), (2, 0x1249249249249249)):
            v = (v | (v << np.uint64(sh))) & np.uint64(m)
        return v

    c = np.arange(nx * ny * nz, dtype=np.int64)
    key = spread(c % nx) | (spread(c // nx % ny) << np.uint64(1)) | (spread(c // (nx * ny)) << np.uint64(2))
    rank = np.empty(len(c), dtype=np.int32)
    rank[np.argsort(key, kind="stable")] = np.arange(len(c), dtype=np.int32)
    return rank


class Particles:
    """Host arrays of N particle slots: state [N, 4] (x, y, z, then elem in the low and garbage in the high 32 bits
    of the fourth double), origin [N, 3] or None, dest [N, 3], weights [N], flying [N] int8 or None."""

    def __init__(self, state, origin, dest, weights, flying, begin, end):
        self.state, self.origin, self.dest, self.weights, self.flying = state, origin, dest, weights, flying
        self.begin, self.end, self.N = begin, end, len(state)

    def start(self):
        return self.state[:, :3] if self.origin is None else self.origin

    def flies(self):
        return np.ones(self.N, bool) if self.flying is None else self.flying == 1


def rows_ref(P, ids):
    """the PackedRow of every particle id, as int64[8]: origin (the stored position without an origin array), dest
    and weight as bit copies, then id | elem << 32 with elem = (state.elem & kIdMask) | moved << 31, moved the IEEE
    test origin != stored position on any axis"""
    s = P.state[ids]
    o = s[:, :3] if P.origin is None else P.origin[ids]
    moved = (o != s[:, :3]).any(axis=1).astype(np.uint64)
    elem = (s[:, 3].view(np.uint64) & np.uint64(ID_MASK)) | (moved << np.uint64(31))
    row = np.empty((len(ids), 8), dtype=np.int64)
    row[:, 0:3] = o.view(np.int64)
    row[:, 3:6] = P.dest[ids].view(np.int64)
    row[:, 6] = P.weights[ids].view(np.int64)
    row[:, 7] = (ids.astype(np.uint64) | (elem << np.uint64(32))).view(np.int64)
    return row


@functools.lru_cache(maxsize=2)
def _ranks(dims, kind):
    """(host rank or None, device Guarded or None, bin -> cell)"""
    n = int(np.prod(dims))
    if kind is None:
        return None, None, np.arange(n)
    rank = morton_rank(dims) if kind == "morton" else np.random.default_rng(n).permutation(n).astype(np.int32)
    inv = np.empty(n, dtype=np.int64)
    inv[rank] = np.arange(n)
    return rank, Guarded(rank, seed=11), inv


# ---------------------------------------------------------------------------------------------------------------------
# One binning call, checked in full
# ---------------------------------------------------------------------------------------------------------------------
def run_binning(L, g, rank_kind, P, mid, packed, label):
    """launch_bin_particles (mid: key by the midpoint towards dest) or launch_bin_pack_particles (mid: midpoint_key)
    on P's slots [begin, end), and check every output and every canary."""
    rank, grank, _ = _ranks(tuple(map(int, g.dims)), rank_kind)
    n, b0 = P.end - P.begin, P.begin
    keep = [Guarded(P.state.reshape(-1), seed=1), Guarded(P.dest.reshape(-1), seed=2), Guarded(P.weights, seed=3)]
    gs, gd, gw = keep
    go = Guarded(P.origin.reshape(-1), seed=4) if P.origin is not None else None
    gf = Guarded(P.flying, seed=5) if P.flying is not None else None
    keep += [x for x in (go, gf) if x is not None]
    pcell = Guarded(np.full(P.N, -7, dtype=np.int32), seed=6)
    count = Guarded(np.zeros(g.ncell, dtype=np.uint32), seed=7)
    sums = Guarded(np.zeros(g.ncell // SCAN_BLOCK + 2, dtype=np.uint32), seed=8)  # as build_seed_grid allocates it
    wc = Guarded(np.array([0xdeadbeef], dtype=np.uint32), seed=9)
    out = Guarded(np.zeros(max(n, 0) * (8 if packed else 1), dtype=np.int64 if packed else np.int32), seed=10)
    ptr = lambda x: x.ptr() if x is not None else None  # noqa: E731
    if packed:
        err = L.ptb_test_bin_pack_particles(*g.args(), ptr(grank), ptr(go), gd.ptr(), gw.ptr(), ptr(gf), gs.ptr(), b0,
                                            P.end, pcell.ptr(), count.ptr(), sums.ptr(), out.ptr(), wc.ptr(), int(mid),
                                            _stream())
    else:
        err = L.ptb_test_bin_particles(*g.args(), ptr(grank), ptr(go), gs.ptr(), gd.ptr() if mid else None, ptr(gf),
                                       b0, P.end, pcell.ptr(), count.ptr(), sums.ptr(), out.ptr(), wc.ptr(), _stream())
    assert err == 0, label
    for x in keep + ([grank] if grank is not None else []):
        x.assert_unchanged_outside(0, 0, label + " read-only input")
    if n <= 0:  # only the work count is written
        assert wc.values()[0] == 0, label
        for x in (pcell, count, sums, out):
            x.assert_unchanged_outside(0, 0, label)
        return 0
    sl = slice(b0, P.end)
    fly = P.flies()[sl]
    cell = cell_ref(g, key_position(P.start()[sl], P.dest[sl] if mid else None))
    key = cell if rank is None else rank[cell].astype(np.int64)
    hist = np.bincount(key[fly], minlength=g.ncell)
    nfly = int(fly.sum())
    assert wc.values()[0] == nfly, label + " work count"
    wc.assert_unchanged_outside(0, 1, label + " work count")
    assert np.array_equal(pcell.values(b0, P.end), np.where(fly, key, -1)), label + " pcell"
    pcell.assert_unchanged_outside(b0, P.end, label + " pcell")
    # the scatter leaves every cursor at the end of its cell's segment: the inclusive scan of the histogram
    incl = np.cumsum(hist)
    got = count.values().astype(np.int64)
    if not np.array_equal(got, incl):
        bad = np.flatnonzero(got != incl)
        raise AssertionError(f"{label} count: {len(bad)} of {g.ncell} differ, first at {bad[0]}: {got[bad[0]]} != "
                             f"{incl[bad[0]]}")
    count.assert_unchanged_outside(0, g.ncell, label + " count")
    nb = -(-g.ncell // SCAN_BLOCK)
    bsum = np.bincount(np.arange(g.ncell) // SCAN_BLOCK, weights=hist, minlength=nb).astype(np.int64)
    assert np.array_equal(sums.values(0, nb).astype(np.int64), np.cumsum(bsum) - bsum), label + " block sums"
    sums.assert_unchanged_outside(0, nb, label + " block sums")
    # segment b of the output is [incl[b] - hist[b], incl[b]): exactly the flying ids of key b, in any order
    seg = np.repeat(np.arange(g.ncell), hist)
    ids = b0 + np.flatnonzero(fly)
    if packed:
        rows = out.values(0, 8 * nfly).reshape(nfly, 8)
        got_ids = (rows[:, 7] & 0xffffffff).astype(np.int64)
    else:
        got_ids = out.values(0, nfly).astype(np.int64)
    assert np.array_equal(np.sort(got_ids), ids), label + " ids"
    assert np.array_equal(key[got_ids - b0], seg), label + " segments"
    if packed:
        want = rows_ref(P, got_ids)
        if not np.array_equal(rows, want):
            bad = np.flatnonzero((rows != want).any(axis=1))
            raise AssertionError(f"{label} rows: {len(bad)} of {nfly} differ, first id {got_ids[bad[0]]}: "
                                 f"{rows[bad[0]]} != {want[bad[0]]}")
    out.assert_unchanged_outside(0, nfly * (8 if packed else 1), label + " output past the work count")
    return nfly


# ---------------------------------------------------------------------------------------------------------------------
# Scan sizes and populations
# ---------------------------------------------------------------------------------------------------------------------
SCAN_GRIDS = {  # ncell: dims
    1: (1, 1, 1), 2: (1, 2, 1), 255: (5, 17, 3), 1023: (11, 31, 3), 1024: (16, 8, 8), 1025: (5, 41, 5),
    4099: (4099, 1, 1), 2**20 - 1: (75, 341, 41), 2**20: (128, 128, 64), 2**20 + 1: (17, 61681, 1),
    2**20 + 1025: (21, 151, 331), 5 * 2**20 + 3: (5 * 2**20 + 3, 1, 1),
    257**3: (257, 257, 257),  # choose_seed_grid's cube at the cell cap
    1024 * 1024 * 17: (1024, 1024, 17),  # choose_seed_grid's 1000 x 1000 x 15.63 slab
}
LARGEST = (257**3, 1024 * 1024 * 17)
# (population, n, begin, flying, origin array, midpoint)
POPULATIONS = [
    ("uniform", 100_003, 257, "mixed", True, True),
    ("uniform", 257, 1, None, False, False),
    ("first", 256, 0, "mixed", True, False),
    ("last", 255, 1, None, True, True),
    ("in last tile", 257, 257, "mixed", False, True),
    ("last tile", 100_003, 0, None, True, False),
    ("none flying", 257, 1, "none", True, True),
    ("single", 1, 257, None, True, False),
    ("single", 1, 0, "mixed", False, True),
]
BIG = ("uniform", 4_000_037, 1, "mixed", True, True)


def make_particles(rng, g, inv_rank, population, n, begin, flying, origin, mid):
    """n particles in slots [begin, begin + n) of an array with 3 more slots after them (slots outside the range hold
    positions in other cells and must not be binned).  Positions are drawn in the bins the population names (bin ->
    cell through inv_rank), away from cell faces; a fifth of the stored positions differ from the origin, one in
    fifty by the sign of a zero only; NaN payloads in dest and weights."""
    N = begin + n + 3
    last_tile = (g.ncell - 1) // TILE * TILE
    bins = {"first": np.zeros(N, np.int64), "last": np.full(N, g.ncell - 1),
            "in last tile": np.full(N, last_tile + (g.ncell - 1 - last_tile) // 2),
            "last tile": rng.integers(last_tile, g.ncell, N)}.get(population)
    if bins is None:
        bins = rng.integers(0, g.ncell, N)
    cell = inv_rank[bins]
    nx, ny, _ = g.dims
    c = np.stack([cell % nx, cell // nx % ny, cell // (nx * ny)], axis=1)
    pos = g.lo + (c + rng.uniform(0.05, 0.95, (N, 3))) * g.h
    state = np.empty((N, 4))
    state[:, :3] = pos
    other = rng.random(N) < 0.2
    state[other, :3] = g.lo + rng.uniform(0.0, 1.0, (int(other.sum()), 3)) * g.dims * g.h
    zero = rng.random(N) < 0.02
    pos[zero, 1], state[zero, 1] = 0.0, -0.0
    state[:, 3] = (rng.integers(-2**31, 2**31, N) & 0xffffffff | rng.integers(0, 2**32, N) << 32).view(np.float64)
    dest = pos.copy() if population in ("first", "last", "in last tile") else pos + rng.normal(0.0, g.h, (N, 3))
    dest[rng.random(N) < 0.01, rng.integers(0, 3)] = np.nan
    dest.reshape(-1)[rng.integers(0, 3 * N, max(N // 100, 1))] = np.array([0x7ff4000000000123], np.uint64).view(float)
    w = rng.lognormal(0.0, 1.0, N)
    w[rng.random(N) < 0.01] = np.array([0x7ff80000cafe0001], np.uint64).view(np.float64)[0]
    fl = None
    if flying == "mixed":
        fl = rng.choice(np.array([1, 1, 1, 0, 2, -1], dtype=np.int8), N)
        if n == 1:
            fl[begin] = 1
    elif flying == "none":
        fl = rng.choice(np.array([0, 2, -1], dtype=np.int8), N)
    if not origin:
        state[:, :3] = pos
    return Particles(state, pos if origin else None, dest, w, fl, begin, begin + n)


SCAN_CASES = [(ncell, rank) for ncell in SCAN_GRIDS for rank in (None, "perm", "morton")]


@gpu
@pytest.mark.parametrize("ncell, rank", SCAN_CASES, ids=[f"{n}-{r or 'cells'}" for n, r in SCAN_CASES])
def test_binning_is_exact(harness, ncell, rank):
    dims = SCAN_GRIDS[ncell]
    g = Grid(dims)
    _, _, inv = _ranks(dims, rank)
    rng = np.random.default_rng([ncell, (None, "perm", "morton").index(rank)])
    for k, (pop, n, begin, fl, origin, mid) in enumerate(POPULATIONS + ([BIG] if ncell in LARGEST else [])):
        P = make_particles(rng, g, inv, pop, n, begin, fl, origin, mid)
        for packed in (False, True):
            label = f"{dims} {rank} {pop} n {n} begin {begin} flying {fl} origin {origin} mid {mid} packed {packed}"
            nfly = run_binning(harness, g, rank, P, mid, packed, label)
            assert (nfly == 0) == (fl == "none"), label


@gpu
def test_empty_range_writes_only_the_work_count(harness):
    g = Grid((5, 17, 3))
    P = make_particles(np.random.default_rng(0), g, np.arange(g.ncell), "uniform", 0, 5, "mixed", True, True)
    for packed in (False, True):
        assert run_binning(harness, g, "perm", P, True, packed, f"empty packed {packed}") == 0


# ---------------------------------------------------------------------------------------------------------------------
# The key at its edges
# ---------------------------------------------------------------------------------------------------------------------
TINY = 5e-324
BIGF = 1.7976931348623157e308
EDGE_GRIDS = {
    "h0.25": Grid((7, 5, 3), lo=(-2.3, -0.7, -1e-310), h=0.25),  # inv_h exact; z0 subnormal
    "h0.1": Grid((7, 5, 3), lo=(-2.3, -0.7, -1e-310), h=0.1),  # inv_h = 10 is not 1 / 0.1
    "far": Grid((7, 5, 3), lo=(-1e308, -0.7, -1.1), h=0.25),  # x - x0 overflows
}


def axis_points(g, a):
    """the coordinates that probe the key of axis a"""
    x0, h, n = g.lo[a], g.h, int(g.dims[a])
    ks = x0 + np.arange(n + 1) * h  # cell faces, up to x0 + n h where the key clamps
    pts = [-np.inf, np.nan, -1e300, x0 - 1e-300, np.nextafter(x0, -np.inf), x0, x0 + TINY, np.nextafter(x0, np.inf),
           *ks, *np.nextafter(ks, -np.inf), *np.nextafter(ks, np.inf), x0 + (n + 5) * h,
           x0 + 2.0**31 * h, np.nextafter(x0 + 2.0**31 * h, -np.inf), x0 + 2.0**40 * h, 1e300, BIGF, -BIGF, np.inf]
    if x0 < -1e300:
        pts += [1e308, 0.0, x0 + 1e292, np.nextafter(x0, np.inf)]
    return np.array(pts)


def edge_particles(rng, g, origin, begin=1):
    """every probe point on each axis with the other two axes inside the box, random combinations of probe points on
    all three, and midpoints: finite, with one NaN or one infinite component, and overflowing x + mx"""
    inside = lambda m: g.lo + (rng.integers(0, g.dims, (m, 3)) + rng.uniform(0.1, 0.9, (m, 3))) * g.h  # noqa: E731
    pts = [axis_points(g, a) for a in range(3)]
    rows = []
    for a in range(3):
        p = inside(len(pts[a]))
        p[:, a] = pts[a]
        rows.append(p)
    combo = np.stack([rng.choice(pts[a], 3000) for a in range(3)], axis=1)
    pos = np.concatenate(rows + [combo, inside(500)])
    m = len(pos)
    dest = np.concatenate([inside(m // 2), np.stack([rng.choice(pts[a], m - m // 2) for a in range(3)], axis=1)])
    dest = dest[rng.permutation(m)]
    pick = rng.permutation(m)
    q = m // 10
    dest[pick[:q], rng.integers(0, 3, q)] = np.nan
    dest[pick[q:2 * q], rng.integers(0, 3, q)] = rng.choice([np.inf, -np.inf], q)
    big = pick[2 * q:2 * q + 50]
    pos[big, 0], dest[big, 0] = 1.5e308, 1.5e308  # x + mx overflows: the midpoint is +inf
    pos[big[:25], 0], dest[big[:25], 0] = -1.5e308, -1.5e308
    N = begin + m + 2
    state = np.empty((N, 4))
    state[:, :3] = inside(N)
    state[begin:begin + m, :3] = pos
    if origin:  # stored positions: mostly the origin, some elsewhere, some the origin's zero of the other sign
        o = state[:, :3].copy()
        other = rng.random(N) < 0.3
        state[other, :3] = rng.permutation(state[:, :3])[other]
        z = np.flatnonzero(o[:, 2] == 0.0)
        state[z, 2] = -o[z, 2]
    state[:, 3] = rng.integers(0, 2**63, N).view(np.float64)
    full_dest = inside(N)
    full_dest[begin:begin + m] = dest
    fl = rng.choice(np.array([1, 1, 1, 0, 2, -1], dtype=np.int8), N)
    return Particles(state, o if origin else None, full_dest, rng.lognormal(0.0, 1.0, N), fl, begin, begin + m)


def test_key_reference_edges():
    """cell_ref at the probe points, spelled out: faces belong to the cell above, the box clamps, NaN and -inf give
    cell 0, +inf and saturating values the last cell, and the h = 0.1 faces round to either side."""
    g = EDGE_GRIDS["h0.25"]
    inside = np.array([[-2.0, -0.5, 0.1]])

    def cx(x):
        p = np.repeat(inside, len(x), axis=0)
        p[:, 0] = x
        return cell_ref(g, p) % 7

    assert list(cx([-np.inf, np.nan, -1e300, -2.3, np.nextafter(-2.3, np.inf)])) == [0, 0, 0, 0, 0]
    faces = -2.3 + np.arange(8) * 0.25
    assert list(cx(faces)) == [0, 1, 2, 3, 4, 5, 6, 6]
    assert list(cx([-2.3 + 2.0**31 * 0.25, 1e300, np.inf, BIGF])) == [6, 6, 6, 6]
    # in z, the subnormal z0: z0 + a subnormal is above it
    assert cell_ref(g, np.array([[-2.0, -0.5, -1e-310 + TINY]]))[0] == cell_ref(g, np.array([[-2.0, -0.5, 0.0]]))[0]
    g1 = EDGE_GRIDS["h0.1"]
    ks = -2.3 + np.arange(8) * 0.1
    p = np.repeat(inside, 8, axis=0)
    p[:, 0] = ks
    c = cell_ref(g1, p) % 7
    assert (c != np.minimum(np.arange(8), 6)).any()  # some rounded faces land in the cell below
    far = EDGE_GRIDS["far"]
    q = np.array([[1e308, -0.5, -1.0], [0.0, -0.5, -1.0], [-1e308, -0.5, -1.0]])
    assert list(cell_ref(far, q) % 7) == [6, 6, 0]  # 1e308 - x0 overflows to +inf


@gpu
@pytest.mark.parametrize("origin", [True, False], ids=["origin", "stored"])
@pytest.mark.parametrize("rank", [None, "perm"])
@pytest.mark.parametrize("name", list(EDGE_GRIDS))
def test_key_edges_are_exact(harness, name, rank, origin):
    g = EDGE_GRIDS[name]
    rng = np.random.default_rng([list(EDGE_GRIDS).index(name), rank is None, origin])
    P = edge_particles(rng, g, origin)
    for mid in (False, True):
        for packed in (False, True):
            run_binning(harness, g, rank, P, mid, packed, f"{name} {rank} origin {origin} mid {mid} packed {packed}")


# ---------------------------------------------------------------------------------------------------------------------
# The initial-weight sum (sum_flying_weights_kernel): *total += the finite weights of the flying particles
# ---------------------------------------------------------------------------------------------------------------------
SUM_N = [1, 31, 32, 33, "wrap-1", "wrap+1", "3wrap+17"]


def _sum_len(n):
    """the grid-stride wrap is 8 blocks of 256 threads per SM"""
    if isinstance(n, int):
        return n
    wrap = 8 * _sms() * 256
    return {"wrap-1": wrap - 1, "wrap+1": wrap + 1, "3wrap+17": 3 * wrap + 17}[n]


def weights_case(rng, N, dyadic):
    """weights with NaN, +-inf, negative and subnormal entries; dyadic: every finite one an integer times 2^-20, with
    a sum of magnitudes below 2^32, so every partial sum of the counted ones is exact"""
    if dyadic:
        w = np.ldexp(rng.integers(-2**20, 2**20, N).astype(np.float64), -20)
    else:
        w = rng.normal(0.0, 1.0, N) * rng.lognormal(0.0, 3.0, N)
    special = rng.random(N) < 0.05
    w[special] = rng.choice(np.array([np.nan, np.inf, -np.inf, TINY, -TINY, 3 * TINY]), int(special.sum()))
    return w


def counted(w, fl):
    """the weights the sum takes: finite, of particles with flying == 1 (every particle without a flying array)"""
    return w[(np.ones(len(w), bool) if fl is None else fl == 1) & np.isfinite(w)]


@gpu
@pytest.mark.parametrize("flying", ["null", "mixed"])
@pytest.mark.parametrize("begin", [0, 13])
@pytest.mark.parametrize("n", SUM_N, ids=str)
def test_flying_weight_sum(harness, n, begin, flying):
    """dyadic weights: start + the counted weights bit for bit, whatever order the atomics take; other weights:
    within (terms + 32) 2^-53 (|start| + sum |w|) of the exact sum.  The second call adds onto the first one's total,
    as each score-bin pass of a binned move does."""
    n = _sum_len(n)
    N = begin + n + 5
    rng = np.random.default_rng([n, begin, flying == "null"])
    fl = None if flying == "null" else rng.choice(np.array([1, 1, 0, 2, -1], dtype=np.int8), N)
    gf = Guarded(fl, seed=1) if fl is not None else None
    for dyadic in (True, False):
        w = weights_case(rng, N, dyadic)
        gw = Guarded(w, 1, seed=2)
        start = np.ldexp(12345.0, -20) if dyadic else 0.75
        total = Guarded(np.array([start]), seed=3)
        c = counted(w[begin:begin + n], None if fl is None else fl[begin:begin + n])
        for call in (1, 2):
            label = f"n {n} begin {begin} flying {flying} dyadic {dyadic} call {call}"
            assert harness.ptb_test_sum_flying_weights(gf.ptr() if gf else None, gw.ptr(), begin, begin + n,
                                                       total.ptr(), _stream()) == 0
            got = total.values()
            want = math.fsum([start, *c, *(c if call == 2 else [])])
            if dyadic:
                assert want != 0.0
                assert_bits(got, np.array([want]), label)
            else:
                bound = (call * len(c) + 33) * 2.0**-53 * (abs(start) + call * float(np.abs(c).sum()))
                assert abs(got[0] - want) <= bound, (label, got[0], want, bound)
            total.assert_unchanged_outside(0, 1, label + " total")
        gw.assert_unchanged_outside(0, 0, "weights")
    if gf is not None:
        gf.assert_unchanged_outside(0, 0, "flying")


@gpu
@pytest.mark.parametrize("case", ["none flying", "no finite weight", "empty range"])
def test_flying_weight_sum_of_nothing_keeps_negative_zero(harness, case):
    n = _sum_len("wrap+1")
    rng = np.random.default_rng(7)
    w = rng.normal(0.0, 1.0, n)
    fl = rng.choice(np.array([0, 2, -1], dtype=np.int8), n) if case == "none flying" else np.ones(n, dtype=np.int8)
    if case == "no finite weight":
        w[:] = rng.choice(np.array([np.nan, np.inf, -np.inf]), n)
    gf, gw = Guarded(fl, seed=1), Guarded(w, seed=2)
    total = Guarded(np.array([-0.0]), seed=3)
    end = 0 if case == "empty range" else n
    assert harness.ptb_test_sum_flying_weights(gf.ptr(), gw.ptr(), 0, end, total.ptr(), _stream()) == 0
    assert_bits(total.values(), np.array([-0.0]), case)
    total.assert_unchanged_outside(0, 1, case)


def test_dyadic_sums_are_exact_in_any_order():
    """the premise of the bit-for-bit check: sequential sums in any order, and numpy's pairwise sum, all give the
    exact sum of dyadic weights (subnormal ones included: a nonzero total absorbs them)"""
    rng = np.random.default_rng(1)
    w = counted(weights_case(rng, 3 * 8 * 132 * 256 + 17, True), None)
    start = np.ldexp(12345.0, -20)
    want = math.fsum([start, *w])
    assert want != 0.0 and (np.abs(w) < 2.0**-1000).any()
    for _ in range(3):
        p = np.r_[start, rng.permutation(w)]
        assert np.cumsum(p)[-1] == want and p.sum() == want and np.cumsum(p[::-1])[-1] == want
