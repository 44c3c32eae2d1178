"""Brute-force point location for the point-query tests: barycentric coordinates of every point in every tet (numpy),
and the point sets the tests use on the Kuhn, Delaunay, L-shaped and carved-void meshes."""
import numpy as np

from helpers import carve, l_shaped_mesh
from pumiumtally_b200.mesh import delaunay_box, kuhn_box

BAND = 1e-10  # times the mesh extent: points this close to the hull may get a hull element or -1 (pumitally_c.h)


def barycentric(coords, t2v, pts, elems=None):
    """lam [npts, ntets, 4] (elems None) or lam [npts, 4] of the given element per point (elems >= 0)."""
    v = np.asarray(coords, dtype=np.float64)[np.asarray(t2v)]  # [E, 4, 3]
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    T = np.transpose(v[:, 1:] - v[:, :1], (0, 2, 1))  # columns v1-v0, v2-v0, v3-v0
    Tinv = np.linalg.inv(T)
    if elems is not None:
        e = np.asarray(elems)
        lam123 = np.einsum("nij,nj->ni", Tinv[e], pts - v[e, 0])
        return np.concatenate([1.0 - lam123.sum(1, keepdims=True), lam123], axis=1)
    out = np.empty((len(pts), len(v), 4))
    for a in range(0, len(pts), 256):
        d = pts[a:a + 256, None, :] - v[None, :, 0]
        lam123 = np.einsum("eij,nej->nei", Tinv, d)
        out[a:a + 256] = np.concatenate([1.0 - lam123.sum(2, keepdims=True), lam123], axis=2)
    return out


def containing(coords, t2v, pts, tol=1e-9):
    """bool [npts, ntets]: the tet contains the point (every barycentric coordinate >= -tol)."""
    return (barycentric(coords, t2v, pts) >= -tol).all(axis=2)


def assert_contains(coords, t2v, pts, elems, label, tol=1e-9):
    elems = np.asarray(elems)
    assert (elems >= 0).all(), f"{label}: {(elems < 0).sum()} points inside the mesh got -1"
    lam = barycentric(coords, t2v, pts, elems)
    bad = ~(lam >= -tol).all(axis=1)
    assert not bad.any(), f"{label}: {bad.sum()} points not in their element, e.g. {np.asarray(pts)[bad][:3]}"


def extent(coords):
    c = np.asarray(coords)
    return float((c.max(0) - c.min(0)).max())


# ---- meshes and point sets --------------------------------------------------------------------------------------------
def void_mesh():
    """Kuhn box 5x5x5 with the unit cube [2, 3]^3 carved out: an interior void, hull not convex."""
    c, t = kuhn_box(5, 5, 5)
    cen = c[t].mean(1)
    return carve(c, t, ~(np.abs(cen - 2.5) < 0.5).all(1))


MESHES = {
    "kuhn": lambda: kuhn_box(6, 5, 4),
    "delaunay": lambda: delaunay_box(600),
    "l_shape": lambda: l_shaped_mesh(8, 8, 2),
    "void": void_mesh,
}


def _inside_shape(name, p, margin):
    """Points of the box that lie in the mesh (and not within `margin` of the notch or the void)."""
    if name == "l_shape":
        return ~((p[:, 0] > 4 - margin) & (p[:, 1] > 4 - margin))
    if name == "void":
        return ~(np.abs(p - 2.5) < 0.5 + margin).all(1)
    return np.ones(len(p), dtype=bool)


def generic_points(name, coords, t2v, n, rng):
    """Random points inside the mesh, each at least 1e-7 (barycentric) from every face of its unique tet: (pts, tet)."""
    lo, hi = coords.min(0), coords.max(0)
    p = rng.uniform(lo + 1e-3, hi - 1e-3, size=(4 * n, 3))
    p = p[_inside_shape(name, p, 1e-3)]
    lam = barycentric(coords, t2v, p)
    inside = (lam >= -1e-12).all(axis=2)
    cnt = inside.sum(1)
    tet = inside.argmax(1)
    margin = lam[np.arange(len(p)), tet].min(1)
    keep = (cnt == 1) & (margin > 1e-7)
    return p[keep][:n], tet[keep][:n]


def special_points(coords, t2v):
    """Vertices, edge midpoints and face centres of every tet, minus those on the hull's bounding box (the Kuhn,
    Delaunay and carved meshes put every point of their outer hull there; the notch and void faces are dealt with by
    the caller)."""
    v = coords[t2v]
    edges = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    faces = [(1, 2, 3), (0, 2, 3), (0, 1, 3), (0, 1, 2)]
    pts = np.concatenate([coords] + [0.5 * (v[:, a] + v[:, b]) for a, b in edges] +
                         [(v[:, a] + v[:, b] + v[:, c]) / 3.0 for a, b, c in faces])
    pts = np.unique(pts, axis=0)
    lo, hi = coords.min(0), coords.max(0)
    tol = 1e-9 * extent(coords)
    return pts[~((pts <= lo + tol) | (pts >= hi - tol)).any(1)]


def outside_points(name, coords, rng, n=200):
    lo, hi = coords.min(0), coords.max(0)
    L = hi - lo
    far = np.array([[lo[0] - 100.0, lo[1], lo[2]], [hi[0] + 1.0, 0.5 * (lo[1] + hi[1]), 0.5 * (lo[2] + hi[2])],
                    [1e300, 0.0, 0.0], [-1e300, -1e300, -1e300]])
    shell = rng.uniform(lo - L, hi + L, size=(4 * n, 3))
    shell = shell[((shell < lo - 1e-3 * L) | (shell > hi + 1e-3 * L)).any(1)][:n]
    pts = [far, shell]
    if name == "l_shape":  # the notch x > 4, y > 4
        pts.append(np.column_stack([rng.uniform(4.01, 7.99, n), rng.uniform(4.01, 7.99, n), rng.uniform(0.01, 1.99, n)]))
    if name == "void":
        pts.append(rng.uniform(2.01, 2.99, size=(n, 3)))
    return np.concatenate(pts)


def band_points(name, coords, rng, n=200):
    """Points within BAND * extent of the hull, inside and outside: either answer is right."""
    lo, hi = coords.min(0), coords.max(0)
    ext = extent(coords)
    p = rng.uniform(lo, hi, size=(n, 3))
    axis = rng.integers(0, 3, n)
    side = rng.integers(0, 2, n)
    p[np.arange(n), axis] = np.where(side == 1, hi[axis], lo[axis]) + rng.uniform(-0.9, 0.9, n) * BAND * ext
    p = p[_inside_shape(name, p, 1e-3)]
    extra = []
    if name == "l_shape":  # on the notch's faces x = 4 (y > 4) and y = 4 (x > 4)
        m = n // 2
        q = np.column_stack([4.0 + rng.uniform(-0.9, 0.9, m) * BAND * ext, rng.uniform(4.1, 7.9, m), rng.uniform(0.1, 1.9, m)])
        extra += [q, q[:, [1, 0, 2]]]
    if name == "void":  # on the void's faces
        m = n // 2
        q = rng.uniform(2.1, 2.9, size=(m, 3))
        ax = rng.integers(0, 3, m)
        q[np.arange(m), ax] = rng.choice([2.0, 3.0], m) + rng.uniform(-0.9, 0.9, m) * BAND * ext
        extra.append(q)
    return np.concatenate([p] + extra)


def non_finite_points():
    nan, inf = np.nan, np.inf
    return np.array([[nan, 0.5, 0.5], [0.5, nan, 0.5], [0.5, 0.5, nan], [inf, 0.5, 0.5], [0.5, -inf, 0.5],
                     [0.5, 0.5, inf], [nan, nan, nan]])
