"""Exact reference for the linear flux moments, shared by the host-build and the GPU tests: every tallied segment is
clipped against every tet's four half-spaces, and each piece adds w * r * l and w * r * l * (x_mid - c_e)."""
import numpy as np

from time_bins_ref import time_pieces


def tet_geometry(coords, t2v):
    """Per tet: centroid [E, 3], diameter [E], and the half-spaces n . x <= c as normals [E, 4, 3], offsets [E, 4]."""
    v = np.asarray(coords, dtype=np.float64)[np.asarray(t2v)]  # [E, 4, 3]
    cen = v.mean(axis=1)
    diam = np.max(np.linalg.norm(v[:, :, None, :] - v[:, None, :, :], axis=-1), axis=(1, 2))
    normals = np.empty((len(v), 4, 3))
    offsets = np.empty((len(v), 4))
    for f in range(4):
        a, b, c = (v[:, q] for q in range(4) if q != f)
        n = np.cross(b - a, c - a)
        off = np.einsum("ij,ij->i", n, a)
        inside = np.einsum("ij,ij->i", n, v[:, f]) > off  # make the opposite vertex satisfy n . x <= c
        n[inside] *= -1.0
        off[inside] *= -1.0
        normals[:, f], offsets[:, f] = n, off
    return cen, diam, normals, offsets


def segment_moments(coords, t2v, a, b, wr):
    """Track-length tally of segments a -> b with weights wr [n, nscores]: m0 [nscores, E], m1 [nscores, E, 3] about
    the tet centroids, abs_sum [nscores, E] = sum |wr * l| (the scale of the tolerance) and abs_w [nscores, E] = sum
    |wr| over the segments that cross the tet (the scale of an error in where a segment starts or ends)."""
    a, b = np.asarray(a, dtype=np.float64).reshape(-1, 3), np.asarray(b, dtype=np.float64).reshape(-1, 3)
    wr = np.asarray(wr, dtype=np.float64).reshape(len(a), -1)
    cen, _, normals, offsets = tet_geometry(coords, t2v)
    E, ns = len(cen), wr.shape[1]
    m0, m1, abs_sum, abs_w = np.zeros((ns, E)), np.zeros((ns, E, 3)), np.zeros((ns, E)), np.zeros((ns, E))
    d = b - a
    length = np.linalg.norm(d, axis=1)
    for lo in range(0, E, 64):
        sl = slice(lo, min(E, lo + 64))
        alpha = np.einsum("efk,nk->efn", normals[sl], a) - offsets[sl][:, :, None]  # [e, 4, n]
        beta = np.einsum("efk,nk->efn", normals[sl], d)
        with np.errstate(divide="ignore", invalid="ignore"):
            t = -alpha / beta
        t0 = np.where(beta < 0, t, -np.inf).max(axis=1).clip(0.0, 1.0)
        t1 = np.where(beta > 0, t, np.inf).min(axis=1).clip(0.0, 1.0)
        blocked = ((beta == 0) & (alpha > 0)).any(axis=1)
        frac = np.where(blocked, 0.0, np.maximum(t1 - t0, 0.0))  # [e, n]
        ell = frac * length[None, :]
        mid = a[None] + (0.5 * (t0 + t1))[:, :, None] * d[None]  # [e, n, 3]
        rel = mid - cen[sl][:, None, :]
        for k in range(ns):
            wl = ell * wr[None, :, k]
            m0[k, sl] = wl.sum(axis=1)
            m1[k, sl] = np.einsum("en,enk->ek", wl, rel)
            abs_sum[k, sl] = np.abs(wl).sum(axis=1)
            abs_w[k, sl] = ((frac > 0) * np.abs(wr[None, :, k])).sum(axis=1)
    return m0, m1, abs_sum, abs_w


def reference_moments(coords, t2v, start, end, alive, w, r, edges=None, times=None, speeds=None):
    """m0 [ntime, nscores, E], m1 [ntime, nscores, E, 3], abs_sum and abs_w [ntime, nscores, E] of flights start -> end
    (already clipped where the walk stops); with edges, every flight is cut at the time-bin edges first."""
    w = np.asarray(w, dtype=np.float64)
    r = np.asarray(r, dtype=np.float64).reshape(len(w), -1)
    start, end = np.asarray(start, dtype=np.float64).reshape(-1, 3), np.asarray(end, dtype=np.float64).reshape(-1, 3)
    if edges is None:
        ids = np.nonzero(alive)[0]
        pieces = [(start[ids], end[ids], ids)]
    else:
        pieces = time_pieces(start, end, times, speeds, edges, alive)
    out = [segment_moments(coords, t2v, a, b, w[ids, None] * r[ids]) for a, b, ids in pieces]
    return tuple(np.stack([o[q] for o in out]) for q in range(4))


def assert_moments_close(m1, want_m1, abs_sum, diam, what, rtol=1e-9, cut=0.0, abs_w=0.0):
    """|m1 - want| <= rtol * diam_e * sum |w r l|_e per element and component (a tolerance relative to |m1| would be
    meaningless where the moment is near zero).  cut: the error in the position of a piece's end that the reference
    itself computes differently from the walk (the time-bin cuts), weighted by abs_w."""
    tol = diam[None, :, None] * (rtol * abs_sum + cut * np.asarray(abs_w))[..., None] + 1e-300
    err = np.abs(np.asarray(m1) - want_m1)
    worst = np.unravel_index(np.argmax(err / tol), err.shape)
    assert (err <= tol).all(), f"{what}: m1 off by {err[worst]:.3e} (tolerance {tol[worst]:.3e}) at {worst}"


def assert_m0_close(m0, want_m0, abs_sum, what, rtol=1e-9, cut=0.0, abs_w=0.0):
    err = np.abs(np.asarray(m0) - want_m0)
    tol = rtol * abs_sum + cut * np.asarray(abs_w) + 1e-300
    assert (err <= tol).all(), f"{what}: m0 off by up to {err.max():.3e}"


def tet_quadrature_moments(coords, t2v, centre, value, grad):
    """Exact moments of the linear field phi(x) = value + grad . (x - centre) on every tet, from the 4-point rule
    that integrates quadratics exactly: m0 = int phi, R = int (x - centre) phi."""
    v = np.asarray(coords, dtype=np.float64)[np.asarray(t2v)]
    e1, e2, e3 = v[:, 1] - v[:, 0], v[:, 2] - v[:, 0], v[:, 3] - v[:, 0]
    vol = np.abs(np.einsum("ij,ij->i", e1, np.cross(e2, e3))) / 6.0
    al, be = 0.5854101966249685, 0.1381966011250105
    m0, R = np.zeros(len(v)), np.zeros((len(v), 3))
    for q in range(4):
        lam = np.full(4, be)
        lam[q] = al
        x = np.einsum("q,eqk->ek", lam, v)
        phi = value + (x - centre) @ grad
        m0 += 0.25 * vol * phi
        R += 0.25 * vol[:, None] * (x - centre) * phi[:, None]
    return m0, R, vol
