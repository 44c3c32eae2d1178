"""Numpy reference of the point detectors (walk_core.cuh, detector_event): every ray's optical depth from the clip of its
segment against every tet (moments_ref.segment_moments), tau = fsum(Sigma * l), then the scoring rules of
include/pumitally_c.h.  Shared by the host-build and the GPU tests."""
import math

import numpy as np

from locate_ref import barycentric
from moments_ref import segment_moments


def ball_g(x):
    return -math.expm1(-x) / x if x > 0 else 1.0


def locate(coords, t2v, pts, tol=1e-12):
    """The first tet that contains each point (every barycentric coordinate >= -tol), -1 outside."""
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    inside = (barycentric(coords, t2v, pts) >= -tol).all(axis=2)
    return np.where(inside.any(1), inside.argmax(1), -1)


def ray_lengths(coords, t2v, a, b):
    """Length of the segment a -> b inside every tet [E]."""
    m0, _, _, _ = segment_moments(coords, t2v, a[None], b[None], np.ones((1, 1)))
    return m0[0]


def reference_detectors(coords, t2v, elem, pts, w, pdf, r, bins, times, speeds, edges, nbins, nscores, sigma, det, r0):
    """out [T, nbins, nscores, D] and counts (traced, shadowed, lost, inside_r0, crossings (None: not modelled), outside,
    rejected) for the events at pts in elements elem (caller's numbering, -1 outside); sigma [nbins, E]."""
    n, D = len(pts), len(det)
    T = 1 if edges is None else len(edges) - 1
    out = np.zeros((T, nbins, nscores, D))
    counts = [0, 0, 0, 0, None, 0, 0]
    for i in range(n):
        wr = w[i] * (np.ones(nscores) if r is None else r[i])
        bad = not np.isfinite(pts[i]).all() or not np.isfinite(wr).all()
        if edges is not None:
            bad = bad or not math.isfinite(times[i]) or not (speeds[i] > 0)
        if pdf is not None:
            bad = bad or not np.isfinite(pdf[i]).all() or (pdf[i] < 0).any()
        if not bad:  # an event exactly on a detector without an exclusion radius
            bad = any(r0[d] == 0.0 and float(np.sqrt(((det[d] - pts[i]) ** 2).sum())) == 0.0 for d in range(D))
        if bad:
            counts[6] += 1
            continue
        if elem[i] < 0:
            counts[5] += 1
            continue
        b = 0 if bins is None else int(bins[i])
        for d in range(D):
            p = 0.25 / math.pi if pdf is None else pdf[i, d]
            R = float(np.sqrt(((det[d] - pts[i]) ** 2).sum()))
            j = 0
            if edges is not None:
                j = int(np.searchsorted(edges, times[i] + R / speeds[i], side="right")) - 1
            if not (0 <= b < nbins) or j < 0 or j >= T:
                continue
            if R < r0[d]:
                f = p * 3.0 * ball_g(sigma[b, elem[i]] * r0[d]) / r0[d] ** 2
                counts[3] += 1
            else:
                ell = ray_lengths(coords, t2v, pts[i], det[d])
                if ell.sum() < R * (1.0 - 1e-9):  # part of the line lies outside the mesh: shadowed
                    counts[1] += 1
                    continue
                tau = math.fsum(sigma[b] * ell)
                f = p * math.exp(-tau) / R ** 2
                counts[0] += 1
            out[j, b, :, d] += wr * f
    return out, tuple(counts)
