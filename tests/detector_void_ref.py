"""Numpy reference of the detector void (pumitally_set_detector_void): tests/detectors_ref.py without its shadow test.
Every ray's optical depth is the clip of its whole segment against every tet, tau = fsum(Sigma * l), so the parts
outside the mesh add nothing; events outside the mesh are traced like the others, and inside r0 they score the ball
formula with Sigma = 0.  Shared by the host-build and the GPU tests."""
import math

import numpy as np

from detectors_ref import ball_g, ray_lengths
from helpers import carve
from pumiumtally_b200.mesh import kuhn_box


def reference_void(coords, t2v, elem, pts, w, pdf, r, bins, times, speeds, edges, nbins, nscores, sigma, det, r0):
    """out [T, nbins, nscores, D] and counts (traced, shadowed, lost, inside_r0, crossings (None: not modelled),
    outside, rejected) for the events at pts in elements elem (caller's numbering, -1 outside); sigma [nbins, E]."""
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
        if not bad:
            bad = any(r0[d] == 0.0 and float(np.sqrt(((det[d] - pts[i]) ** 2).sum())) == 0.0 for d in range(D))
        if bad:
            counts[6] += 1
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
                s = sigma[b, elem[i]] if elem[i] >= 0 else 0.0
                f = p * 3.0 * ball_g(s * r0[d]) / r0[d] ** 2
                counts[3] += 1
            else:
                tau = math.fsum(sigma[b] * ray_lengths(coords, t2v, pts[i], det[d]))
                f = p * math.exp(-tau) / R ** 2
                counts[0] += 1
            out[j, b, :, d] += wr * f
    return out, tuple(counts)


def comb_mesh(slots=4, ny=3, nz=2):
    """A Kuhn box [0, 2 slots + 1] x [0, ny] x [0, nz] with open slots x in [2k + 1, 2k + 2], y > 1 carved across x: the
    slabs x in [2k, 2k + 1] are joined by the bridge y < 1.  Hull not convex."""
    c, t = kuhn_box(2 * slots + 1, ny, nz)
    cen = c[t].mean(1)
    slot = (np.floor(cen[:, 0]).astype(int) % 2 == 1) & (cen[:, 1] > 1.0)
    return carve(c, t, ~slot)


def comb_slab_of(x):
    """Index of the comb's slab that holds x (x in [2k, 2k + 1]), -1 in a slot or outside."""
    k = math.floor(x / 2.0)
    return k if x - 2.0 * k <= 1.0 else -1
