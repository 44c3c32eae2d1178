"""numpy reference of the collision estimator, shared by the host-build and the GPU tests: every event adds w * r[k] to
score k of its element, score bin and time bin (np.add.at), and with moments w * r[k] * (x - C); and the event mixes the
tests feed it (inside, outside and non-finite points, bins and times in and out of range)."""
import numpy as np

from locate_ref import generic_points, non_finite_points, outside_points


def reference_collisions(elem, pts, w, r, bins, times, nbins, edges, nelem, centre):
    """elem: the caller's element of every event (-1 outside).  Returns m0 [T, B, S, E], R [T, B, S, E, 3] (first
    moment about centre), the sums of |addends| of both (the scale of the tolerance) and (tallied, outside, rejected)."""
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    n = len(pts)
    w = np.asarray(w, dtype=np.float64)
    r = np.ones((n, 1)) if r is None else np.asarray(r, dtype=np.float64).reshape(n, -1)
    nscores = r.shape[1]
    bins = np.zeros(n, dtype=np.int64) if bins is None else np.asarray(bins, dtype=np.int64)
    nt = 0 if edges is None else len(edges) - 1
    with np.errstate(invalid="ignore", over="ignore"):
        wr = w[:, None] * r
    bad = ~np.isfinite(pts).all(1) | ~np.isfinite(wr).all(1)
    if nt:
        bad |= ~np.isfinite(times)
    outside = ~bad & (np.asarray(elem) < 0)
    j = np.searchsorted(edges, np.nan_to_num(times), side="right") - 1 if nt else np.zeros(n, dtype=np.int64)
    ok = ~bad & ~outside & (bins >= 0) & (bins < nbins) & (j >= 0) & (j < max(nt, 1))
    T = max(nt, 1)
    m0, a0 = np.zeros((T, nbins, nscores, nelem)), np.zeros((T, nbins, nscores, nelem))
    R, aR = np.zeros((T, nbins, nscores, nelem, 3)), np.zeros((T, nbins, nscores, nelem, 3))
    ids = np.nonzero(ok)[0]
    rel = pts[ids] - np.asarray(centre)
    for k in range(nscores):
        idx = (j[ids], bins[ids], np.full(len(ids), k), np.asarray(elem)[ids])
        v = wr[ids, k]
        np.add.at(m0, idx, v)
        np.add.at(a0, idx, np.abs(v))
        np.add.at(R, idx, v[:, None] * rel)
        np.add.at(aR, idx, np.abs(v[:, None] * rel))
    return m0, R, a0, aR, (int(ok.sum()), int(outside.sum()), int(bad.sum()))


def assert_close(got, want, abs_sum, what, rtol=1e-12):
    err = np.abs(np.asarray(got) - want)
    tol = rtol * abs_sum + 1e-300
    worst = np.unravel_index(np.argmax(err / tol), err.shape)
    assert (err <= tol).all(), f"{what}: off by {err[worst]:.3e} (tolerance {tol[worst]:.3e}) at {worst}"


def event_mix(name, coords, t2v, rng, n, nscores, nbins, edges):
    """n generic interior points (each in one known tet), points outside the mesh and non-finite points, with weights,
    responses, bins (some outside [0, nbins)) and times (some on edges, before T_0 and at or after T_n), a few
    weights, responses and times non-finite; in random order.  Returns pts, elem (-1 outside), w, r, bins, times."""
    p_in, tet = generic_points(name, coords, t2v, n, rng)
    p_out = outside_points(name, coords, rng, 60)
    p_nf = non_finite_points()
    pts = np.concatenate([p_in, p_out, p_nf])
    elem = np.concatenate([tet, -np.ones(len(p_out) + len(p_nf), dtype=np.int64)]).astype(np.int64)
    m = len(pts)
    w = rng.uniform(0.1, 2.0, m)
    r = rng.uniform(-1.0, 2.0, (m, nscores))
    bins = rng.integers(-1, nbins + 1, m).astype(np.int32)
    times = None
    if edges is not None:
        times = rng.uniform(edges[0] - 1.0, edges[-1] + 1.0, m)
        on_edge = rng.random(m) < 0.2
        times[on_edge] = rng.choice(edges, on_edge.sum())
    bad = rng.choice(len(p_in), 24, replace=False)
    w[bad[:8]] = np.nan
    r[bad[8:16], rng.integers(0, nscores, 8)] = np.inf
    if times is not None:
        times[bad[16:]] = rng.choice([np.nan, np.inf, -np.inf], 8)
    else:
        w[bad[16:]] = -np.inf
    order = rng.permutation(m)
    return (pts[order].copy(), elem[order].copy(), w[order].copy(), r[order].copy(), bins[order].copy(),
            None if times is None else times[order].copy())
