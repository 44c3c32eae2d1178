"""Reference for the time filter, shared by the host-build and the GPU tests: every flight is cut at the time-bin
edges and the pieces of bin j are tallied by the oracle's brute-force integrator, one score at a time."""
import numpy as np

from oracle.oracle import bruteforce_tally


def time_pieces(start, end, times, speeds, edges, alive):
    """Pieces of the flights start -> end (already clipped where the walk stops) per time bin.

    Particle i is at time times[i] at start[i] and moves at speeds[i].  Returns a list over the bins of
    (a, b, ids): piece start and end points and the particles that have a piece of non-zero length in the bin."""
    start, end = np.asarray(start, dtype=np.float64).reshape(-1, 3), np.asarray(end, dtype=np.float64).reshape(-1, 3)
    length = np.linalg.norm(end - start, axis=1)
    ok = alive & (length > 0)
    out = []
    for j in range(len(edges) - 1):
        with np.errstate(invalid="ignore", over="ignore"):
            s_lo = np.clip((edges[j] - times) * speeds, 0.0, length)
            s_hi = np.clip((edges[j + 1] - times) * speeds, 0.0, length)
        ids = np.nonzero(ok & (s_hi > s_lo))[0]
        f_lo = (s_lo[ids] / length[ids])[:, None]
        f_hi = (s_hi[ids] / length[ids])[:, None]
        d = end[ids] - start[ids]
        out.append((start[ids] + f_lo * d, start[ids] + f_hi * d, ids))
    return out


def reference_time_tally(coords, t2v, start, end, times, speeds, edges, alive, w, r):
    """flux[time, score, element]: score k of time bin j is the brute-force tally of bin j's pieces with weights
    w * r[:, k]."""
    r = np.asarray(r, dtype=np.float64).reshape(len(w), -1)
    nt, ns = len(edges) - 1, r.shape[1]
    flux = np.zeros((nt, ns, len(t2v)))
    for j, (a, b, ids) in enumerate(time_pieces(start, end, times, speeds, edges, alive)):
        if len(ids) == 0:
            continue
        for k in range(ns):
            flux[j, k] = bruteforce_tally(coords, t2v, a, b, w[ids] * r[ids, k])[0]
    return flux


def time_workload(rng, o, d, box_scale, edges):
    """Times and speeds for flights o -> d such that most flights cross an edge, some cross several, and some start
    before the first edge or after the last one."""
    n = len(o)
    span = edges[-1] - edges[0]
    width = span / (len(edges) - 1)
    times = rng.uniform(edges[0] - 0.25 * span, edges[-1] + 0.1 * span, n)
    duration = rng.uniform(0.3 * width, 4.0 * width, n)
    length = np.maximum(np.linalg.norm(np.asarray(d).reshape(-1, 3) - np.asarray(o).reshape(-1, 3), axis=1),
                        1e-3 * box_scale)
    speeds = length / duration
    return times, speeds


def edge_crossings(o, d, times, speeds, edges, alive):
    """Edges strictly inside each flight's time span (the unclipped flight)."""
    length = np.linalg.norm(np.asarray(d).reshape(-1, 3) - np.asarray(o).reshape(-1, 3), axis=1)
    t1 = times + length / speeds
    inner = (edges[None, :] > times[:, None]) & (edges[None, :] < t1[:, None])
    return np.where(alive, inner.sum(axis=1), 0)
