"""Exact reference for the face currents: every flight is walked tet by tet by clipping it against the current tet's
four half-spaces (the planes of tet_geometry in moments_ref.py).  The exit face is the face with the smallest exit
parameter; a flight stops when its destination lies in the tet or when it leaves through a hull face.

Flights whose walk is not decided far from rounding are reported as ambiguous, and the tests do not fly them: an
origin within 1e-7 of a face of its tet, a crossing within 1e-7 (in track length) of a second face (an edge), a
destination within 1e-9 of a face, and, with time bins, a crossing time within 1e-9 of a bin edge."""
import numpy as np

from moments_ref import tet_geometry


def unit_planes(coords, t2v):
    _, _, normals, offsets = tet_geometry(coords, t2v)
    norm = np.linalg.norm(normals, axis=-1)
    return normals / norm[..., None], offsets / norm


def face_walk(planes, adj, start, a, b, alive, t0=None, tpp=None, edges=None, max_iters=None):
    """Crossings of the flights a[i] -> b[i] (alive[i]) from element start[i] (caller's numbering, adj [E, 4] from the
    engine's adjacency).  Returns (ids, elem, face, time_bin, ambiguous[n]): one entry per crossing, elem the element
    left through its local face; time_bin 0 without edges.  max_iters: the walk's crossing limit -- step k >= max_iters
    stops the flight, and its face counts only when it is a hull face."""
    normals, offsets = planes
    a, b = np.asarray(a, dtype=np.float64).reshape(-1, 3), np.asarray(b, dtype=np.float64).reshape(-1, 3)
    d = b - a
    length = np.linalg.norm(d, axis=1)
    n = len(a)
    cur = np.asarray(start, dtype=np.int64).copy()
    amb = np.zeros(n, dtype=bool)
    # the origin must lie clearly inside its element
    ids = np.nonzero(alive)[0]
    dist = np.einsum("ifk,ik->if", normals[cur[ids]], a[ids]) - offsets[cur[ids]]
    amb[ids[dist.max(axis=1) > -1e-7]] = True
    active = np.asarray(alive, dtype=bool) & (length > 0)
    out = ([], [], [], [])
    for it in range(len(adj) + 16):
        ids = np.nonzero(active)[0]
        if len(ids) == 0:
            break
        e = cur[ids]
        alpha = np.einsum("ifk,ik->if", normals[e], a[ids]) - offsets[e]
        beta = np.einsum("ifk,ik->if", normals[e], d[ids])
        with np.errstate(divide="ignore", invalid="ignore"):
            t = np.where(beta > 1e-12 * length[ids, None], -alpha / beta, np.inf)
        order = np.argsort(t, axis=1)
        f = order[:, 0]
        tmin = np.take_along_axis(t, order[:, :1], 1)[:, 0]
        t2 = np.take_along_axis(t, order[:, 1:2], 1)[:, 0]
        reached = tmin >= 1.0
        amb[ids[np.abs(tmin - 1.0) * length[ids] < 1e-9]] = True
        amb[ids[~reached & ((t2 - tmin) * length[ids] < 1e-7)]] = True
        over = max_iters is not None and it + 1 >= max_iters
        cross = ~reached
        j = np.zeros(len(ids), dtype=np.int64)
        if edges is not None:
            tc = t0[ids] + tmin * tpp[ids]
            j = np.searchsorted(edges, tc, side="left") - 1  # a crossing exactly on an edge stays in the bin below
            with np.errstate(invalid="ignore"):
                near = np.min(np.abs(tc[:, None] - edges[None, :]), axis=1) < 1e-9 * (1.0 + np.abs(tc))
            amb[ids[cross & near]] = True
        nxt = adj[e, f]
        hull = cross & (nxt < 0)
        counted = cross & (hull | (not over))
        for lst, v in zip(out, (ids, e, f, j)):
            lst.append(v[counted])
        active[ids[reached | hull]] = False
        if over:
            active[ids] = False
        step = cross & ~hull
        cur[ids[step]] = nxt[step]
    return tuple(np.concatenate(x) if x else np.zeros(0, dtype=np.int64) for x in out) + (amb,)


def reference_currents(adj, crossings, w, bins, ntime, nbins):
    """(out, in) [ntime, nbins, E, 4] of the crossings face_walk returned, for the flights that flew: a crossing out of
    (e, f) adds w to out[e, f] and, for an interior face, to in of the neighbour's face that matches it."""
    ids, e, f, j = crossings[:4]
    E = len(adj)
    out = np.zeros((ntime, nbins, E, 4))
    inn = np.zeros((ntime, nbins, E, 4))
    b = np.zeros(len(ids), dtype=np.int64) if bins is None else np.asarray(bins)[ids]
    keep = (b >= 0) & (b < nbins) & (j >= 0) & (j < ntime)
    ids, e, f, j, b = ids[keep], e[keep], f[keep], j[keep], b[keep]
    np.add.at(out, (j, b, e, f), w[ids])
    nb = adj[e, f]
    interior = nb >= 0
    back = np.argmax(adj[nb[interior]] == e[interior, None], axis=1)
    np.add.at(inn, (j[interior], b[interior], nb[interior], back), w[ids[interior]])
    return out, inn


def back_faces(adj):
    """back[e, f]: the neighbour's local index of face f of e (-1 on the hull)."""
    E = len(adj)
    back = -np.ones((E, 4), dtype=np.int64)
    e, f = np.nonzero(adj >= 0)
    back[e, f] = np.argmax(adj[adj[e, f]] == e[:, None], axis=1)
    return back
