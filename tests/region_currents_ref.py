"""Independent numpy construction of the region-current pair plan (batch_stats.cuh, build_region_current_plan) from the
face adjacency and a region map: which face-current slots belong to which ordered pair of regions, the reverse of
every pair, the face areas, and the order in which the engine sums a pair's slots."""
import numpy as np

from face_currents_ref import back_faces

CHUNK = 32      # kRegionChunk
OUTSIDE = -2    # kOutside: the region of "outside the mesh"


def pair_plan(adj, region):
    """(frm, to, first, slots): the pairs in ascending (from, to) order, and pair p's slots, ascending, in
    slots[first[p]:first[p + 1]].  Slot 4 n + b is the incoming current of face b of element n (an interior face),
    slot 4 e + f of a hull face its outgoing current, in the numbering of adj."""
    adj = np.asarray(adj, dtype=np.int64)
    region = np.asarray(region, dtype=np.int64)
    E = len(adj)
    back = back_faces(adj)
    e = np.repeat(np.arange(E), 4)
    f = np.tile(np.arange(4), E)
    nb = adj[e, f]
    hull = nb < 0
    nbc = np.where(hull, 0, nb)
    a = region[e]
    b = np.where(hull, OUTSIDE, region[nbc])
    slot = np.where(hull, 4 * e + f, 4 * nbc + back[e, f])
    keep = hull | (a != b)
    a, b, slot = a[keep], b[keep], slot[keep]
    order = np.lexsort((slot, b, a))
    a, b, slot = a[order], b[order], slot[order]
    new = np.ones(len(a), dtype=bool)
    new[1:] = (a[1:] != a[:-1]) | (b[1:] != b[:-1])
    starts = np.flatnonzero(new)
    first = np.append(starts, len(a))
    return a[starts].astype(np.int32), b[starts].astype(np.int32), first, slot


def reverse(frm, to):
    """rev[p]: the index of pair to[p] -> frm[p], -1 where there is none"""
    index = {(int(x), int(y)): i for i, (x, y) in enumerate(zip(frm, to))}
    return np.array([index.get((int(y), int(x)), -1) for x, y in zip(frm, to)], dtype=np.int32)


def face_areas(coords, t2v):
    """[E, 4] |(b - a) x (c - a)| / 2 of the face opposite each local vertex, a, b, c the other vertices in local order,
    every operation rounded separately (as face_area)"""
    coords = np.asarray(coords, dtype=np.float64)
    out = np.empty((len(t2v), 4))
    for f in range(4):
        q = [i for i in range(4) if i != f]
        v0, v1, v2 = (coords[np.asarray(t2v)[:, i]] for i in q)
        u, w = v1 - v0, v2 - v0
        x = u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1]
        y = u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2]
        z = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
        s = x * x + y * y
        out[:, f] = np.sqrt(s + z * z) * 0.5
    return out


def plan_sum(x):
    """The sum of x in the order of the region sums: chunks of CHUNK summed left to right, level by level"""
    x = [float(v) for v in x]
    while True:
        c = (len(x) + CHUNK - 1) // CHUNK if len(x) > CHUNK else 1
        sums = []
        for j in range(c):
            part = x[j * CHUNK:(j + 1) * CHUNK] if c > 1 else x
            acc = part[0] if part else 0.0
            for v in part[1:]:
                acc += v
            sums.append(acc)
        x = sums
        if c == 1:
            return x[0]


def pair_values(values, first, slots):
    """[..., P]: the sums of values[..., slot] over each pair's slots (numpy's order, for comparisons to a
    tolerance)"""
    values = np.asarray(values)
    return np.stack([values[..., slots[first[p]:first[p + 1]]].sum(axis=-1) for p in range(len(first) - 1)], axis=-1)
