"""numpy restatement of the mesh source (pumitally_c.h, pumitally_set_source / pumitally_sample_source), every operation
rounded as the contract rounds it: the CDF is the sequential sum np.cumsum, sample i of seed takes four SplitMix64
uniforms u = ((z >> 12) + 0.5) * 2^-52, the first entry with C[k] > u_0 T, and the Rocchini-Cignoni fold of
(u_1, u_2, u_3) in the element's vertices."""
import numpy as np

from pumiumtally_b200.workload import _GOLD, _K_STREAM, _M1, _M2

MASK = (1 << 64) - 1


def mix(seed, ids, stream):
    """z of workload._NumpyOps.uniform(ids, seed, step=0, stream) before its final shift (uint64)"""
    ids = np.asarray(ids, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = ids * np.uint64(_GOLD) + np.uint64((int(seed) + stream * _K_STREAM) & MASK)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(_M1)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(_M2)
        return z ^ (z >> np.uint64(31))


def uniform(z):
    return ((np.asarray(z, dtype=np.uint64) >> np.uint64(12)).astype(np.float64) + 0.5) * 2.0 ** -52


def volumes(coords, t2v):
    """|det(v1 - v0, v2 - v0, v3 - v0)| / 6 per element (any volumes will do for the host build; the GPU tests take
    the engine's)"""
    v = np.asarray(coords, dtype=np.float64)[np.asarray(t2v)]
    return np.abs(np.linalg.det(np.transpose(v[:, 1:] - v[:, :1], (0, 2, 1)))) / 6.0


class Table:
    """The table set_source builds from strength q [G, E] (caller's numbering), optional bias b, volumes V [E]."""

    def __init__(self, q, volume, bias=None, per_volume=False):
        q = np.asarray(q, dtype=np.float64)
        self.G, self.E = q.reshape(-1, len(volume)).shape
        q = q.reshape(self.G, self.E)
        qv = q * np.asarray(volume)[None, :] if per_volume else q
        p = qv * np.asarray(bias, dtype=np.float64).reshape(self.G, self.E) if bias is not None else qv
        self.p = p.ravel()
        self.C = np.cumsum(self.p)
        self.T = float(self.C[-1])
        self.Q = float(np.cumsum(qv.ravel())[-1])
        self.bias = None if bias is None else np.asarray(bias, dtype=np.float64).ravel()
        nz = np.nonzero(self.p > 0)[0]
        self.klast = int(nz[-1]) if len(nz) else -1

    def entry(self, x):
        k = np.searchsorted(self.C, x, side="right")
        return np.where(k < len(self.C), k, self.klast)


def fold(s, t, u):
    a = s + t > 1.0
    s, t = np.where(a, 1.0 - s, s), np.where(a, 1.0 - t, t)
    b = t + u > 1.0
    c = ~b & ((s + t) + u > 1.0)
    s2 = np.where(c, (1.0 - t) - u, s)
    t2 = np.where(b, 1.0 - u, t)
    u2 = np.where(b, (1.0 - s) - t, np.where(c, ((s + t) + u) - 1.0, u))
    return s2, t2, u2


def sample(table, coords, t2v, seed, first, n):
    """(xyz [n, 3], elem [n], group [n], weight [n]) of samples first .. first + n - 1"""
    ids = np.arange(n, dtype=np.uint64) + np.uint64(first)
    u0, s, t, u = (uniform(mix(seed, ids, k)) for k in range(4))
    k = table.entry(u0 * table.T)
    s, t, u = fold(s, t, u)
    g, e = k // table.E, k % table.E
    v = np.asarray(coords, dtype=np.float64)[np.asarray(t2v)[e]]  # [n, 4, 3]
    xyz = v[:, 0] + ((s[:, None] * (v[:, 1] - v[:, 0]) + t[:, None] * (v[:, 2] - v[:, 0])) +
                     u[:, None] * (v[:, 3] - v[:, 0]))
    w = (table.T / table.Q) / table.bias[k] if table.bias is not None else np.ones(n)
    return xyz, e.astype(np.int32), g.astype(np.int32), w
