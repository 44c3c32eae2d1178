"""Exact reference for the cosine bins of the face currents, on top of face_currents_ref.face_walk (unchanged): the
cosine of a crossing is the unit normal of the face it leaves through dotted with the unit direction of its flight,
taken from the unit planes, clamped at 1.  A crossing whose cosine lies within 1e-9 of a cosine edge is ambiguous (the
engine's normals carry a payload byte and its n.u is rounded differently), and the tests do not fly it."""
import numpy as np

from face_currents_ref import face_walk, reference_currents


def cosine_bins(mu, mu_edges):
    """OpenMC's MuFilter rule: bin k holds edges[k] <= mu < edges[k + 1], mu == edges[-1] the last bin; -1 outside."""
    C = len(mu_edges) - 1
    k = np.searchsorted(mu_edges, mu, side="right") - 1
    k = np.where(mu == mu_edges[-1], C - 1, k)
    return np.where((mu >= mu_edges[0]) & (mu <= mu_edges[-1]), k, -1)


def cosine_walk(planes, adj, start, a, b, alive, mu_edges, t0=None, tpp=None, edges=None, max_iters=None):
    """face_walk's crossings with each crossing's cosine: (ids, elem, face, time_bin, mu, ambiguous[n]).  A flight with
    a crossing within 1e-9 of a cosine edge is ambiguous as well."""
    ids, e, f, j, amb = face_walk(planes, adj, start, a, b, alive, t0, tpp, edges, max_iters)
    normals = planes[0]
    a, b = np.asarray(a, dtype=np.float64).reshape(-1, 3), np.asarray(b, dtype=np.float64).reshape(-1, 3)
    d = b - a
    u = d / np.linalg.norm(d, axis=1, keepdims=True).clip(1e-300)
    mu = np.minimum(np.einsum("ik,ik->i", normals[e, f], u[ids]), 1.0)
    near = np.min(np.abs(mu[:, None] - np.asarray(mu_edges)[None, :]), axis=1) < 1e-9
    amb = amb.copy()
    amb[ids[near]] = True
    return ids, e, f, j, mu, amb


def reference_cosine_currents(adj, crossings, w, bins, ntime, nbins, mu_edges):
    """(out, in) [ntime, nbins, C, E, 4]: reference_currents of the crossings of each cosine bin."""
    ids, e, f, j, mu = crossings[:5]
    k = cosine_bins(mu, np.asarray(mu_edges))
    C = len(mu_edges) - 1
    out = np.zeros((ntime, nbins, C, len(adj), 4))
    inn = np.zeros_like(out)
    for c in range(C):
        m = k == c
        out[:, :, c], inn[:, :, c] = reference_currents(adj, (ids[m], e[m], f[m], j[m]), w, bins, ntime, nbins)
    return out, inn
