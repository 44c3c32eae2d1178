"""The point-detector kernels (csrc/detector_kernels.cu) bit for bit, on both sides of the shared-memory slot limit
(kDetSmemSlots), across the per-launch ray split of the located calls and past 2^31 rays.

Each kernel is built twice: up to kDetSmemSlots slots (ntime * nbins * nscores * D) the block aggregates into a shared
copy of the slots; above that each warp groups the lanes of one slot with match.any and one lane adds their shuffled
sum.  The tests here reach both, in all four kernels (located or at the particles, with the detector void or without).

Most of them use an exactly summable construction (exact_case): Sigma_t = 0, so that exp(-tau) = 1 whatever tets a ray
crosses; every event sits 2^k (k in -2..1) from its home detector along one axis, on a 1/64 grid; the pdf is m / 64 at
the home detector and 0 at every other one, weights +-m / 4, responses m / 4, exclusion radii and speeds powers of two.
Every score is then an integer multiple of 2^-12 far below 2^53 (asserted), any order of summation gives the same bits,
and the reference is an int64 sum.  Every other ray is still traced, counted and aggregated: it scores exactly 0."""
import json
import math
import os
import re
from fractions import Fraction

import numpy as np
import pytest

from detector_void_ref import comb_mesh, reference_void
from detectors_ref import reference_detectors
from helpers import ROOT, l_shaped_mesh
from locate_ref import MESHES, generic_points
from pumiumtally_b200.mesh import kuhn_box
from test_gpu_stats_kernels import kernels_launched, run_in_fresh_process

U = 4096  # every score of exact_case is an integer multiple of 1 / U
COUNTERS = ("detector_rays", "detector_rays_shadowed", "detector_rays_lost", "detector_inside_r0",
            "detector_events_outside", "detector_events_rejected", "detector_hull_entries")


def smem_slots():
    """kDetSmemSlots, as walk_kernels.hpp defines it."""
    src = open(os.path.join(ROOT, "pumiumtally_b200", "csrc", "walk_kernels.hpp")).read()
    return int(re.search(r"constexpr int64_t kDetSmemSlots = (\d+);", src).group(1))


# ---- the exactly summable construction ------------------------------------------------------------------------------
def _box_margin(L):
    L = np.asarray(L, dtype=np.float64)
    return lambda p: np.minimum(p, L - p).min(-1)


def _l_margin(p):
    """Distance (a lower bound) from p into l_shaped_mesh(8, 8, 2): [0, 8]^2 x [0, 2] less the notch x > 4, y > 4;
    negative outside."""
    box = np.minimum(p, np.array([8.0, 8.0, 2.0]) - p).min(-1)
    return np.minimum(box, np.maximum(4.0 - p[..., 0], 4.0 - p[..., 1]))


def _notch_crossing(a, b, m):
    """The segments a -> b [..., 3]: 1 where their xy projection runs through the notch (4, 8)^2 of the L-shaped mesh
    for a length > m, 0 where it stays m away from it, -1 in between."""
    def clipped(c):
        t0, t1 = np.zeros(a.shape[:-1]), np.ones(a.shape[:-1])
        for ax in (0, 1):
            u = b[..., ax] - a[..., ax]
            with np.errstate(divide="ignore", invalid="ignore"):
                s = (c - a[..., ax]) / u
            up = u > 0
            dn = u < 0
            t0 = np.where(up, np.maximum(t0, s), t0)
            t1 = np.where(dn, np.minimum(t1, s), t1)
            par = u == 0  # parallel: inside the half plane x > c or not at all
            t1 = np.where(par & ~(a[..., ax] > c), -1.0, t1)
        return np.maximum(t1 - t0, 0.0) * np.sqrt(((b - a)[..., :2] ** 2).sum(-1))

    inner, outer = clipped(4.0 + m), clipped(4.0 - m)
    return np.where(inner > m, 1, np.where(outer == 0.0, 0, -1))


def _place(rng, D, lo, hi, margin, face, offs, sep):
    """D distinct detectors on the 1/64 grid in [lo, hi], at least 0.5 inside; the first `face` at x = 0.5.  None
    lies closer than sep to another's candidate event positions (det + offs)."""
    det = []
    seen = set()
    while len(det) < D:
        p = rng.integers(np.round(lo * 64), np.round(hi * 64) + 1) / 64.0
        if len(det) < face:
            p[0] = 0.5
        if margin(p) < 0.5 or tuple(p) in seen:
            continue
        if sep and det and (((p - np.array(det)[:, None, :] - offs[None]) ** 2).sum(-1) < sep * sep).any():
            continue
        seen.add(tuple(p))
        det.append(p)
    return np.array(det)


def exact_case(seed, D, n, T=0, nbins=1, nscores=1, L=(8, 8, 8), shape="box", ks=(-2, -1, 0, 1),
               r0s=(0.125, 0.5, 1.0), n_outside=0, specials=("nan", "negpdf", "bin", "bin_neg", "late", "early"),
               cover=0.75, n_cancel=8, hot=None, isolate=False, lost=False, step=1.0, fracs=(0.0, 0.25, 0.5, 0.75),
               arrive=None):
    """Events, detectors and the exact expectation (see the module docstring).

    Events: one per home group (time bin, score bin, detector) for a fraction `cover` of the groups, with positive
    weights; n_cancel pairs of opposite weights, each alone in a group (their slots cancel to 0); n_outside events
    outside the box by at least 0.25, homed on detectors at x = 0.5; special events that score nothing (a NaN weight or
    a negative pdf value: rejected; a score bin out of range, or a home arrival on T_nt or 2^-12 before T_0: skipped),
    each in a warp next to an event that scores into slot 0; the rest in random groups (all in group `hot` if given).
    The time edges are step * (0..T), step a power of two.  Every home arrival a = step (j + f), f in fracs, is dyadic
    and t = a - R / v, so that t + R / v == a: with f = 0 some a lie on an edge (the upper bin).  arrive(j, f), if
    given, is the home arrival instead (dyadic, in bin j).
    isolate: no event lies within r0 of another detector.  lost: every traced ray stops at its first crossing
    (max_iters = 1 on a mesh whose tets are smaller than every R), so only the rays inside r0 score."""
    rng = np.random.default_rng(seed)
    L = np.asarray(L, dtype=np.float64)
    margin = _l_margin if shape == "l" else _box_margin(L)
    Tp = max(T, 1)
    kmax = 2.0 ** max(ks)
    lo = np.minimum(0.25 + kmax, L / 2 - 0.25)
    hi = L - lo
    face = min(D, 2) if n_outside else 0
    for _ in range(200):
        # candidate event positions: det + s 2^k e_a, at least 0.25 inside (or, for the outside events, outside)
        offs = np.array([s * 2.0 ** k * np.eye(3)[a] for k in ks for s in (-1, 1) for a in range(3)])
        det = _place(rng, D, lo, hi, margin, face, offs, max(r0s) if isolate else 0.0)
        r0 = rng.choice(np.asarray(r0s), D)
        cand = (det[:, None, :] + offs[None]).reshape(-1, 3)
        chome = np.repeat(np.arange(D), len(offs))
        ck = np.tile(np.repeat(np.array(ks), 6), D)
        m = margin(cand)
        keep = (m >= 0.25) | ((m <= -0.25) & (chome < face))
        cand, chome, ck = cand[keep], chome[keep], ck[keep]
        cout = margin(cand) < 0
        # R^2 of every candidate to every detector, in units of 2^-12 (exact: both on the 1/64 grid)
        diff = np.round((det[None, :, :] - cand[:, None, :]) * 64).astype(np.int64)
        R2 = (diff ** 2).sum(-1)
        r02 = np.round(r0 * 64).astype(np.int64) ** 2
        nonhome = chome[:, None] != np.arange(D)[None, :]
        assert not (isolate and (nonhome & (R2 < r02[None, :])).any())
        if lost:  # tets smaller than every ray that is walked
            assert (R2[nonhome] > (0.125 * 64) ** 2).all()
        shadow = np.zeros(R2.shape, dtype=np.int8)
        if shape == "l":
            shadow = _notch_crossing(np.broadcast_to(cand[:, None, :], R2.shape + (3,)),
                                     np.broadcast_to(det[None, :, :], R2.shape + (3,)), 1e-6)
            ok = (shadow >= 0).all(1)  # drop the candidates with a ray too close to the notch to call
            cand, chome, ck, cout, R2, shadow = cand[ok], chome[ok], ck[ok], cout[ok], R2[ok], shadow[ok]
            assert not shadow[np.arange(len(cand)), chome].any()  # home rays run along one axis: never shadowed
        inside_c = [np.flatnonzero((chome == d) & ~cout) for d in range(D)]
        outside_c = [np.flatnonzero((chome == d) & cout) for d in range(D)]
        if all(len(c) for c in inside_c) and all(len(outside_c[d]) for d in range(face)):
            break
    else:
        raise AssertionError("no detector placement found")
    G = Tp * nbins * D

    def group(g):  # flat group id -> (time bin, score bin, detector)
        return g // (nbins * D), (g // D) % nbins, g % D

    covered = rng.permutation(G)[:int(round(cover * G))] if hot is None else np.array([], dtype=np.int64)
    free = np.setdiff1d(np.arange(G), covered)
    cancel = rng.choice(free, min(n_cancel, len(free)), replace=False) if len(free) and hot is None else []
    kinds = [s for s in specials if T > 0 or s not in ("late", "early")]
    nspec = min(2 * len(kinds), max(0, (n - 9) // 32 + 1)) if kinds else 0
    spec = [kinds[k % len(kinds)] for k in range(nspec)]
    hg = 0 if hot is None else (hot[0] * nbins + hot[1]) * D + hot[2]
    open_g = np.setdiff1d(np.arange(G), cancel)  # the rest stay out of the cancelling pairs' groups
    cancel = np.repeat(np.asarray(cancel, dtype=np.int64), 2)
    og = rng.integers(Tp * nbins, size=n_outside) * D + rng.integers(face, size=n_outside) if n_outside else []
    parts = [  # (groups, kind, sign +-1 or 0 for random, outside)
        (covered, "cover", 1, False), (cancel, "pair", 1, False), (np.zeros(nspec, np.int64), "anchor", 1, False),
        (np.zeros(nspec, np.int64), "spec", 1, False), (np.asarray(og, np.int64), "", 0, True)]
    rest = n - sum(len(p[0]) for p in parts)
    assert rest >= 0, (n, n - rest)
    parts.append((np.full(rest, hg) if hot is not None else rng.choice(open_g, rest), "", 0, False))
    g = np.concatenate([p[0] for p in parts]).astype(np.int64)
    kind = np.concatenate([np.full(len(p[0]), p[1], dtype="<U8") for p in parts])
    kind[kind == "spec"] = spec
    sign = np.concatenate([np.full(len(p[0]), p[2]) if p[2] else rng.choice([-1, 1], len(p[0])) for p in parts])
    outside = np.concatenate([np.full(len(p[0]), p[3]) for p in parts])
    # positions: the anchors and specials at 32 k + 7 and 32 k + 8, the rest in random order
    order = np.full(n, -1, dtype=np.int64)
    anchors, specs = np.flatnonzero(kind == "anchor"), np.flatnonzero(np.isin(kind, spec))
    order[32 * np.arange(nspec) + 7] = anchors
    order[32 * np.arange(nspec) + 8] = specs
    others = np.setdiff1d(np.arange(n), np.concatenate([anchors, specs]))
    order[order < 0] = rng.permutation(others)
    g, sign, kind, outside = (x[order] for x in (g, sign, kind, outside))
    j, b, h = group(g)
    # a random candidate of the home detector, inside (or outside) the mesh; candidates are sorted by home
    pos_id = np.empty(n, dtype=np.int64)
    for o in (False, True):
        ids = np.flatnonzero(cout == o)
        lo_, cnt = np.searchsorted(chome[ids], np.arange(D)), np.bincount(chome[ids], minlength=D)
        e = outside == o
        pos_id[e] = ids[lo_[h[e]] + (rng.random(e.sum()) * cnt[h[e]]).astype(np.int64)]
    w4 = sign * rng.integers(1, 9, n)
    r4 = rng.integers(1, 9, (n, nscores))
    p64 = rng.integers(1, 65, n)
    v = rng.choice([0.5, 1.0, 2.0, 4.0], n)
    frac = rng.choice(np.asarray(fracs), n)
    pairs = np.flatnonzero(kind == "pair")  # the two of a pair share everything but the sign
    for gg in np.unique(g[pairs]):
        ii = pairs[g[pairs] == gg]
        pos_id[ii], r4[ii], p64[ii], v[ii], frac[ii] = pos_id[ii[0]], r4[ii[0]], p64[ii[0]], v[ii[0]], frac[ii[0]]
        w4[ii] = np.abs(w4[ii[0]]) * np.array([1, -1])
    Rh = 2.0 ** ck[pos_id]
    a = step * (j + frac) if arrive is None else arrive(j, frac)
    a[kind == "late"] = step * T
    a[kind == "early"] = -2.0 ** -12
    t = a - Rh / v
    assert np.array_equal(t + Rh / v, a)
    w = w4 / 4.0
    w[kind == "nan"] = np.nan
    bins = b.astype(np.int32)
    bins[kind == "bin"] = nbins
    bins[kind == "bin_neg"] = -1
    neg = np.flatnonzero(kind == "negpdf")
    neg_d = np.array([(hh + 1) % D for hh in h[neg]], dtype=np.int64)
    return dict(
        D=D, n=n, T=T, nbins=nbins, nscores=nscores, shape=shape, L=L, lost=lost, det=det, r0=r0,
        edges=step * np.arange(T + 1, dtype=np.float64) if T > 0 else None, pts=cand[pos_id], w=w, r=r4 / 4.0,
        home=h, pd=p64 / 64.0, neg=(neg, neg_d), bins=bins, times=t, speeds=v, outside=outside, kind=kind,
        pos_id=pos_id, R2=R2, r02=r02, shadow=shadow, w4=w4, r4=r4, p64=p64, hj=j, a=a)


def dense_pdf(case, sel=None):
    idx = np.arange(case["n"]) if sel is None else np.flatnonzero(sel)
    pdf = np.zeros((case["n"], case["D"]))
    pdf[np.arange(case["n"]), case["home"]] = case["pd"]
    pdf[case["neg"][0], case["neg"][1]] = -1.0 / 64
    return pdf[idx]


def expected(case, void=False, sel=None):
    """(want [max(T, 1), nbins, nscores, D], counters as COUNTERS) of the events sel (all if None)."""
    idx = np.arange(case["n"]) if sel is None else np.flatnonzero(sel)
    D, T, nbins, nscores = case["D"], case["T"], case["nbins"], case["nscores"]
    kind, pos, h = case["kind"][idx], case["pos_id"][idx], case["home"][idx]
    out_ev = case["outside"][idx]
    rejected = (kind == "nan") | (kind == "negpdf")
    outside = out_ev & ~rejected & (not void)
    bins = case["bins"][idx]
    live = ~rejected & ~outside & (bins >= 0) & (bins < nbins)
    t, v = case["times"][idx], case["speeds"][idx]
    traced = inside = shadowed = lost = entries = 0
    R2, r02 = case["R2"], case["r02"]
    ins_tab, sh_tab = R2 < r02[None, :], case["shadow"].astype(bool)
    if T == 0:  # every ray of a live event is walked or inside r0: count them per candidate position
        per = np.bincount(pos[live], minlength=len(R2))[:, None]
        per_out = np.bincount(pos[live & out_ev], minlength=len(R2))[:, None]
        inside = int((per * ins_tab).sum())
        if case["lost"]:
            lost = int((per * ~ins_tab).sum())
        elif void:
            traced = int((per * ~ins_tab).sum())
            entries = int((per * (~ins_tab & sh_tab)).sum() + (per_out * ~ins_tab).sum())
        else:
            traced = int((per * (~ins_tab & ~sh_tab)).sum())
            shadowed = int((per * (~ins_tab & sh_tab)).sum())
    if T > 0:  # per detector, from tables over the candidate positions [D, P]
        RT = np.sqrt(R2.T.astype(np.float64) / U)  # the kernel's R: its square is exact, sqrt correctly rounded
        inexT = RT * RT != R2.T / U
        insT, shT = np.ascontiguousarray(ins_tab.T), np.ascontiguousarray(sh_tab.T)
        step = case["edges"][1] - case["edges"][0]
    for d in range(D if T > 0 else 0):
        arr = t + RT[d][pos] / v  # in range iff in [T_0, T_nt); the bin of a ray that scores 0 does not matter
        near = np.abs(arr - step * np.round(arr / step))  # the distance to the nearest edge
        assert not (inexT[d][pos] & live & (near <= 1e-9) & (arr > -0.5 * step) & (arr < (T + 0.5) * step)).any()
        ok = live & (arr >= case["edges"][0]) & (arr < case["edges"][-1])
        ins = insT[d][pos]
        walked = ok & ~ins
        inside += int(np.count_nonzero(ok & ins))
        sh = shT[d][pos]
        if case["lost"]:
            lost += int(np.count_nonzero(walked))
        elif void:
            traced += int(np.count_nonzero(walked))
            entries += int(np.count_nonzero(walked & sh) + np.count_nonzero(walked & out_ev))  # a notch crossing
        else:                                                                                # enters again
            traced += int(np.count_nonzero(walked & ~sh))
            shadowed += int(np.count_nonzero(walked & sh))
    # the home rays carry every nonzero score
    r2h = R2[pos, h]
    ball = r2h < r02[h]
    g4 = np.where(ball, 12 * 4096 // np.maximum(r02[h], 1), 4 * 4096 // r2h)  # 12 / r0^2 or 4 / R^2, times 4
    assert np.array_equal(np.where(ball, 12 * 4096 % np.maximum(r02[h], 1), 4 * 4096 % r2h), np.zeros(len(idx)))
    jh = np.searchsorted(case["edges"], case["a"][idx], side="right") - 1 if T > 0 else np.zeros(len(idx), int)
    scores = live & (jh >= 0) & (jh < max(T, 1)) & (ball | (not case["lost"]))
    val = case["w4"][idx, None] * case["r4"][idx] * case["p64"][idx, None] * g4[:, None]
    acc = np.zeros((max(T, 1), nbins, nscores, D), dtype=np.int64)
    bound = np.zeros_like(acc)
    s = np.flatnonzero(scores)
    for k in range(nscores):
        np.add.at(acc, (jh[s], bins[s], k, h[s]), val[s, k])
        np.add.at(bound, (jh[s], bins[s], k, h[s]), np.abs(val[s, k]))
    assert bound.max(initial=0) < 2 ** 53  # every partial sum, in any order, is exact
    cnt = (traced, shadowed, lost, inside, int(outside.sum()), int(rejected.sum()), entries)
    return acc.astype(np.float64) / U, cnt


def test_exact_case_against_fractions():
    """The generator's expectation equals an independent per-ray sum in exact rationals (CPU only)."""
    case = exact_case(7, D=5, n=300, T=3, nbins=2, nscores=2, n_outside=6)
    D, T = case["D"], case["T"]
    pdf = dense_pdf(case)
    for void in (False, True):
        want, cnt = expected(case, void)
        ref = {}
        traced = inside = outside = rejected = entries = 0
        for i in range(case["n"]):
            x, w, r, b = case["pts"][i], case["w"][i], case["r"][i], int(case["bins"][i])
            if not math.isfinite(w) or (pdf[i] < 0).any():
                rejected += 1
                continue
            out = (np.minimum(x, case["L"] - x) < 0).any()
            if out and not void:
                outside += 1
                continue
            if not 0 <= b < case["nbins"]:
                continue
            for d in range(D):
                R2 = sum(Fraction(float(q)) ** 2 for q in case["det"][d] - x)
                R = math.sqrt(float(R2))
                j = int(np.searchsorted(case["edges"], case["times"][i] + R / case["speeds"][i], side="right")) - 1
                if not 0 <= j < T:
                    continue
                r0 = Fraction(float(case["r0"][d]))
                if R2 < r0 * r0:
                    inside += 1
                    f = Fraction(float(pdf[i, d])) * 3 / (r0 * r0)
                else:
                    traced += 1
                    entries += int(out)
                    f = Fraction(float(pdf[i, d])) / R2
                for k in range(case["nscores"]):
                    key = (j, b, k, d)
                    ref[key] = ref.get(key, Fraction(0)) + Fraction(float(w)) * Fraction(float(r[k])) * f
        got = np.zeros_like(want)
        for key, val in ref.items():
            assert val.denominator <= U  # a multiple of 2^-12
            got[key] = float(val)
        assert np.array_equal(got, want)
        assert cnt == (traced, 0, 0, inside, outside, rejected, entries if void else 0)
        assert (want == 0).any() and (want < 0).any() and (want > 0).any() and rejected and inside and traced
    assert case["kind"].tolist().count("late") and case["kind"].tolist().count("early")
    assert (case["a"] == np.floor(case["a"])).any()  # arrivals on an edge


# ---- running the four calls -----------------------------------------------------------------------------------------
def _mesh(case):
    if case["shape"] == "l":
        return l_shaped_mesh(8, 8, 2)
    if case["lost"]:
        L = case["L"]
        return kuhn_box(*(int(x * 16) for x in L), *L)
    return kuhn_box(*(int(x) for x in case["L"]))


def _engine(case, c, t, nparticles, void, edges=None):
    from pumiumtally_b200.tally import PumiTally

    eng = PumiTally.from_arrays(c, t, nparticles)
    if case["nbins"] > 1:
        eng.set_score_bins(case["nbins"])
    if case["nscores"] > 1:
        eng.set_scores(case["nscores"])
    edges = case["edges"] if edges is None else edges
    if edges is not None:
        eng.set_time_bins(edges)
    eng.set_detector_void(void)
    eng.set_point_detectors(case["det"], case["r0"])
    eng.set_detector_cross_sections(np.zeros((case["nbins"], len(t))))
    return eng


def _to_device(*arrays):
    import torch

    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _run(eng, path, case, sel=None, max_iters=0, pdf=None):
    """One call on the events sel (all if None) after a reset: (results, counters).  max_iters applies to the call
    only, not to the location of the particles; pdf [n, D] (None: exact_case's)."""
    import torch

    idx = np.arange(case["n"]) if sel is None else np.flatnonzero(sel)
    timed = eng.time_bins > 0
    kw = dict(pdf=dense_pdf(case, sel) if pdf is None else pdf[idx], responses=case["r"][idx], bins=case["bins"][idx],
              times=case["times"][idx] if timed else None, speeds=case["speeds"][idx] if timed else None)
    pts, w = case["pts"][idx], case["w"][idx]
    eng.reset_tally()
    if path == "host":
        eng.set_option("chunk", 1024)
        eng.tally_detectors(pts, w, **kw)
    elif path == "device":
        dev = {k: _to_device(a)[0] for k, a in kw.items()}
        eng.tally_detectors_device(*_to_device(pts, w), **dev)
    else:
        el = eng.locate(pts).astype(np.int32)
        assert (el >= 0).all()
        x, el = _to_device(pts, el)
        eng.set_state_device(x.data_ptr(), el.data_ptr(), 0, len(pts))
        torch.cuda.synchronize()
        eng.set_option("max_iters", max_iters)
        flag = np.ones(len(pts), dtype=np.int8)
        if path == "particles":
            eng.set_option("chunk", 1024)
            eng.tally_detectors_at_particles(flag, w, **kw)
        else:
            dev = {k: _to_device(a)[0] for k, a in kw.items()}
            eng.tally_detectors_at_particles_device(*_to_device(flag, w), **dev)
    torch.cuda.synchronize()
    return eng.detector_results(0), tuple(eng.get_option(k) for k in COUNTERS)


PATHS = ("host", "device", "particles", "particles_device")

# (D, T, nbins, nscores, n): slots = max(T, 1) nbins nscores D on both sides of 2048, D and n not multiples of 32
EXACT = {
    "slots1": (1, 0, 1, 1, 33),
    "slots592": (37, 4, 2, 2, 1031),
    "slots2047": (89, 23, 1, 1, 2057),
    "slots2048": (256, 8, 1, 1, 2081),
    "slots2048_2x2": (32, 16, 2, 2, 1057),
    "slots2049": (3, 683, 1, 1, 2089),
    "slots2108": (31, 17, 1, 4, 1001),
    "slots2112": (33, 32, 2, 1, 2113),
    "slots2295": (255, 3, 1, 3, 1283),
    "slots4096": (256, 4, 2, 2, 2593),
    "slots4194304": (256, 1024, 2, 8, 524288 + 37),
}


def _exact(name):
    D, T, nbins, nscores, n = EXACT[name]
    top = name == "slots4194304"
    return exact_case(len(name) + D, D=D, n=n, T=T, nbins=nbins, nscores=nscores, n_outside=0 if D == 1 else 5,
                      cover=1.0 if top else 0.75, n_cancel=0 if top else 8)


@pytest.mark.gpu
@pytest.mark.parametrize("void", [False, True], ids=["void_off", "void_on"])
@pytest.mark.parametrize("name", list(EXACT))
def test_exact_all_four_calls(name, void):
    """Every call equals the int64 reference bit for bit, with exact counters; the particle calls take the events inside
    the box.  With the void off the events outside count once each and score nothing; with it on they are traced and
    each of their traced rays enters the box once."""
    case = _exact(name)
    c, t = _mesh(case)
    inside = ~case["outside"]
    eng = _engine(case, c, t, 16, void)
    eng_p = _engine(case, c, t, int(inside.sum()), void)
    want, cnt = expected(case, void)
    want_p, cnt_p = expected(case, void, inside)
    if name == "slots4194304":
        assert want.size == 4194304 and (want != 0).all()
    assert cnt[5] > 0 or case["D"] == 1
    for path in PATHS:
        located = path in ("host", "device")
        got, got_cnt = _run(eng if located else eng_p, path, case, None if located else inside)
        assert np.array_equal(got, want if located else want_p), path
        assert got_cnt == (cnt if located else cnt_p), path


@pytest.mark.gpu
def test_shared_memory_and_warp_agree_across_the_limit():
    """The same events with 8 time bins (D = 256: 2048 slots, shared memory) and 9 (2304 slots, warp), no home ray
    arriving in bin 8: bins 0-7 equal bit for bit in all four kernels, bin 8 is 0."""
    S = smem_slots()
    case = exact_case(11, D=256, n=3001, T=8, specials=("nan", "negpdf", "bin", "early"), n_outside=5)
    assert 8 * 256 == S
    c, t = _mesh(case)
    inside = ~case["outside"]
    for void in (False, True):
        for path in ("device", "particles_device"):
            sel = None if path == "device" else inside
            want, _ = expected(case, void, sel)
            n = 16 if sel is None else int(inside.sum())
            a, _ = _run(_engine(case, c, t, n, void), path, case, sel)
            b, _ = _run(_engine(case, c, t, n, void, edges=np.arange(10.0)), path, case, sel)
            assert np.array_equal(a, want) and np.array_equal(b[:8], a) and not b[8].any(), (void, path)


@pytest.mark.gpu
@pytest.mark.parametrize("hot", [None, (517, 3, 0)], ids=["one_slot_smem", "one_hot_slot_of_8192"])
def test_contention_on_one_slot(hot):
    """2^20 home rays into one slot: the call's only slot (shared memory), or one of 8192 (warp path)."""
    n = (1 << 20) + 11
    if hot is None:
        case = exact_case(3, D=1, n=n, cover=1.0, n_cancel=0)
    else:
        case = exact_case(4, D=1, n=n, T=1024, nbins=8, hot=hot, specials=())
    c, t = _mesh(case)
    want, cnt = expected(case)
    assert (want != 0).sum() == 1 and cnt[0] + cnt[3] >= (1 << 20)
    for void in (False, True):
        for path in ("device", "particles_device"):
            got, got_cnt = _run(_engine(case, c, t, n, void), path, case)
            assert np.array_equal(got, want) and got_cnt == cnt, (void, path)


@pytest.mark.gpu
def test_shadowed_lanes_in_the_warp_path():
    """L-shaped mesh, 33 detectors, 64 time bins (2112 slots): with the void off the rays whose xy projection runs
    through the notch are shadowed, as the clip predicts; with it on they are traced and enter the mesh again once."""
    case = exact_case(5, D=33, n=2081, T=64, L=(8, 8, 2), shape="l")
    c, t = _mesh(case)
    res = {}
    for void in (False, True):
        want, cnt = expected(case, void)
        for path in PATHS:
            got, got_cnt = _run(_engine(case, c, t, case["n"], void), path, case)
            assert np.array_equal(got, want) and got_cnt == cnt, (void, path)
        res[void] = cnt
    assert res[False][1] > 0 and res[True][6] == res[False][1] and res[True][1] == 0
    assert res[True][0] == res[False][0] + res[False][1]


@pytest.mark.gpu
def test_lost_lanes_in_the_warp_path():
    """max_iters = 1 on a mesh whose tets are smaller than every ray: every walked ray is lost and scores 0, only the
    rays inside r0 score; 3 detectors, 683 time bins (2049 slots).  The particle calls only: the located calls find
    their events under the same limit."""
    case = exact_case(6, D=3, n=2501, T=683, L=(3.0, 3.0, 3.0), ks=(-2, -1), r0s=(0.5, 1.0), lost=True)
    c, t = _mesh(case)
    for void in (False, True):
        want, cnt = expected(case, void)
        assert cnt[2] > 0 and cnt[3] > 0 and cnt[0] == 0 and want.any()
        for path in ("particles", "particles_device"):
            got, got_cnt = _run(_engine(case, c, t, case["n"], void), path, case, max_iters=1)
            assert got_cnt == cnt, (void, path)
            assert np.array_equal(got, want), (void, path)


# ---- which kernel ran -----------------------------------------------------------------------------------------------
def print_kernel_choice():
    """For kDetSmemSlots and one more slot (score bins), the detector kernels each of the four calls launched."""
    S = smem_slots()
    out = {}
    for slots in (S, S + 1):
        case = exact_case(1, D=1, n=40, nbins=slots, specials=(), cover=0.0, n_cancel=0)
        c, t = _mesh(case)
        for void in (False, True):
            for path in ("device", "particles_device"):
                eng = _engine(case, c, t, case["n"], void)
                _run(eng, path, case)  # loads the module
                names = kernels_launched(lambda: _run(eng, path, case), "detect_")
                out[f"{path} {int(void)} {slots}"] = names
    print(json.dumps(out))


@pytest.mark.gpu
def test_each_instantiation_runs_at_its_slot_count():
    """kDetSmemSlots slots launch the shared-memory kernel, one more the warp one: each of the eight exactly once."""
    S = smem_slots()
    got = run_in_fresh_process("test_gpu_detector_slots", "print_kernel_choice")
    for path, fam in (("device", "detect_located"), ("particles_device", "detect_particles")):
        for void in (0, 1):
            for slots, smem in ((S, "true"), (S + 1, "false")):
                names = got[f"{path} {void} {slots}"]
                want = f"{fam}{'_void' if void else ''}_kernel<{smem}>"
                assert len(names) == 1 and want in names[0], (path, void, slots, names)


# ---- general data past kDetSmemSlots ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mesh", ["kuhn", "void"])
def test_general_data_past_the_limit_match_the_reference(mesh):
    """test_gpu_detectors' comparison at D = 65, 4 time bins, 2 score bins, 4 scores (2080 slots: the warp path), with
    random per-element Sigma."""
    from pumiumtally_b200.tally import PumiTally

    c, t = MESHES[mesh]()
    D, nbins, nscores = 65, 2, 4
    assert 4 * nbins * nscores * D > smem_slots()
    rng = np.random.default_rng(len(mesh) + 65)
    pts, _ = generic_points(mesh, c, t, 90, rng)
    det, _ = generic_points(mesh, c, t, D, rng)
    n = len(pts)
    edges = np.array([0.0, 0.5, 1.0, 2.0, 5.0])
    sigma = rng.uniform(0.05, 1.0, size=(nbins, len(t)))
    r0 = rng.uniform(0.0, 0.8, D)
    w = rng.uniform(0.5, 2.0, n)
    pdf = rng.uniform(0.0, 0.3, size=(n, D))
    r = rng.uniform(0.2, 2.0, size=(n, nscores))
    bins = rng.integers(0, nbins + 1, n).astype(np.int32)
    times = rng.uniform(0.0, 1.5, n)
    speeds = rng.uniform(1.0, 4.0, n)
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_score_bins(nbins)
    eng.set_scores(nscores)
    eng.set_time_bins(edges)
    eng.set_point_detectors(det, r0)
    eng.set_detector_cross_sections(sigma)
    want, wcnt = reference_detectors(c, t, eng.locate(pts), pts, w, pdf, r, bins, times, speeds, edges, nbins, nscores,
                                     sigma, det, r0)
    case = dict(n=n, pts=pts, w=w, r=r, bins=bins, times=times, speeds=speeds)
    for path in PATHS:
        got, cnt = _run(eng, path, case, pdf=pdf)
        np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-14 * np.abs(want).max())
        assert cnt[:4] + cnt[4:6] == wcnt[:4] + wcnt[5:], path
    assert wcnt[0] > 0 and wcnt[3] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mesh", ["l_shape", "void", "comb"])
def test_general_void_data_past_the_limit_match_the_reference(mesh):
    """test_gpu_detector_void's comparison at D = 65, 4 time bins, 2 score bins, 4 scores (2080 slots)."""
    from pumiumtally_b200.tally import PumiTally
    from test_host_emul_detector_void import cavity_points, outside_points

    c, t = {"l_shape": MESHES["l_shape"], "void": MESHES["void"], "comb": comb_mesh}[mesh]()
    D, nbins, nscores = 65, 2, 4
    rng = np.random.default_rng(3 * len(mesh) + 65)
    ni = 50
    pts = np.concatenate([generic_points(mesh, c, t, ni, rng)[0], cavity_points(mesh, c, rng, ni // 4),
                          outside_points(c, rng, ni // 4, far=3.0)])
    det = np.concatenate([generic_points(mesh, c, t, D // 3, rng)[0], cavity_points(mesh, c, rng, D // 3),
                          outside_points(c, rng, D, far=50.0)])[:D]
    n = len(pts)
    edges = np.array([0.0, 0.5, 1.0, 2.0, 80.0])
    sigma = rng.uniform(0.05, 1.0, size=(nbins, len(t)))
    r0 = rng.uniform(0.0, 0.8, D)
    w = rng.uniform(0.5, 2.0, n)
    pdf = rng.uniform(0.0, 0.3, size=(n, D))
    r = rng.uniform(0.2, 2.0, size=(n, nscores))
    bins = rng.integers(0, nbins + 1, n).astype(np.int32)
    times = rng.uniform(0.0, 1.5, n)
    speeds = rng.uniform(1.0, 4.0, n)

    def engine(np_):
        e = PumiTally.from_arrays(c, t, np_)
        e.set_score_bins(nbins)
        e.set_scores(nscores)
        e.set_time_bins(edges)
        e.set_detector_void(True)
        e.set_point_detectors(det, r0)
        e.set_detector_cross_sections(sigma)
        return e

    eng = engine(n)
    elem = eng.locate(pts)
    inn = elem >= 0
    eng_p = engine(int(inn.sum()))
    case = dict(n=n, pts=pts, w=w, r=r, bins=bins, times=times, speeds=speeds)
    for path in PATHS:
        located = path in ("host", "device")
        sel = None if located else inn
        s = slice(None) if located else inn
        want, wcnt = reference_void(c, t, elem[s], pts[s], w[s], pdf[s], r[s], bins[s], times[s], speeds[s], edges,
                                    nbins, nscores, sigma, det, r0)
        got, cnt = _run(eng if located else eng_p, path, case, sel, pdf=pdf)
        np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-14 * np.abs(want).max())
        assert cnt[:4] + cnt[4:6] == wcnt[:4] + wcnt[5:], path
        assert cnt[6] > 0 or not located
    assert wcnt[0] > 0 and wcnt[3] > 0


# ---- the per-launch split and the int64 ray index ---------------------------------------------------------------------
@pytest.mark.gpu
def test_located_call_split_into_two_launches_is_exact():
    """D = 256 and 2^22 + 37 events: the located call makes two launches of at most 2^30 rays, the second with every
    input offset: positions, weights, pdf (by D rows), responses (by 2 per event), score bins, times and speeds, all of
    which vary between events (2 time bins, 2 score bins, 2 scores: 2048 slots, shared memory).  Bit for bit with the
    int64 reference, every ray traced: the edges are 0, 128 and 256, every arrival lies inside [0, 256), and every home
    arrival within 0.5 of 128, so that another event's time or speed moves many across that edge."""
    import torch

    D, n = 256, (1 << 22) + 37
    case = exact_case(9, D=D, n=n, T=2, nbins=2, nscores=2, L=(10, 10, 10), r0s=(0.125,), specials=(), cover=1.0,
                      n_cancel=0, isolate=True, step=128.0, fracs=(0.0, 0.25),
                      arrive=lambda j, f: 128.0 + np.where(j == 0, -0.25 - f, f))
    assert 2 * 2 * 2 * D <= smem_slots()
    c, t = _mesh(case)
    want, cnt = expected(case)
    assert cnt == (n * D, 0, 0, 0, 0, 0, 0)
    tail = slice((1 << 22) - 37, None)  # the first launch's last events and the second's: all of them vary
    for x in (case["bins"], case["times"], case["speeds"], case["r"][:, 1]):
        assert len(np.unique(x[tail])) > 1
    eng = _engine(case, c, t, 16, False)
    pdf = torch.zeros((n, D), dtype=torch.float64, device="cuda")
    pdf[torch.arange(n, device="cuda"), torch.from_numpy(case["home"]).cuda()] = torch.from_numpy(case["pd"]).cuda()
    pts, w, r, bins, times, speeds = _to_device(case["pts"], case["w"], case["r"], case["bins"], case["times"],
                                                case["speeds"])
    eng.reset_tally()
    eng.tally_detectors_device(pts, w, pdf=pdf, responses=r, bins=bins, times=times, speeds=speeds)
    torch.cuda.synchronize()
    del pdf
    torch.cuda.empty_cache()
    assert np.array_equal(eng.detector_results(0), want)
    assert tuple(eng.get_option(k) for k in COUNTERS) == cnt


@pytest.mark.gpu
def test_particle_call_past_two_to_the_31_rays():
    """D = 256 at 8.4 M particles (2.15e9 rays, q past 2^31), Sigma = 0, no pdf: the four ray counters exactly, and each
    detector within the rigorous bound of a float64 sum of w / (4 pi R^2), which the smallest single ray exceeds."""
    import torch

    from pumiumtally_b200.tally import PumiTally

    D, n = 256, 8_400_000
    assert n * D > 2 ** 31
    c, t = kuhn_box(8, 8, 8)
    rng = np.random.default_rng(12)
    det = rng.uniform(3.0, 5.0, size=(D, 3))
    r0 = np.full(D, 0.125)
    eng = PumiTally.from_arrays(c, t, n)
    eng.set_point_detectors(det, r0)
    eng.set_detector_cross_sections(np.zeros((1, len(t))))
    g = torch.Generator(device="cuda").manual_seed(5)
    pts = (torch.rand((n, 3), dtype=torch.float64, device="cuda", generator=g) * 7.9 + 0.05).contiguous()
    w = 1.0 + torch.rand(n, dtype=torch.float64, device="cuda", generator=g)
    el = eng.locate_device(pts)
    eng.set_state_device(pts.data_ptr(), el.data_ptr(), 0, n)
    torch.cuda.synchronize()
    eng.tally_detectors_at_particles_device(torch.ones(n, dtype=torch.int8, device="cuda"), w)
    torch.cuda.synchronize()
    got = eng.detector_results(0)[0, 0, 0]
    cnt = tuple(eng.get_option(k) for k in COUNTERS)
    u = 2.0 ** -53
    inside = 0
    for d in range(D):
        R = (torch.tensor(det[d], device="cuda") - pts).norm(dim=1)
        assert float((R - r0[d]).abs().min()) > 1e-12
        ins = R < r0[d]
        inside += int(ins.sum())
        v = torch.where(ins, w * (0.25 / math.pi) * 3.0 / (r0[d] * r0[d]), w * (0.25 / math.pi) / (R * R))
        total = float(v.sum())
        tol = 2 * (n + 8) * u * total
        assert float(v.min()) > tol
        assert abs(got[d] - total) <= tol, (d, got[d], total, tol)
    assert cnt[:6] == (n * D - inside, 0, 0, inside, 0, 0) and inside > 0
