"""Lane refill in the persistent walk kernels (8, 16 and 24): a lane that finishes a track takes the next particle of
its warp's stage at once, so its score slots, time slots and time bin, and the stage, ticket or packed row it reads
from, carry over from one track to the next.  At the particle counts of the feature tests most lanes walk a single
track; here every launch holds at least REFILLS times as many flying particles as the GPU has resident lanes, so by
pigeonhole most lanes walk several.  Scored, timed and moment moves must then give, element by element, what the
thread-per-particle kernel (0, no lane state) gives, what the per-particle oracle gives on the cut flights, and the
closed-form totals of every score and time bin."""
import types

import numpy as np
import pytest

from helpers import assert_flux_close
from oracle.oracle import OraclePumiTally
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.workload import SyntheticWorkload
from test_gpu_moments import _configure, _move
from test_gpu_scores import assert_same_particles, assert_scores_equal, engine, responses
from time_bins_ref import time_pieces, time_workload

pytestmark = pytest.mark.gpu

CELLS = (30, 30, 30)  # 162,000 tets, a 20.7 MB tet table: below twice the L2 of an H100, where kernels 8 and 24 run
N = 2_200_000  # more than one stage of a host move (2 Mi particles for the binned and sorted kernels)
LANES = 128  # threads per block of every persistent kernel
REFILLS = 4  # flying particles per resident lane in every launch, at least
PERSISTENT = (8, 16, 24)
TOTAL_RTOL = 1e-10  # closed-form totals, relative to the sum of the absolute contributions

# (a) scored, 5 scores (stride 8) x 3 score bins; (b) timed, the maximum 8 scores x 16 time bins with moments;
# (c) timed, 1 score x the maximum 1024 time bins, log-spaced; (d) the plain move with moments (no responses array)
CONFIGS = {
    "scored": dict(nscores=5, nbins=3, edges=None, moments=0),
    "timed_moments": dict(nscores=8, nbins=1, edges=np.linspace(0.0, 4.0, 17), moments=1),
    "fine_time_bins": dict(nscores=1, nbins=1, edges=np.geomspace(1e-3, 1e3, 1025), moments=0),
    "plain_moments": dict(nscores=1, nbins=1, edges=None, moments=1),
}
KERNELS = [(0, None), (8, None), (16, 1), (16, 2), (16, 4), (24, None)]
KERNEL_IDS = ["v0", "v8", "v16-run1", "v16-run2", "v16-run4", "v24"]


def _kind(cfg):
    if cfg["edges"] is not None:
        return "timed"
    return "scored" if cfg["nscores"] > 1 or cfg["nbins"] > 1 else "plain"


def _score_bins(rng, n, nbins):
    """Bins in [0, nbins), 5 % of them outside: those particles fly unscored."""
    b = rng.integers(0, nbins, n)
    out = rng.random(n) < 0.05
    b[out] = rng.choice([-1, nbins, 1 << 30], int(out.sum()))
    return b.astype(np.int32)


def _log_times(rng, o, d, edges):
    """Times and speeds for log-spaced edges: starts uniform in log time from before T_0 to after T_n, a few at
    negative times, and durations of 0.2 to 6 times the start time, so that a typical flight spans tens to hundreds
    of bins."""
    n = len(o)
    t = np.exp(rng.uniform(np.log(edges[0]) - 1.0, np.log(edges[-1]) + 0.3, n))
    duration = t * np.exp(rng.uniform(np.log(0.2), np.log(6.0), n))
    t[rng.random(n) < 0.02] *= -1.0
    length = np.maximum(np.linalg.norm(np.asarray(d).reshape(-1, 3) - np.asarray(o).reshape(-1, 3), axis=1), 1e-3)
    return t, length / duration


def _times(rng, cfg, o, d):
    if cfg["edges"][0] > 0.0:
        return _log_times(rng, o, d, cfg["edges"])
    return time_workload(rng, o, d, float(CELLS[0]), cfg["edges"])


def _wr(cfg, x):
    """w * r[:, k] of every particle and score; r is 1 without a responses array."""
    return x["w"][:, None] * (x["r"] if "r" in x else np.ones((len(x["w"]), cfg["nscores"])))


def _bad(cfg, x):
    """Flying tracks the walk must refuse and count as lost: non-finite weight * response, time or speed, speed <= 0."""
    with np.errstate(invalid="ignore"):
        bad = ~np.isfinite(x["d"]).all(axis=1) | ~np.isfinite(_wr(cfg, x)).all(axis=1)
        if cfg["edges"] is not None:
            bad |= ~np.isfinite(x["t"]) | ~np.isfinite(x["v"]) | ~(x["v"] > 0.0)
    return (x["f"] == 1) & bad


def _launch_counts(cfg, x):
    """Flying particles in each reported launch of a device move: one launch over all of them, or one per score bin.
    A binned move makes one more launch for the particles whose bin is outside [0, nbins): a few per cent of them,
    flying unscored into an array that is never reported, so it is left out."""
    fly = x["f"] == 1
    if "b" in x:
        return [int((fly & (x["b"] == b)).sum()) for b in range(cfg["nbins"])]
    return [int(fly.sum())]


def _run(work, cfg, moves, variant, claim_run=None, states=None, refill=True, label=""):
    """An engine on `variant` after CopyInitialPosition and the device-pointer moves `moves`.  states: the particles
    a plain engine holds after each move.  refill: assert that every launch of a persistent kernel holds at least
    REFILLS flying particles per resident lane."""
    import torch

    eng = engine(work.coords, work.t2v, N, variant, **({"claim_run": claim_run} if claim_run else {}))
    _configure(eng, cfg["nscores"], cfg["edges"], cfg["moments"], cfg["nbins"])
    eng.CopyInitialPosition(work.init.reshape(-1).copy())
    s = torch.cuda.current_stream().cuda_stream
    for m, x in enumerate(moves):
        launches = eng.get_option("launches")
        dev = {k: torch.from_numpy(np.ascontiguousarray(a)).cuda() for k, a in x.items()}
        ptr = {k: t.data_ptr() for k, t in dev.items()}
        base = (ptr["o"], ptr["d"], ptr["f"], ptr["w"])
        kind = _kind(cfg)
        if kind == "timed":
            eng.move_device_timed(*base, ptr["t"], ptr["v"], ptr.get("r"), ptr.get("b"), s)
        elif kind == "scored":
            eng.move_device_scored(*base, ptr["r"], ptr.get("b"), s)
        else:
            eng.move_device(*base, s)
        torch.cuda.synchronize()
        del dev
        if refill and variant in PERSISTENT:
            # walk_blocks_per_sm is the occupancy of the last persistent launch in the process: it describes this move
            # only if this move ran the requested persistent kernel, once per pass (and per score bin)
            passes = cfg["nbins"] + 1 if "b" in x else 1
            assert eng.get_option("variant") == variant, (label, eng.get_option("variant"))
            assert eng.get_option("launches") - launches >= passes, (label, "no walk launch in this move")
            occ = eng.get_option("walk_blocks_per_sm")
            resident = work.sms * occ * LANES
            least = min(_launch_counts(cfg, x))
            print(f"{label} move {m}: walk_blocks_per_sm {occ}, {resident} resident lanes, fewest flying particles in "
                  f"a reported launch {least}")
            assert occ > 0 and least >= REFILLS * resident, (
                f"{label} move {m}: kernel {variant} runs {occ} blocks of {LANES} lanes per SM on {work.sms} SMs "
                f"({resident} lanes); its fewest flying particles in one reported launch, {least}, are fewer than "
                f"{REFILLS} per lane (the unscored pass of the bins outside [0, nbins) is not counted)")
        if states is not None:
            np.testing.assert_array_equal(eng.elem_ids, states[m + 1][1], err_msg=f"{label} move {m}")
            np.testing.assert_array_equal(eng.positions, states[m + 1][0], err_msg=f"{label} move {m}")
    return eng


def _results(eng, cfg):
    """Every reported array: m0 [time][bin][score][element] and, with moments, m1 [...][element][3]."""
    return eng.flux_time, (eng.flux_moments() if cfg["moments"] else None)


def _assert_results_equal(got, want, label):
    for idx in np.ndindex(*want[0].shape[:3]):
        assert_scores_equal(got[0][idx], want[0][idx], f"{label} m0 {idx}")
        if want[1] is not None:
            assert_scores_equal(got[1][idx], want[1][idx], f"{label} m1 {idx}")


def piece_sums(start, end, alive, wr, times=None, speeds=None, edges=None, centre=None, block=1 << 15):
    """Closed-form totals per time bin and score of the flights start -> end (already clipped): m0[j, k] = sum of
    wr[:, k] * (length of the piece in bin j), and with a centre C, m1[j, k] = sum of wr[:, k] * length * (piece
    midpoint - C); a0 and a1 are the same sums of absolute values, the scale of their rounding.  The pieces are those
    of time_bins_ref.time_pieces; without edges the one bin holds whole flights."""
    start, end = np.asarray(start).reshape(-1, 3), np.asarray(end).reshape(-1, 3)
    length = np.linalg.norm(end - start, axis=1)
    nt, ns = (1 if edges is None else len(edges) - 1), wr.shape[1]
    m0, a0, m1, a1 = np.zeros((nt, ns)), np.zeros((nt, ns)), np.zeros((nt, ns, 3)), np.zeros((nt, ns, 3))
    ok = alive & (length > 0)
    for lo in range(0, len(start), block):
        i = lo + np.nonzero(ok[lo:lo + block])[0]
        if edges is None:
            p, j, s_lo, s_hi = i, np.zeros(len(i), dtype=np.int64), np.zeros(len(i)), length[i]
        else:  # one piece per bin from the start's bin to the end's, clipped to [T_0, T_n)
            t1 = times[i] + length[i] / speeds[i]
            first = np.clip(np.searchsorted(edges, times[i], "right") - 1, 0, nt - 1)
            cnt = np.clip(np.searchsorted(edges, t1, "right") - 1, 0, nt - 1) - first + 1
            q = np.repeat(np.arange(len(i)), cnt)
            j = first[q] + np.arange(len(q)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
            p = i[q]
            s_lo = np.clip((edges[j] - times[p]) * speeds[p], 0.0, length[p])
            s_hi = np.clip((edges[j + 1] - times[p]) * speeds[p], 0.0, length[p])
        ell = s_hi - s_lo
        keep = ell > 0
        p, j, s_lo, ell = p[keep], j[keep], s_lo[keep], ell[keep]
        if centre is not None:
            rel = start[p] + ((s_lo + 0.5 * ell) / length[p])[:, None] * (end[p] - start[p]) - centre
        for k in range(ns):
            x = wr[p, k] * ell
            m0[:, k] += np.bincount(j, x, nt)
            a0[:, k] += np.bincount(j, np.abs(x), nt)
            if centre is not None:
                for c in range(3):
                    m1[:, k, c] += np.bincount(j, x * rel[:, c], nt)
                    a1[:, k, c] += np.bincount(j, np.abs(x * rel[:, c]), nt)
    return m0, a0, m1, a1


def _oracle_indices(name, cfg):
    """The (time bin, score bin, score) arrays checked against the oracle."""
    if name == "timed_moments":
        return [(j, 0, k) for j in range(len(cfg["edges"]) - 1) for k in (0, cfg["nscores"] - 1)]
    if name == "fine_time_bins":
        picks = np.random.default_rng(3).choice(len(cfg["edges"]) - 1, 8, replace=False)
        return [(int(j), 0, 0) for j in sorted(picks)]
    return [(0, b, k) for b in range(cfg["nbins"]) for k in range(cfg["nscores"])]


def reference(work, name, cfg, moves, starts, ends):
    """The oracle's m0 of the checked arrays and the closed-form totals of every array, for the moves `moves` that
    start from the particles `starts` (positions, elements) and end at the positions `ends`.  The oracle walks each
    move's flights of one score bin, or their pieces in one time bin, with weights w * r[:, k]."""
    orc, edges = work.oracle, cfg["edges"]
    alive = [(x["f"] == 1) & ~_bad(cfg, x) for x in moves]
    oracle = {}
    for idx in _oracle_indices(name, cfg):
        j, b, k = idx
        orc.reset_flux()
        for x, ok, (xyz, elem), end in zip(moves, alive, starts, ends):
            sel = ok & (x["b"] == b) if "b" in x else ok
            if edges is None:
                o, d, fly = x["o"], x["d"], sel
            else:
                a, e, ids = time_pieces(x["o"], end, x["t"], x["v"], edges[j:j + 2], sel)[0]
                o, d, fly = xyz.copy(), xyz.copy(), np.zeros(N, dtype=bool)
                o[ids], d[ids], fly[ids] = a, e, True
            wk = np.where(fly, _wr(cfg, x)[:, k], 0.0)
            if fly.any():
                orc.set_state(xyz, elem)
                orc.MoveToNextLocation(o.reshape(-1).copy(), d.reshape(-1).copy(), fly.astype(np.int8), wk)
        oracle[idx] = orc.flux
    nt = 1 if edges is None else len(edges) - 1
    shape = (nt, cfg["nbins"], cfg["nscores"])
    m0, a0, m1, a1 = np.zeros(shape), np.zeros(shape), np.zeros(shape + (3,)), np.zeros(shape + (3,))
    for x, ok, end in zip(moves, alive, ends):
        wr = np.where(ok[:, None], _wr(cfg, x), 0.0)
        for b in range(cfg["nbins"]):
            sel = ok & (x["b"] == b) if "b" in x else ok
            s = piece_sums(x["o"], end, sel, wr, x.get("t"), x.get("v"), edges, work.C0 if cfg["moments"] else None)
            m0[:, b] += s[0]
            a0[:, b] += s[1]
            m1[:, b] += s[2]
            a1[:, b] += s[3]
    assert (a0 > 0).all(), "every time bin, score bin and score has pieces"
    return types.SimpleNamespace(oracle=oracle, m0=m0, a0=a0, m1=m1, a1=a1)


def _assert_reference(res, ref, work, label):
    m0, m1 = res
    for idx, want in ref.oracle.items():
        assert_flux_close(m0[idx], want, f"{label} oracle {idx}")
    err = np.abs(m0.sum(axis=-1) - ref.m0)
    assert (err <= TOTAL_RTOL * ref.a0).all(), f"{label}: m0 totals off at {np.argwhere(err > TOTAL_RTOL * ref.a0)[:5]}"
    if m1 is not None:  # the centred first moment: sum_e (m1_e + (c_e - C) m0_e)
        got = m1.sum(axis=-2) + np.einsum("ec,tbse->tbsc", work.cen - work.C0, m0)
        err = np.abs(got - ref.m1)
        assert (err <= TOTAL_RTOL * ref.a1).all(), f"{label}: m1 totals off at {np.argwhere(err > TOTAL_RTOL * ref.a1)[:5]}"


@pytest.fixture(scope="module")
def work():
    """The mesh, two moves of the synthetic workload (the second re-sources the particles that left the box), the
    particles a plain engine holds before and after each move, and one oracle."""
    import torch

    coords, t2v = kuhn_box(*CELLS)
    wl = SyntheticWorkload(box=tuple(float(c) for c in CELLS), num_particles=N, mean_length=3.0, mu_min=-1.0)
    init = wl.initial_positions()
    moves = [wl.next_step() for _ in range(2)]
    plain = engine(coords, t2v, N)
    plain.CopyInitialPosition(init.reshape(-1).copy())
    states = [(plain.positions, plain.elem_ids)]
    for o, d, f, w in moves:
        _move(plain, "plain", o, d, f, w)
        states.append((plain.positions, plain.elem_ids))
    o2, f2 = moves[1][0], moves[1][2]
    assert ((f2 == 1) & (o2 != states[1][0]).any(axis=1)).mean() > 0.05, "the second move re-sources particles"
    stats = plain.stats()
    plain.close()
    cen = coords[t2v].mean(axis=1)
    C0 = 0.5 * (coords.min(axis=0) + coords.max(axis=0))
    return types.SimpleNamespace(coords=coords, t2v=t2v, init=init, moves=moves, states=states, stats=stats,
                                 oracle=OraclePumiTally(coords, t2v, N), cen=cen, C0=C0,
                                 sms=torch.cuda.get_device_properties(0).multi_processor_count)


@pytest.fixture(scope="module", params=list(CONFIGS))
def case(request, work):
    """One configuration: its side arrays for the two moves; its references and its kernel-0 results once needed."""
    name = request.param
    cfg = CONFIGS[name]
    rng = np.random.default_rng(list(CONFIGS).index(name))
    moves = []
    for o, d, f, w in work.moves:
        x = dict(o=o, d=d, f=f, w=w)
        if cfg["nscores"] > 1:
            x["r"] = responses(rng, N, cfg["nscores"])
        if cfg["nbins"] > 1:
            x["b"] = _score_bins(rng, N, cfg["nbins"])
        if cfg["edges"] is not None:
            x["t"], x["v"] = _times(rng, cfg, o, d)
        moves.append(x)
    return types.SimpleNamespace(name=name, cfg=cfg, moves=moves, ref=None, v0=None)


@pytest.mark.parametrize("variant,claim_run", KERNELS, ids=KERNEL_IDS)
def test_moves_at_refill_scale(work, case, variant, claim_run):
    name, cfg = case.name, case.cfg
    label = f"{name} kernel {variant}" + (f" claim_run {claim_run}" if claim_run else "")
    if case.ref is None:  # the oracle runs once per configuration
        case.ref = reference(work, name, cfg, case.moves, work.states[:2], [st[0] for st in work.states[1:]])
    eng = _run(work, cfg, case.moves, variant, claim_run, states=work.states, label=label)
    st = eng.stats()
    for k in ("segments", "tracks", "lost"):
        assert st[k] == work.stats[k], (label, k, st[k], work.stats[k])
    res = _results(eng, cfg)
    eng.close()
    _assert_reference(res, case.ref, work, label)
    if variant == 0:
        case.v0 = res
    else:
        if case.v0 is None:
            v0 = _run(work, cfg, case.moves, 0, states=work.states, label=f"{name} kernel 0")
            case.v0 = _results(v0, cfg)
            v0.close()
        _assert_results_equal(res, case.v0, f"{label} against kernel 0")
    if name == "fine_time_bins":
        _assert_bins_conserve(work, cfg, case.moves, variant, claim_run, label)


def _assert_bins_conserve(work, cfg, moves, variant, claim_run, label):
    """The time bins of the flights that lie wholly inside [T_0, T_n) sum to those flights' plain tally."""
    edges = cfg["edges"]
    inside = []
    for x, end in zip(moves, (st[0] for st in work.states[1:])):
        length = np.linalg.norm(end - x["o"], axis=1)
        with np.errstate(invalid="ignore"):
            t1 = x["t"] + length / x["v"]
        inside.append(dict(x, f=((x["f"] == 1) & (x["t"] >= edges[0]) & (t1 <= edges[-1])).astype(np.int8)))
    assert 0.05 < np.mean([x["f"].mean() for x in inside]) < 0.9
    part = _run(work, cfg, inside, variant, claim_run, refill=False, label=f"{label} inside")
    summed = part.flux_time[:, 0, 0].sum(axis=0)
    part.close()
    plain = dict(nscores=1, nbins=1, edges=None, moments=0)
    whole = _run(work, plain, inside, -1, refill=False, label=f"{label} plain")
    assert_flux_close(summed, whole.flux, f"{label} conservation")
    whole.close()


def _lane_mix(work, cfg, seed):
    """One move from the initial positions, every 16-particle chunk (rotated from chunk to chunk) one of each:
    0 not flying, 1 flying flag 2, 2 NaN weight, 3 NaN time, 4 speed 0, 5 time at or after the last edge, 6 time
    before T_0 with the flight crossing T_0, 7 zero-length flight, 8 re-sourced origin, 9 negative responses,
    10 score bin outside [0, nbins), 11 a long flight spanning many bins, 12-15 ordinary flights.  Kernel 8 hands
    out the particles in storage order, so every lane's later tracks follow one of these."""
    rng = np.random.default_rng(seed)
    n = N
    role = (np.arange(n) + 5 * (np.arange(n) // 16)) % 16
    o = work.init.reshape(-1, 3).copy()
    re = role == 8
    o[re] = rng.uniform(0.05, 0.95, (int(re.sum()), 3)) * np.array(CELLS, dtype=float)
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    length = rng.exponential(3.0, n)
    length[role == 11] = rng.uniform(20.0, 50.0, int((role == 11).sum()))
    d = o + length[:, None] * u
    d[role == 7] = o[role == 7]
    f = np.ones(n, dtype=np.int8)
    f[role == 0], f[role == 1] = 0, 2
    w = rng.uniform(0.5, 1.0, n)
    w[role == 2] = np.nan
    x = dict(o=o, d=d, f=f, w=w)
    if cfg["nscores"] > 1:
        r = responses(rng, n, cfg["nscores"])
        r[role == 9] = -rng.uniform(0.1, 2.0, (int((role == 9).sum()), cfg["nscores"]))
        x["r"] = r
    if cfg["nbins"] > 1:
        b = rng.integers(0, cfg["nbins"], n).astype(np.int32)
        b[role == 10] = rng.choice([-1, cfg["nbins"], 1 << 30], int((role == 10).sum()))
        x["b"] = b
    edges = cfg["edges"]
    if edges is not None:
        t, v = _times(rng, cfg, o, d)
        nt = len(edges) - 1
        t[role == 3] = np.nan
        v[role == 4] = 0.0
        late = np.nonzero(role == 5)[0]
        t[late[::2]] = edges[-1]
        t[late[1::2]] = edges[-1] + rng.uniform(0.0, 1.0, len(late[1::2])) * (edges[-1] - edges[0])
        early = role == 6  # starts before T_0 and reaches it after 5 % to 50 % of its (unclipped) duration
        t[early] = edges[0] - rng.uniform(0.05, 0.5, int(early.sum())) * length[early] / v[early]
        lng = np.nonzero(role == 11)[0]  # from an edge in the first tenth of the bins to one in the last tenth
        t0 = edges[rng.integers(0, max(nt // 10, 1), len(lng))]
        t[lng] = t0
        v[lng] = length[lng] / (edges[rng.integers(nt - max(nt // 10, 1), nt, len(lng)) + 1] - t0)
        x["t"], x["v"] = t, v
    return x


def test_adversarial_lane_order(work, case):
    """Kernel 8 on the lane mix of _lane_mix: every result against the oracle and kernel 0, the lost tracks counted
    exactly, every track without a piece adding exactly nothing, and the staged host path (in stages and in one) the
    same as the device move."""
    name, cfg = case.name, case.cfg
    x = _lane_mix(work, cfg, 100 + list(CONFIGS).index(name))
    label = f"{name} lane mix"
    v0 = _run(work, cfg, [x], 0, label=f"{label} kernel 0")
    v8 = _run(work, cfg, [x], 8, label=f"{label} kernel 8")
    assert_same_particles(v8, v0, label)
    bad = _bad(cfg, x)
    assert v8.stats()["lost"] == int(bad.sum()) > 0
    end = v8.positions
    np.testing.assert_array_equal(end[bad], x["o"][bad])  # relocated to the origin, no further
    r0, r8 = _results(v0, cfg), _results(v8, cfg)
    v0.close()
    ref = reference(work, name, cfg, [x], work.states[:1], [end])
    _assert_reference(r8, ref, work, f"{label} kernel 8")
    _assert_reference(r0, ref, work, f"{label} kernel 0")
    _assert_results_equal(r8, r0, f"{label} kernel 8 against kernel 0")
    del r0
    # a second engine fed only the tracks that have a piece to tally
    length = np.linalg.norm(end - x["o"], axis=1)
    piece = (x["f"] == 1) & ~bad & (length > 0)
    if "b" in x:
        piece &= (x["b"] >= 0) & (x["b"] < cfg["nbins"])
    if cfg["edges"] is not None:
        with np.errstate(invalid="ignore"):
            piece &= np.maximum(x["t"], cfg["edges"][0]) < np.minimum(x["t"] + length / x["v"], cfg["edges"][-1])
    assert 0.3 < piece.mean() < 0.95
    good = _run(work, cfg, [dict(x, f=piece.astype(np.int8))], 8, refill=False, label=f"{label} good tracks")
    _assert_results_equal(_results(good, cfg), r8, f"{label}: the tracks without a piece")
    good.close()
    # the staged host path: in stages of the default size, and in one stage
    for chunk in (None, -(-N // 1024) * 1024):
        host = engine(work.coords, work.t2v, N, 8, **({"chunk": chunk} if chunk else {}))
        _configure(host, cfg["nscores"], cfg["edges"], cfg["moments"], cfg["nbins"])
        host.CopyInitialPosition(work.init.reshape(-1).copy())
        _move(host, _kind(cfg), x["o"], x["d"], x["f"], x["w"], x.get("r"), x.get("t"), x.get("v"), x.get("b"))
        assert_same_particles(host, v8, f"{label} host chunk {chunk}")
        _assert_results_equal(_results(host, cfg), r8, f"{label} host chunk {chunk}")
        host.close()
    v8.close()
