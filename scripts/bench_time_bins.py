"""Cost of a time filter: a timed move with T time bins against the scored move (the plain move for K = 1) of the
same inputs, device-resident, one engine each, the two alternated move by move in this process (same batches, same
positions before every move), plus the end-to-end time of the host-pointer timed move.  Prints one JSON line: ms per
move and segments/s of both, their ratio, the mean number of time-bin edges a track crosses (from the inputs), the
kernel that ran, the e2e ms per move, and the card name and power limit.
The time bins split [0, 4) evenly; particle i starts at a time in [0, 2) and flies for a time in [0.5, 2), so with
T bins a track crosses about 1.25 * T / 4 edges.
Usage: python scripts/bench_time_bins.py --time-bins T [--scores K] [--config c2] [--steps 10] [--warmup 3]
       [--dump-outputs DIR]
--dump-outputs writes the timed engine's flux of every time bin and score as DIR/flux_t<j>_score<k>.npy (float64;
over 2^20 elements as a fixed seeded sample, with flux_index.npy)."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

DUMP_ROWS = 1 << 20
T_END = 4.0

ap = argparse.ArgumentParser()
ap.add_argument("--time-bins", type=int, required=True, metavar="T", help="time bins, 1..1024")
ap.add_argument("--scores", type=int, default=1, metavar="K", help="scores, 1..8")
ap.add_argument("--config", default="c2")
ap.add_argument("--particles", type=int, default=0, help="override the config's particle count")
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--variant", type=int, default=-1)
ap.add_argument("--dump-outputs", metavar="DIR", default=None)
args = ap.parse_args()
if not 1 <= args.time_bins <= 1024 or not 1 <= args.scores <= 8 or args.steps < 1:
    raise SystemExit("bench_time_bins.py: --time-bins must be 1..1024, --scores 1..8 and --steps at least 1")

cfg = CONFIGS[args.config]
cells = cfg["cells"]
box = tuple(float(c) for c in cells)
spec = f"box:{cells[0]},{cells[1]},{cells[2]}"
n, K, T, steps, warmup = args.particles or cfg["particles"], args.scores, args.time_bins, args.steps, max(args.warmup, 0)
dev = torch.device("cuda", 0)
stream = torch.cuda.current_stream().cuda_stream
edges = np.linspace(0.0, T_END, T + 1)
edges_dev = torch.from_numpy(edges).to(dev)


def workload():
    return SyntheticWorkload(box=box, num_particles=n, mean_length=cfg["mean_length"], mu_min=cfg["mu_min"],
                             backend="torch", device=dev)


def new_engine(timed):
    e = PumiTally.from_spec(spec, n, device=0)
    e.set_option("variant", args.variant)  # -1 = the engine's own choice for this mesh
    if K > 1:
        e.set_scores(K)
    if timed:
        e.set_time_bins(edges)
    return e


def times_speeds(o, d, g):
    """Start times in [0, 2), flight times in [0.5, 2); mean edges crossed per flying track from the inputs."""
    length = torch.linalg.norm(d.view(-1, 3) - o.view(-1, 3), dim=1).clamp_min(1e-9)
    t = (torch.rand(n, dtype=torch.float64, device=dev, generator=g) * 2.0).contiguous()
    dur = 0.5 + torch.rand(n, dtype=torch.float64, device=dev, generator=g) * 1.5
    v = (length / dur).contiguous()
    t1 = t + length / v
    inner = ((edges_dev[None, :] > t[:, None]) & (edges_dev[None, :] < t1[:, None])).sum(dim=1) if T <= 64 else \
        (torch.searchsorted(edges_dev, t1, right=False) - torch.searchsorted(edges_dev, t, right=True))
    return t, v, inner


wl = workload()
init = wl.initial_positions().contiguous()
g = torch.Generator(device=dev).manual_seed(17)
resp = (torch.rand((n, K), dtype=torch.float64, device=dev, generator=g) * 2.0).contiguous()

# ---- device-resident: timed and untimed moves alternated on the same batches
timed, base = new_engine(True), new_engine(False)
for e in (timed, base):
    e.copy_initial_position_device(init.data_ptr(), stream)
ms = {"timed": 0.0, "untimed": 0.0}
st0 = {}
cross_sum, cross_n = 0.0, 0
for k in range(warmup + steps):
    o, d, f, w = (x.contiguous() for x in wl.next_step())
    t, v, inner = times_speeds(o, d, g)
    fly = f == 1
    if k >= warmup:
        cross_sum += float(inner[fly].sum())
        cross_n += int(fly.sum())
    if k == warmup:
        torch.cuda.synchronize()
        st0 = {"timed": timed.stats(), "untimed": base.stats()}
    for name in ("timed", "untimed"):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        if name == "timed":
            timed.move_device_timed(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), t.data_ptr(), v.data_ptr(),
                                    resp.data_ptr() if K > 1 else None, None, stream)
        elif K > 1:
            base.move_device_scored(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), resp.data_ptr(), None, stream)
        else:
            base.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), stream)
        ev1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            ms[name] += ev0.elapsed_time(ev1)
out = {"time_bins": T, "nscores": K, "config": args.config, "particles": n, "steps": steps,
       "untimed_move": "scored" if K > 1 else "plain",
       "timing": "per-move CUDA events, timed and untimed moves alternated on the same batches",
       "mean_edges_crossed_per_track": cross_sum / max(cross_n, 1)}
for name, e in (("timed", timed), ("untimed", base)):
    segs = e.stats()["segments"] - st0[name]["segments"]
    out[name] = {"ms_per_move": ms[name] / steps, "segments_per_s": segs / (ms[name] * 1e-3),
                 "variant": e.get_option("variant"), "walk_blocks_per_sm": e.get_option("walk_blocks_per_sm")}
out["ratio_timed_to_untimed"] = out["timed"]["ms_per_move"] / out["untimed"]["ms_per_move"]
if args.dump_outputs:
    os.makedirs(args.dump_outputs, exist_ok=True)
    ft = timed.flux_time[:, 0]
    E = ft.shape[-1]
    idx = None if E <= DUMP_ROWS else np.sort(np.random.default_rng(0x5EED).choice(E, DUMP_ROWS, replace=False))
    if idx is not None:
        np.save(os.path.join(args.dump_outputs, "flux_index.npy"), idx.astype(np.float64))
    for j in range(T):
        for k in range(K):
            np.save(os.path.join(args.dump_outputs, f"flux_t{j}_score{k}.npy"),
                    np.ascontiguousarray(ft[j, k] if idx is None else ft[j, k][idx], dtype=np.float64))
del timed, base

# ---- end to end: the host-pointer timed move on pageable arrays the caller reuses for every move
e2 = new_engine(True)
wl2 = workload()
e2.CopyInitialPosition(wl2.initial_positions().cpu().numpy().reshape(-1))
O, D, F, W = np.empty(3 * n), np.empty(3 * n), np.empty(n, dtype=np.int8), np.empty(n)
TT, V = np.empty(n), np.empty(n)
R = resp.cpu().numpy() if K > 1 else None
ke, kw, dt = min(steps, 5), min(warmup, 2), 0.0
for k in range(kw + ke):
    step = wl2.next_step()
    for dst, src in zip((O, D, F, W), step):
        dst[:] = src.reshape(-1).cpu().numpy()
    t, v, _ = times_speeds(step[0].contiguous(), step[1].contiguous(), g)
    TT[:], V[:] = t.cpu().numpy(), v.cpu().numpy()
    t0 = time.perf_counter()
    e2.MoveToNextLocationTimed(O, D, F, W, TT, V, R)
    e2.stats()  # device->host read of the step's result (synchronises)
    if k >= kw:
        dt += time.perf_counter() - t0
out["e2e_ms_per_move"] = 1e3 * dt / ke
del e2
out["card"] = torch.cuda.get_device_name(dev)
try:
    out["power_limit_w"] = float(subprocess.check_output(
        ["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], text=True, timeout=30).strip())
except Exception:
    out["power_limit_w"] = None
print(json.dumps(out), flush=True)
