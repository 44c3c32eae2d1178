"""Cost of scores: a K-score move against a plain move of the same inputs, device-resident, one engine each,
the two alternated move by move in this process (same batches, same positions before every move), plus the
end-to-end time of the host-pointer scored move.  Prints one JSON line: ms per move and segments/s of both,
their ratio, the kernel that ran, the e2e ms per move, and the card name and power limit.
Usage: python scripts/bench_scores.py --scores K [--config c2] [--steps 10] [--warmup 3] [--dump-outputs DIR]
--dump-outputs writes the scored engine's flux of every score as DIR/flux_score<k>.npy (float64; over 2^20
elements as a fixed seeded sample, with flux_index.npy)."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

DUMP_ROWS = 1 << 20

ap = argparse.ArgumentParser()
ap.add_argument("--scores", type=int, required=True, metavar="K", help="scores of the scored move, 1..8")
ap.add_argument("--config", default="c2")
ap.add_argument("--particles", type=int, default=0, help="override the config's particle count")
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--variant", type=int, default=-1)
ap.add_argument("--dump-outputs", metavar="DIR", default=None)
args = ap.parse_args()
if not 1 <= args.scores <= 8 or args.steps < 1:
    raise SystemExit("bench_scores.py: --scores must be between 1 and 8 and --steps at least 1")

cfg = CONFIGS[args.config]
cells = cfg["cells"]
box = tuple(float(c) for c in cells)
spec = f"box:{cells[0]},{cells[1]},{cells[2]}"
n, K, steps, warmup = args.particles or cfg["particles"], args.scores, args.steps, max(args.warmup, 0)
dev = torch.device("cuda", 0)
stream = torch.cuda.current_stream().cuda_stream


def workload():
    return SyntheticWorkload(box=box, num_particles=n, mean_length=cfg["mean_length"], mu_min=cfg["mu_min"],
                             backend="torch", device=dev)


def new_engine(k):
    e = PumiTally.from_spec(spec, n, device=0)
    e.set_option("variant", args.variant)  # -1 = the engine's own choice for this mesh
    if k > 1:
        e.set_scores(k)
    return e


wl = workload()
init = wl.initial_positions().contiguous()
g = torch.Generator(device=dev).manual_seed(17)
resp = (torch.rand((n, K), dtype=torch.float64, device=dev, generator=g) * 2.0).contiguous()

# ---- device-resident: scored and plain moves alternated on the same batches
scored, plain = new_engine(K), new_engine(1)
for e in (scored, plain):
    e.copy_initial_position_device(init.data_ptr(), stream)
ms = {"scored": 0.0, "plain": 0.0}
st0 = {}
for k in range(warmup + steps):
    o, d, f, w = (x.contiguous() for x in wl.next_step())
    if k == warmup:
        torch.cuda.synchronize()
        st0 = {"scored": scored.stats(), "plain": plain.stats()}
    for name in ("scored", "plain"):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        if name == "scored":
            scored.move_device_scored(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), resp.data_ptr(), None, stream)
        else:
            plain.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), stream)
        ev1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            ms[name] += ev0.elapsed_time(ev1)
out = {"nscores": K, "config": args.config, "particles": n, "steps": steps,
       "timing": "per-move CUDA events, scored and plain moves alternated on the same batches"}
for name, e in (("scored", scored), ("plain", plain)):
    segs = e.stats()["segments"] - st0[name]["segments"]
    out[name] = {"ms_per_move": ms[name] / steps, "segments_per_s": segs / (ms[name] * 1e-3),
                 "variant": e.get_option("variant"), "walk_blocks_per_sm": e.get_option("walk_blocks_per_sm")}
out["ratio_scored_to_plain"] = out["scored"]["ms_per_move"] / out["plain"]["ms_per_move"]
out["ratio_to_k_plain_moves"] = out["scored"]["ms_per_move"] / (K * out["plain"]["ms_per_move"])
if args.dump_outputs:
    os.makedirs(args.dump_outputs, exist_ok=True)
    fs = scored.flux_scores[0]
    idx = None if fs.shape[1] <= DUMP_ROWS else np.sort(np.random.default_rng(0x5EED).choice(fs.shape[1], DUMP_ROWS, replace=False))
    if idx is not None:
        np.save(os.path.join(args.dump_outputs, "flux_index.npy"), idx.astype(np.float64))
    for k in range(K):
        np.save(os.path.join(args.dump_outputs, f"flux_score{k}.npy"),
                np.ascontiguousarray(fs[k] if idx is None else fs[k][idx], dtype=np.float64))
del scored, plain

# ---- end to end: the host-pointer scored move on pageable arrays the caller reuses for every move
e2 = new_engine(K)
wl2 = workload()
e2.CopyInitialPosition(wl2.initial_positions().cpu().numpy().reshape(-1))
O, D, F, W = np.empty(3 * n), np.empty(3 * n), np.empty(n, dtype=np.int8), np.empty(n)
R = resp.cpu().numpy()
ke, kw, dt = min(steps, 5), min(warmup, 2), 0.0
for k in range(kw + ke):
    for dst, src in zip((O, D, F, W), wl2.next_step()):
        dst[:] = src.reshape(-1).cpu().numpy()
    t0 = time.perf_counter()
    e2.MoveToNextLocationScored(O, D, F, W, R)
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
