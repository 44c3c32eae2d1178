"""Cost of face currents: the move with currents against the same move without them (plain for K = 1, scored for
K > 1, timed with --time-bins), device-resident, one engine each, the two alternated move by move in this process
(same batches, same positions before every move).  Prints one JSON line: ms per move and segments/s of both, their
ratio, the kernel that ran, and the card name and power limit.
Usage: python scripts/bench_face_currents.py [--scores K] [--time-bins T] [--config c2] [--steps 10] [--warmup 3]"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

T_END = 4.0

ap = argparse.ArgumentParser()
ap.add_argument("--scores", type=int, default=1, metavar="K", help="scores, 1..8")
ap.add_argument("--time-bins", type=int, default=0, metavar="T", help="time bins, 0 (none) .. 1024")
ap.add_argument("--config", default="c2")
ap.add_argument("--particles", type=int, default=0, help="override the config's particle count")
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--variant", type=int, default=-1)
args = ap.parse_args()
if not 0 <= args.time_bins <= 1024 or not 1 <= args.scores <= 8 or args.steps < 1:
    raise SystemExit("bench_face_currents.py: --scores must be 1..8, --time-bins 0..1024 and --steps at least 1")

cfg = CONFIGS[args.config]
cells = cfg["cells"]
spec = f"box:{cells[0]},{cells[1]},{cells[2]}"
n, K, T, steps, warmup = args.particles or cfg["particles"], args.scores, args.time_bins, args.steps, max(args.warmup, 0)
dev = torch.device("cuda", 0)
stream = torch.cuda.current_stream().cuda_stream
edges = np.linspace(0.0, T_END, T + 1)


def new_engine(currents):
    e = PumiTally.from_spec(spec, n, device=0)
    e.set_option("variant", args.variant)  # -1 = the engine's own choice for this mesh
    if K > 1:
        e.set_scores(K)
    if T:
        e.set_time_bins(edges)
    if currents:
        e.set_face_currents(True)
    return e


wl = SyntheticWorkload(box=tuple(float(c) for c in cells), num_particles=n, mean_length=cfg["mean_length"],
                       mu_min=cfg["mu_min"], backend="torch", device=dev)
init = wl.initial_positions().contiguous()
g = torch.Generator(device=dev).manual_seed(17)
resp = (torch.rand((n, K), dtype=torch.float64, device=dev, generator=g) * 2.0).contiguous()

cur, base = new_engine(True), new_engine(False)
for e in (cur, base):
    e.copy_initial_position_device(init.data_ptr(), stream)
ms = {"currents": 0.0, "plain": 0.0}
st0 = {}
for k in range(warmup + steps):
    o, d, f, w = (x.contiguous() for x in wl.next_step())
    if T:  # start times in [0, 2), flight times in [0.5, 2)
        length = torch.linalg.norm(d.view(-1, 3) - o.view(-1, 3), dim=1).clamp_min(1e-9)
        t = (torch.rand(n, dtype=torch.float64, device=dev, generator=g) * 2.0).contiguous()
        v = (length / (0.5 + torch.rand(n, dtype=torch.float64, device=dev, generator=g) * 1.5)).contiguous()
    if k == warmup:
        torch.cuda.synchronize()
        st0 = {"currents": cur.stats(), "plain": base.stats()}
    for name, e in (("currents", cur), ("plain", base)):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        if T:
            e.move_device_timed(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), t.data_ptr(), v.data_ptr(),
                                resp.data_ptr() if K > 1 else None, None, stream)
        elif K > 1:
            e.move_device_scored(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), resp.data_ptr(), None, stream)
        else:
            e.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), stream)
        ev1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            ms[name] += ev0.elapsed_time(ev1)
out = {"nscores": K, "time_bins": T, "config": args.config, "particles": n, "steps": steps,
       "move": "timed" if T else ("scored" if K > 1 else "plain"),
       "timing": "per-move CUDA events, moves with and without face currents alternated on the same batches"}
for name, e in (("currents", cur), ("plain", base)):
    segs = e.stats()["segments"] - st0[name]["segments"]
    out[name] = {"ms_per_move": ms[name] / steps, "segments_per_s": segs / (ms[name] * 1e-3),
                 "variant": e.get_option("variant"), "walk_blocks_per_sm": e.get_option("walk_blocks_per_sm")}
out["ratio_currents_to_plain"] = out["currents"]["ms_per_move"] / out["plain"]["ms_per_move"]
del cur, base
out["card"] = torch.cuda.get_device_name(dev)
try:
    out["power_limit_w"] = float(subprocess.check_output(
        ["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], text=True, timeout=30).strip())
except Exception:
    out["power_limit_w"] = None
print(json.dumps(out), flush=True)
