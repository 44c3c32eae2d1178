"""Batch statistics: cost of pumitally_end_batch (fold of every reported double into the running mean and M2, then the
tally reset) next to one device move of the same config, device-resident, for
  - scores1: one score (the flux);
  - scores8_time16_collision: 8 scores, 16 time bins and the collision estimator (timed moves, events at the particles).
end_batch synchronises, so it is timed by CUDA events around the call and by the wall clock; the move by CUDA events.
The median of --reps batches after one untimed batch.  Prints one JSON line per variant, with the card name and power
limit.
Usage: python scripts/bench_batch_stats.py [--config c2] [--reps 5] [--dump-outputs DIR]
--dump-outputs writes the batch means of the scores1 run (pumitally_get_batch_results kind 0, float64, one value per
element, caller's numbering) as DIR/<config>_scores1_mean.npy."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

ap = argparse.ArgumentParser()
ap.add_argument("--config", default="c2")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--dump-outputs", metavar="DIR", default=None)
args = ap.parse_args()
dev = torch.device("cuda", 0)
card = torch.cuda.get_device_name(dev)
try:
    power = float(subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                          text=True, timeout=30).strip())
except Exception:
    power = None
if args.dump_outputs:
    os.makedirs(args.dump_outputs, exist_ok=True)

cfg = CONFIGS[args.config]
cells = cfg["cells"]
n = cfg["particles"]
VARIANTS = [("scores1", 1, 0, False), ("scores8_time16_collision", 8, 16, True)]

for label, ns, nt, coll in VARIANTS:
    eng = PumiTally.from_spec(f"box:{cells[0]},{cells[1]},{cells[2]}", n, device=0)
    eng.set_scores(ns)
    if nt:
        eng.set_time_bins(np.linspace(0.0, 16.0, nt + 1))
    eng.set_collision_estimator(coll)
    eng.set_batch_statistics(True)
    eng.set_source_normalization(3)
    wl = SyntheticWorkload(box=tuple(float(c) for c in cells), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    g = torch.Generator(device=dev).manual_seed(1)
    resp = torch.rand((n, ns), dtype=torch.float64, device=dev, generator=g) if ns > 1 else None
    times = torch.rand(n, dtype=torch.float64, device=dev, generator=g) * 16.0
    speeds = torch.ones(n, dtype=torch.float64, device=dev)
    collided = (torch.rand(n, device=dev, generator=g) < 0.5).to(torch.int8)
    cw = torch.rand(n, dtype=torch.float64, device=dev, generator=g) + 0.5
    s = torch.cuda.current_stream().cuda_stream
    eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
    move_ms, end_ms, end_wall_ms = [], [], []
    for rep in range(args.reps + 1):  # batch 0 is untimed
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        a.record()
        if nt:
            eng.move_device_timed(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), times.data_ptr(),
                                  speeds.data_ptr(), resp.data_ptr(), None, s)
        else:
            eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
        b.record()
        if coll:
            eng.tally_collisions_at_particles_device(collided, cw, resp, None, times if nt else None)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b2 = torch.cuda.Event(enable_timing=True)
        b2.record()
        eng.end_batch()  # synchronises
        c.record()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if rep:
            move_ms.append(a.elapsed_time(b))
            end_ms.append(b2.elapsed_time(c))
            end_wall_ms.append(1e3 * (t1 - t0))
    doubles = (max(nt, 1) * ns * eng.num_elements) * (2 if coll else 1)
    stride = 1 if ns == 1 else 2 if ns == 2 else 4 if ns <= 4 else 8  # score slots per element record
    padded = (max(nt, 1) * stride * eng.num_elements) * (2 if coll else 1)
    out = {"config": args.config, "variant": label, "elements": eng.num_elements, "particles": n,
           "card": card, "power_limit_w": power, "batches": eng.batches,
           "reported_doubles": doubles, "folded_doubles": padded,
           "move_device_ms": float(np.median(move_ms)), "end_batch_device_ms": float(np.median(end_ms)),
           "end_batch_wall_ms": float(np.median(end_wall_ms)),
           "end_batch_over_move": float(np.median(end_ms) / np.median(move_ms)),
           # fold: read x, mean, m2, write mean, m2 (40 B); reset: write x (8 B)
           "end_batch_GB_per_s": 48.0 * padded / (np.median(end_ms) * 1e-3) / 1e9}
    if label == "scores1" and args.dump_outputs:
        np.save(os.path.join(args.dump_outputs, f"{args.config}_scores1_mean.npy"), eng.batch_results(0, 0)[0, 0, 0])
    del eng
    torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)
