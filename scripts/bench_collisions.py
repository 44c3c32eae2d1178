"""Collision estimator: kernel time of pumitally_tally_collisions_device (located events) and
pumitally_tally_collisions_at_particles_device (events at the particles) for N events on a config's mesh, with 1, 4 and 8
scores, with moments and with 16 time bins; the end-to-end time of the host-pointer calls; and, in the same run,
pumitally_locate_points_device on the same points (the floor of the located kernel) and one device move of the config's
particles (to put the cost next to a walk).  c3 has ~200 events per element, so it shows reduction contention.
CUDA events around each call, one untimed call first, the median of --reps.  Prints one JSON line per config, with the
card name and power limit.
Usage: python scripts/bench_collisions.py [--configs c2,c3] [--events 10000000] [--reps 5] [--dump-outputs DIR]
--dump-outputs writes the raw collision tally of the 1-score located and at-particles runs as
DIR/<config>_located.npy and DIR/<config>_particles.npy (float64, one value per element, caller's numbering)."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

ap = argparse.ArgumentParser()
ap.add_argument("--configs", default="c2,c3")
ap.add_argument("--events", type=int, default=10_000_000)
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


def timed(fn, reps):
    """median ms between two CUDA events around fn() (after one untimed call)"""
    stream = torch.cuda.current_stream()
    fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def wall(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


VARIANTS = [("scores1", 1, 0, None), ("scores4", 4, 0, None), ("scores8", 8, 0, None), ("scores1_moments", 1, 1, None),
            ("scores1_time16", 1, 0, np.linspace(0.0, 16.0, 17))]

for name in args.configs.split(","):
    cfg = CONFIGS[name]
    cells = cfg["cells"]
    n = args.events
    g = torch.Generator(device=dev).manual_seed(1)
    eng = PumiTally.from_spec(f"box:{cells[0]},{cells[1]},{cells[2]}", n, device=0)
    wl = SyntheticWorkload(box=tuple(float(c) for c in cells), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
    for step in range(2):  # the first move warms up, the second is timed
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
        b.record()
        torch.cuda.synchronize()
    move_ms = a.elapsed_time(b)
    pts = (torch.rand((n, 3), dtype=torch.float64, device=dev, generator=g) *
           torch.tensor(cells, dtype=torch.float64, device=dev)).contiguous()
    weights = torch.rand(n, dtype=torch.float64, device=dev, generator=g) + 0.5
    times = torch.rand(n, dtype=torch.float64, device=dev, generator=g) * 16.0
    collided = torch.ones(n, dtype=torch.int8, device=dev)
    out = {"config": name, "elements": eng.num_elements, "events": n, "points": "uniform in the bounding box",
           "card": card, "power_limit_w": power, "move_device_ms": move_ms,
           "locate_device_ms": timed(lambda: eng.locate_device(pts), args.reps)}
    for label, ns, mo, edges in VARIANTS:
        eng.set_moments(mo)
        eng.set_scores(ns)
        eng.set_time_bins(edges)
        eng.set_collision_estimator(True)
        resp = (torch.rand((n, ns), dtype=torch.float64, device=dev, generator=g) if ns > 1 else None)
        t = times if edges is not None else None
        loc = timed(lambda: eng.tally_collisions_device(pts, weights, resp, None, t), args.reps)
        par = timed(lambda: eng.tally_collisions_at_particles_device(collided, weights, resp, None, t), args.reps)
        out[label] = {"located_ms": loc, "particles_ms": par, "located_events_per_s": n / (loc * 1e-3),
                      "particles_events_per_s": n / (par * 1e-3)}
        if label == "scores1" and args.dump_outputs:
            for kind, fn in (("located", lambda: eng.tally_collisions_device(pts, weights)),
                             ("particles", lambda: eng.tally_collisions_at_particles_device(collided, weights))):
                eng.reset_tally()
                fn()
                torch.cuda.synchronize()
                np.save(os.path.join(args.dump_outputs, f"{name}_{kind}.npy"), eng.collision_results(0)[0, 0, 0])
    eng.set_time_bins(None)
    eng.set_moments(0)
    eng.set_scores(1)
    eng.set_collision_estimator(True)
    hp, hw, hc = pts.cpu().numpy(), weights.cpu().numpy(), collided.cpu().numpy()
    reps = max(args.reps // 2, 1)
    out["host_e2e"] = {"located_ms": wall(lambda: eng.tally_collisions(hp, hw), reps),
                       "particles_ms": wall(lambda: eng.tally_collisions_at_particles(hc, hw), reps)}
    del eng
    print(json.dumps(out), flush=True)
