"""Point detectors: time of pumitally_tally_detectors_device (located events) and
pumitally_tally_detectors_at_particles_device (events at the particles) for N isotropic events at D detectors on a
config's mesh, next to one device move of the config's particles and pumitally_locate_points_device of the same points,
alternated in one process.  Reports ms per call, rays/s and crossings/s (option "detector_crossings").  CUDA events around
each call, one untimed call first, the median of --reps.  Prints one JSON line per config, with the card name and power
limit.
Usage: python scripts/bench_detectors.py [--configs c2,c3] [--events 10000000] [--detectors 1,8] [--reps 5]"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

ap = argparse.ArgumentParser()
ap.add_argument("--configs", default="c2,c3")
ap.add_argument("--events", type=int, default=10_000_000)
ap.add_argument("--detectors", default="1,8")
ap.add_argument("--reps", type=int, default=5)
args = ap.parse_args()
dev = torch.device("cuda", 0)
card = torch.cuda.get_device_name(dev)
try:
    power = float(subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                          text=True, timeout=30).strip())
except Exception:
    power = None


def timed(fn):
    """ms between two CUDA events around fn()"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


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
    o, d, f, w = (x.contiguous() for x in wl.next_step())
    move = lambda: eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)  # noqa: E731
    move()
    torch.cuda.synchronize()
    pts = (torch.rand((n, 3), dtype=torch.float64, device=dev, generator=g) *
           torch.tensor(cells, dtype=torch.float64, device=dev)).contiguous()
    weights = torch.rand(n, dtype=torch.float64, device=dev, generator=g) + 0.5
    flagged = torch.ones(n, dtype=torch.int8, device=dev)
    out = {"config": name, "elements": eng.num_elements, "events": n, "points": "uniform in the bounding box",
           "card": card, "power_limit_w": power}
    rng = np.random.default_rng(2)
    for D in (int(x) for x in args.detectors.split(",")):
        det = rng.uniform(0.1, 0.9, size=(D, 3)) * np.array(cells, dtype=np.float64)
        eng.set_point_detectors(det, np.full(D, 0.5))
        eng.set_detector_cross_sections(np.full((1, eng.num_elements), 0.05))
        calls = {"move": move, "locate": lambda: eng.locate_device(pts),
                 "located": lambda: eng.tally_detectors_device(pts, weights),
                 "particles": lambda: eng.tally_detectors_at_particles_device(flagged, weights)}
        for fn in calls.values():  # warm-up
            fn()
        torch.cuda.synchronize()
        ts = {k: [] for k in calls}
        cross = {"located": 0, "particles": 0}
        for _ in range(args.reps):  # alternated
            for k, fn in calls.items():
                if k in cross:
                    eng.reset_tally()
                ts[k].append(timed(fn))
                if k in cross:
                    cross[k] = eng.get_option("detector_crossings")
        r = {k: float(np.median(v)) for k, v in ts.items()}
        out[f"D{D}"] = {"move_device_ms": r["move"], "locate_device_ms": r["locate"],
                        **{f"{k}_ms": r[k] for k in cross},
                        **{f"{k}_rays_per_s": D * n / (r[k] * 1e-3) for k in cross},
                        **{f"{k}_crossings_per_s": cross[k] / (r[k] * 1e-3) for k in cross},
                        **{f"{k}_crossings_per_ray": cross[k] / (D * n) for k in cross}}
    del eng
    print(json.dumps(out), flush=True)
