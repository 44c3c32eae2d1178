"""Detector void: time of pumitally_tally_detectors_device (located events) for N events uniform in the bounding box at
D detectors, on c2 with the void off, with it on and the detectors inside, and with it on and the detectors outside
the box (1 to 3 box sizes from its centre), alternated in one process; then on a c2-size box with a central cubic cavity
(19^3 of the 55^3 cells carved out), detectors in the cavity and beyond it, the void on.  Reports ms per call, rays/s,
crossings per ray and hull entries per ray.  CUDA events around each call, one untimed call first, the median of --reps.
Prints one JSON line per mesh, with the card name and power limit.
Usage: python scripts/bench_detector_void.py [--events 4000000] [--detectors 1,8] [--reps 5]"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS

ap = argparse.ArgumentParser()
ap.add_argument("--events", type=int, default=4_000_000)
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


def outside(rng, D, cells):
    u = rng.normal(size=(D, 3))
    return 0.5 * cells + u / np.linalg.norm(u, axis=1)[:, None] * cells * rng.uniform(1.0, 3.0, (D, 1))


def run(engines, pts, weights, D):
    """engines: name -> (engine, detectors); alternated; median ms, rays/s, crossings and hull entries per ray"""
    for eng, det in engines.values():
        eng.set_point_detectors(det, np.zeros(D))
        eng.set_detector_cross_sections(np.full((1, eng.num_elements), 0.05))
        eng.tally_detectors_device(pts, weights)  # warm-up (and the hull grid's upload)
    torch.cuda.synchronize()
    ts = {k: [] for k in engines}
    cnt = {}
    for _ in range(args.reps):
        for k, (eng, _) in engines.items():
            eng.reset_tally()
            ts[k].append(timed(lambda: eng.tally_detectors_device(pts, weights)))
            cnt[k] = (eng.get_option("detector_crossings"), eng.get_option("detector_hull_entries"))
    rays = D * len(pts)
    out = {}
    for k in engines:
        ms = float(np.median(ts[k]))
        out[k] = {"ms": ms, "rays_per_s": rays / (ms * 1e-3), "crossings_per_ray": cnt[k][0] / rays,
                  "hull_entries_per_ray": cnt[k][1] / rays}
    return out


n = args.events
g = torch.Generator(device=dev).manual_seed(1)
rng = np.random.default_rng(2)
cells = np.array(CONFIGS["c2"]["cells"], dtype=np.float64)
pts = (torch.rand((n, 3), dtype=torch.float64, device=dev, generator=g) * torch.tensor(cells, device=dev)).contiguous()
weights = torch.rand(n, dtype=torch.float64, device=dev, generator=g) + 0.5

c, t = kuhn_box(*CONFIGS["c2"]["cells"])
out = {"mesh": "c2", "elements": len(t), "events": n, "points": "uniform in the bounding box", "card": card,
       "power_limit_w": power}
off, on, on_out = (PumiTally.from_arrays(c, t, 16, device=0) for _ in range(3))
on.set_detector_void(True)
on_out.set_detector_void(True)
for D in (int(x) for x in args.detectors.split(",")):
    inside = rng.uniform(0.1, 0.9, size=(D, 3)) * cells
    out[f"D{D}"] = run({"void_off": (off, inside), "void_on_inside": (on, inside),
                        "void_on_outside": (on_out, outside(rng, D, cells))}, pts, weights, D)
del off, on, on_out
print(json.dumps(out), flush=True)

cen = c[t].mean(1)
keep = ~((cen > 18.0) & (cen < 37.0)).all(1)
verts, inv = np.unique(t[keep].ravel(), return_inverse=True)
cc, ct = np.ascontiguousarray(c[verts]), inv.reshape(-1, 4).astype(np.int32)
out = {"mesh": "c2 with a central 19^3 cavity", "elements": int(keep.sum()), "events": n,
       "points": "uniform in the bounding box", "card": card, "power_limit_w": power}
eng = PumiTally.from_arrays(cc, ct, 16, device=0)
eng.set_detector_void(True)
out["hull_candidates"] = None
for D in (int(x) for x in args.detectors.split(",")):
    det = np.concatenate([[[27.5, 27.5, 27.5]], outside(rng, D, cells)])[:D]
    out[f"D{D}"] = run({"void_on": (eng, det)}, pts, weights, D)
out["hull_candidates"] = eng.get_option("detector_hull_candidates")
print(json.dumps(out), flush=True)
