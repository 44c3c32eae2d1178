"""Point queries: points/s and kernel time of pumitally_locate_points_device for N uniform points in the mesh's bounding
box (inside and outside the mesh alike), the end-to-end time of the host call, and the end-to-end time of
pumitally_evaluate_points with 1 and 8 scores, with and without moments (the first call builds the evaluation table).
Prints one JSON line per config, with the card name and power limit.
Usage: python scripts/bench_locate.py [--configs c2,c3] [--points 10000000] [--reps 5]"""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS

ap = argparse.ArgumentParser()
ap.add_argument("--configs", default="c2,c3")
ap.add_argument("--points", type=int, default=10_000_000)
ap.add_argument("--reps", type=int, default=5)
args = ap.parse_args()
dev = torch.device("cuda", 0)
card = torch.cuda.get_device_name(dev)
try:
    power = float(subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                          text=True, timeout=30).strip())
except Exception:
    power = None


def timed_device(eng, pts, reps):
    """median ms of one locate_device call between two CUDA events (after one untimed call)"""
    stream = torch.cuda.current_stream()
    eng.locate_device(pts)
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        out = eng.locate_device(pts)
        b.record(stream)
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), out


def wall(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


for name in args.configs.split(","):
    cells = CONFIGS[name]["cells"]
    eng = PumiTally.from_spec(f"box:{cells[0]},{cells[1]},{cells[2]}", 16, device=0)
    n = args.points
    g = torch.Generator(device=dev).manual_seed(1)
    pts = (torch.rand((n, 3), dtype=torch.float64, device=dev, generator=g) *
           torch.tensor(cells, dtype=torch.float64, device=dev)).contiguous()
    out = {"config": name, "elements": eng.num_elements, "npts": n, "points": "uniform in the bounding box",
           "card": card, "power_limit_w": power}
    ms, elem = timed_device(eng, pts, args.reps)
    out["inside_fraction"] = float((elem >= 0).float().mean())
    out["locate_device"] = {"kernel_ms": ms, "points_per_s": n / (ms * 1e-3)}
    host = pts.cpu().numpy()
    ms = wall(lambda: eng.locate(host), max(args.reps // 2, 1))
    out["locate_host_e2e"] = {"ms": ms, "points_per_s": n / (ms * 1e-3)}
    ev = {}
    for k in (1, 8):
        for mo in (0, 1):
            eng.set_moments(mo)
            eng.set_scores(k)
            t0 = time.perf_counter()
            eng.evaluate(host)
            first = 1e3 * (time.perf_counter() - t0)
            ms = wall(lambda: eng.evaluate(host), max(args.reps // 2, 1))
            ev[f"scores{k}_moments{mo}"] = {"ms": ms, "first_call_ms": first, "points_per_s": n / (ms * 1e-3)}
    out["evaluate_host_e2e"] = ev
    del eng
    print(json.dumps(out), flush=True)
