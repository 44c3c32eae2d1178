"""Weight windows on device-resident c2 (998,250 tets, 10 M particles): device time of pumitally_generate_weight_windows
with 1 and 16 groups, of the particle lookup (device and host-pointer calls), of the point lookup next to
locate_points_device, and of one move for scale.  Bytes moved come from the byte model below and are reported as GB/s
against the H100 SXM data-sheet 3.35 TB/s, with the card name and power limit read in the same run.
Byte model (DESIGN section 4.13): generation reads mean, m2 and volume twice (group maximum, then the windows) and writes
16 B, 64 B per (group, element); the particle lookup reads a 32 B state sector, the 4 B group and a 32 B window sector
and writes 16 B, 84 B per particle; the point lookup is the location (not modelled) plus the same window traffic.
Usage: python scripts/bench_weight_windows.py [--reps 10]"""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
args = ap.parse_args()
assert torch.cuda.is_available(), "bench_weight_windows.py measures on a CUDA device"
dev = torch.device("cuda", 0)
card = torch.cuda.get_device_name(dev)
try:
    power = float(subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                                           "0"], text=True, timeout=30).strip())
except Exception:
    power = None
PEAK = 3.35e12


def events(fn, reps):
    """median ms between two CUDA events around fn() on the current stream (after one untimed call)"""
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
    """median ms of fn(), which ends in a device synchronisation (after one untimed call)"""
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def rate(ms, nbytes):
    return {"ms": ms, "model_bytes": nbytes, "GB_per_s": nbytes / (ms * 1e-3) / 1e9,
            "share_of_3.35TB_s": nbytes / (ms * 1e-3) / PEAK}


cfg = CONFIGS["c2"]
coords, t2v = kuhn_box(*cfg["cells"])
n = cfg["particles"]
E = len(t2v)
out = {"config": "c2", "elements": E, "particles": n, "card": card, "power_limit_w": power}
s = torch.cuda.current_stream().cuda_stream
g = torch.Generator(device=dev).manual_seed(2)
for ngroups in (1, 16):
    eng = PumiTally.from_arrays(coords, t2v, n, device=0)
    eng.set_batch_statistics(True)
    eng.set_score_bins(ngroups)
    wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device="cuda")
    eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
    for _ in range(2):
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        bins = torch.randint(0, ngroups, (n,), device=dev, dtype=torch.int32, generator=g)
        move = lambda: eng.move_device_binned(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), bins.data_ptr(), s)  # noqa: E731
        move()
        torch.cuda.synchronize()
        eng.end_batch()
    out[f"generate_{ngroups}_groups"] = rate(wall(lambda: eng.generate_weight_windows(0, 0, 0, 5.0, float("inf")),
                                                  args.reps), 64 * ngroups * E)
    if ngroups == 16:
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        out["move_binned_16_ms"] = events(lambda: eng.move_device_binned(o.data_ptr(), d.data_ptr(), f.data_ptr(),
                                                                          w.data_ptr(), bins.data_ptr(), s), 3)
        groups = torch.randint(0, 16, (n,), device=dev, dtype=torch.int32, generator=g)
        out["particles_device"] = rate(events(lambda: eng.weight_windows_at_particles_device(groups), args.reps),
                                       84 * n)
        gh = groups.cpu().numpy()
        out["particles_host_e2e"] = rate(wall(lambda: eng.weight_windows_at_particles(gh), max(args.reps // 2, 1)),
                                         84 * n)
        cells = torch.tensor(cfg["cells"], dtype=torch.float64, device=dev)
        pts = (torch.rand((n, 3), dtype=torch.float64, device=dev, generator=g) * cells).contiguous()
        out["locate_points_device_ms"] = events(lambda: eng.locate_device(pts), args.reps)
        out["points_device_ms"] = events(lambda: eng.weight_windows_at_points_device(pts, groups), args.reps)
    del eng
    torch.cuda.synchronize()
# one plain move of the flagship workload, for scale
eng = PumiTally.from_arrays(coords, t2v, n, device=0)
wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                       mu_min=cfg["mu_min"], backend="torch", device="cuda")
eng.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
steps = [tuple(x.contiguous() for x in wl.next_step()) for _ in range(4)]
for o, d, f, w in steps[:3]:
    eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
torch.cuda.synchronize()
o, d, f, w = steps[3]
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
b.record()
torch.cuda.synchronize()
out["move_plain_ms"] = a.elapsed_time(b)
print(json.dumps(out), flush=True)
