"""Mesh source on device-resident c2 (998,250 tets, 10 M samples): device time of pumitally_sample_source_device with 1
and 16 groups, with and without bias, with and without placement; the host-pointer call end to end; and, for scale,
locate_points_device of the same points and one plain move.  CUDA events, medians.  The card name and power limit are
read in the same run.
Byte model (DESIGN section 4.15), in 32-byte L2 sectors per sample: the CDF search touches one sector per level,
ceil(log2(K + 1)) levels for K = groups * E entries (the top levels are shared by every sample and stay in L1/L2, so
this counts L2-level traffic, not DRAM); the element's vertices are three sectors (96 B); the bias one more sector; the
outputs are 40 B (xyz 24, element 4, group 4, weight 8); placement adds the 32 B state store and a sector of
internal_of_orig.  The rates below are these bytes over the kernel time, next to the H100 SXM data-sheet 3.35 TB/s.
Usage: python scripts/bench_source.py [--reps 10]"""
import argparse, json, math, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
args = ap.parse_args()
assert torch.cuda.is_available(), "bench_source.py measures on a CUDA device"
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


def model_bytes(K, biased, place):
    return 32 * math.ceil(math.log2(K + 1)) + 96 + (32 if biased else 0) + 40 + (64 if place else 0)


cfg = CONFIGS["c2"]
coords, t2v = kuhn_box(*cfg["cells"])
n = cfg["particles"]
E = len(t2v)
out = {"config": "c2", "elements": E, "samples": n, "card": card, "power_limit_w": power}
s = torch.cuda.current_stream().cuda_stream
eng = PumiTally.from_arrays(coords, t2v, n, device=0)
rng = np.random.default_rng(5)
xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
w = torch.empty(n, dtype=torch.float64, device=dev)
elem, group = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2))
for G in (1, 16):
    q = rng.lognormal(0.0, 1.0, (G, E))
    bias = rng.uniform(0.5, 2.0, (G, E))
    for biased in (False, True):
        eng.set_source(q, bias if biased else None, per_volume=True)
        for place in (False, True):
            def call(seed=[0]):
                seed[0] += 1
                if eng._L.pumitally_sample_source_device(eng._h, seed[0], 0, n, xyz.data_ptr(), elem.data_ptr(),
                                                         group.data_ptr(), w.data_ptr(), int(place), s):
                    raise RuntimeError("sample_source_device failed")
            ms = events(call, args.reps)
            nb = model_bytes(G * E, biased, place) * n
            out[f"device_G{G}_bias{int(biased)}_place{int(place)}"] = {
                "ms": ms, "ns_per_sample": ms * 1e6 / n, "model_bytes_per_sample": nb / n,
                "GB_per_s": nb / (ms * 1e-3) / 1e9, "share_of_3.35TB_s": nb / (ms * 1e-3) / PEAK}
out["host_e2e_G16_bias1_ms"] = wall(lambda: eng.sample_source(n, 99), max(args.reps // 2, 1))
pts, _, _, _ = eng.sample_source_device(n, 7)
torch.cuda.synchronize()
out["locate_points_device_same_points_ms"] = events(lambda: eng.locate_device(pts), args.reps)
# one plain move of the flagship workload, for scale
wl = SyntheticWorkload(box=tuple(float(x) for x in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"],
                       mu_min=cfg["mu_min"], backend="torch", device="cuda")
mv = PumiTally.from_arrays(coords, t2v, n, device=0)
mv.copy_initial_position_device(wl.initial_positions().contiguous().data_ptr(), s)
steps = [tuple(x.contiguous() for x in wl.next_step()) for _ in range(4)]
for o, d, f, ww in steps[:3]:
    mv.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), ww.data_ptr(), s)
torch.cuda.synchronize()
o, d, f, ww = steps[3]
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
mv.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), ww.data_ptr(), s)
b.record()
torch.cuda.synchronize()
out["move_plain_ms"] = a.elapsed_time(b)
print(json.dumps(out), flush=True)
