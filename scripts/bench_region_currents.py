"""Cost of region currents: end_batch and region_current_results on c2 with face currents and batch statistics on,
with region currents against without them, for block maps of 8 (2^3), 64 (4^3) and 4096 (16^3) regions (each element
in the block of its centroid) and for one region per element, the worst case (P about 4E / 2 plus the hull).  Two
engines per map, the same batches, alternated batch by batch; every timed call is bracketed by device synchronisation
and a host clock.  Next to every time it prints the byte model of the added work from the shapes:
  level 0 of the pair sums reads a 4 B slot id and a gathered 32 B sector per slot in a pair (later levels read the
  chunk sums, at most 1/32 of that); the net kernel moves 24 B per (array, pair); the fold moves 40 B per double of the
  2 ntime nbins P added region results;
and that model's time at the H100 SXM data-sheet bandwidth of 3.35 TB/s (a bound, not a measurement).  Prints one JSON
line per map and one with the card name and power limit.
Usage: python scripts/bench_region_currents.py [--config c2] [--steps 5] [--warmup 2]"""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.partition import face_adjacency
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

HBM_BYTES_PER_S = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--config", default="c2")
ap.add_argument("--particles", type=int, default=0, help="override the config's particle count")
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
args = ap.parse_args()
if args.steps < 1:
    raise SystemExit("bench_region_currents.py: --steps must be at least 1")

cfg = CONFIGS[args.config]
cells = cfg["cells"]
n, steps, warmup = args.particles or cfg["particles"], args.steps, max(args.warmup, 0)
dev = torch.device("cuda", 0)
stream = torch.cuda.current_stream().cuda_stream


def block_map(cen, lo, hi, k):
    idx = np.minimum(((cen - lo) / (hi - lo) * k).astype(np.int64), k - 1)
    return ((idx[:, 0] * k + idx[:, 1]) * k + idx[:, 2]).astype(np.int32)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


coords, t2v = kuhn_box(*cells)
adj = face_adjacency(t2v, len(coords))
E = len(t2v)
cen = coords[t2v].mean(axis=1)
lo, hi = coords.min(axis=0), coords.max(axis=0)
maps = {"blocks_8": block_map(cen, lo, hi, 2), "blocks_64": block_map(cen, lo, hi, 4),
        "blocks_4096": block_map(cen, lo, hi, 16), "per_element": np.arange(E, dtype=np.int32)}
e_of = np.repeat(np.arange(E), 4)
nb = adj.reshape(-1)

for name, region in maps.items():
    engines = {}
    for rc in (False, True):
        e = PumiTally.from_arrays(coords, t2v, n, device=0)
        e.set_face_currents(True)
        e.set_batch_statistics(True)
        e.set_regions(region, int(region.max()) + 1)
        if rc:
            e.set_region_currents(True)
        engines[rc] = e
    wl = SyntheticWorkload(box=tuple(float(c) for c in cells), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device=dev)
    init = wl.initial_positions().contiguous()
    for e in engines.values():
        e.copy_initial_position_device(init.data_ptr(), stream)
    ms = {"end_batch_without": 0.0, "end_batch_with": 0.0, "move": 0.0, "partial_results": 0.0, "net_results": 0.0}
    for k in range(warmup + steps):
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        for rc, e in engines.items():
            t_move = timed(lambda: e.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), stream))
            t_p = timed(lambda: e.region_current_results(0, 0)) if rc else 0.0
            t_n = timed(lambda: e.region_current_results(1, 0)) if rc else 0.0
            t_end = timed(e.end_batch)
            if k >= warmup:
                ms["end_batch_with" if rc else "end_batch_without"] += t_end
                if rc:
                    ms["move"] += t_move
                    ms["partial_results"] += t_p
                    ms["net_results"] += t_n
    ms = {key: v / steps for key, v in ms.items()}
    on = engines[True]
    P = len(on.region_current_pairs()[0])
    R = max(on.time_bins, 1) * on.score_bins
    S = int((nb < 0).sum() + ((nb >= 0) & (region[e_of] != region[np.maximum(nb, 0)])).sum())
    model = {"level0_bytes": 36 * S * R, "net_bytes": 24 * R * P, "fold_bytes": 40 * 2 * R * P}
    total = sum(model.values())
    out = {"config": args.config, "particles": n, "map": name, "regions": int(region.max()) + 1, "pairs": P,
           "slots_in_pairs": S, "arrays": R, "steps": steps,
           "ms": ms, "end_batch_added_ms": ms["end_batch_with"] - ms["end_batch_without"],
           "byte_model": model, "byte_model_total": total,
           "byte_model_ms_at_3.35TB_s": total / HBM_BYTES_PER_S * 1e3,
           "timing": "host clock between device synchronisations, engines with and without region currents "
                     "alternated on the same batches"}
    print(json.dumps(out), flush=True)
    del engines, on
    torch.cuda.empty_cache()

card = {"card": torch.cuda.get_device_name(dev)}
try:
    card["power_limit_w"] = float(subprocess.check_output(
        ["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], text=True, timeout=30).strip())
except Exception:
    card["power_limit_w"] = None
print(json.dumps(card), flush=True)
