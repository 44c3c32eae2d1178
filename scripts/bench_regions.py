"""Region tallies: cost of the region pass of pumitally_end_batch (the region sums of every result of the batch, then
their fold) and of one pumitally_get_region_results call, device-resident, for
  - scores1: one score (the flux);
  - scores8_time16_collision: 8 scores, 16 time bins and the collision estimator (timed moves, events at the particles);
each without regions and with 1 region (every element), 64 slabs along z and one region per element.
end_batch synchronises, so it is timed by CUDA events around the call and by the wall clock.  The median of --reps
batches after one untimed batch.  The region pass is end_batch with regions minus end_batch without; the bytes it
reads (the m0 slots of every result of every element in a region, and the element list) over that time are printed
against the H100 SXM data-sheet bandwidth, and so are all the bytes it moves (also the region sums and their fold,
which matter once there are many regions).  Prints one JSON line per (variant, regions), with the card name and power
limit.
Usage: python scripts/bench_regions.py [--config c2] [--reps 5] [--dump-outputs DIR]
--dump-outputs writes the region batch means of the scores1 run with 64 slabs (pumitally_get_region_batch_results
kind 0, float64, one value per slab) as DIR/<config>_scores1_slabs64_mean.npy."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

DATASHEET_GBS = 3350.0  # H100 SXM5 80 GB HBM3

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
coords, t2v = kuhn_box(*cells)
E = len(t2v)
zc = coords[t2v].mean(axis=1)[:, 2]
slabs = np.minimum(((zc - zc.min()) / (zc.max() - zc.min()) * 64).astype(np.int32), 63)
MAPS = [("none", None), ("one", np.zeros(E, dtype=np.int32)), ("slabs64", slabs),
        ("per_element", np.arange(E, dtype=np.int32))]
VARIANTS = [("scores1", 1, 0, False), ("scores8_time16_collision", 8, 16, True)]

for label, ns, nt, coll in VARIANTS:
    eng = PumiTally.from_arrays(coords, t2v, n, device=0)
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
    base_ms = None
    for mname, rmap in MAPS:
        eng.set_regions(rmap)
        end_ms, end_wall_ms, get_ms = [], [], []
        for rep in range(args.reps + 1):  # batch 0 is untimed
            o, d, f, w = (x.contiguous() for x in wl.next_step())
            if nt:
                eng.move_device_timed(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), times.data_ptr(),
                                      speeds.data_ptr(), resp.data_ptr(), None, s)
            else:
                eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
            if coll:
                eng.tally_collisions_at_particles_device(collided, cw, resp, None, times if nt else None)
            torch.cuda.synchronize()
            if rmap is not None:  # one read of the open tally's region sums
                a, b = (torch.cuda.Event(enable_timing=True) for _ in range(2))
                a.record()
                eng.region_results(0, 0)  # synchronises
                b.record()
                torch.cuda.synchronize()
                if rep:
                    get_ms.append(a.elapsed_time(b))
            t0 = time.perf_counter()
            a, b = (torch.cuda.Event(enable_timing=True) for _ in range(2))
            a.record()
            eng.end_batch()  # synchronises
            b.record()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            if rep:
                end_ms.append(a.elapsed_time(b))
                end_wall_ms.append(1e3 * (t1 - t0))
        end = float(np.median(end_ms))
        out = {"config": args.config, "variant": label, "regions": mname, "nregions": eng.regions, "elements": E,
               "particles": n, "card": card, "power_limit_w": power, "batches": eng.batches,
               "end_batch_device_ms": end, "end_batch_wall_ms": float(np.median(end_wall_ms))}
        if rmap is None:
            base_ms = end
        else:
            R = max(nt, 1) * (2 if coll else 1)
            inside = int((rmap >= 0).sum())
            read = R * inside * ns * 8 + inside * 4  # m0 slots of every result array, and the element list
            # and the region sums written, then folded (read x, mean, m2, write mean, m2)
            moved = read + R * eng.regions * ns * 8 * 6
            extra = end - base_ms
            out.update({"end_batch_without_regions_ms": base_ms, "region_pass_ms": extra,
                        "region_pass_over_end_batch": extra / base_ms, "region_pass_bytes_read": read,
                        "region_pass_GB_per_s": read / (extra * 1e-3) / 1e9 if extra > 0 else None,
                        "fraction_of_datasheet": read / (extra * 1e-3) / 1e9 / DATASHEET_GBS if extra > 0 else None,
                        "region_pass_bytes_moved": moved,
                        "region_pass_moved_GB_per_s": moved / (extra * 1e-3) / 1e9 if extra > 0 else None,
                        "get_region_results_ms": float(np.median(get_ms))})
        if label == "scores1" and mname == "slabs64" and args.dump_outputs:
            np.save(os.path.join(args.dump_outputs, f"{args.config}_scores1_slabs64_mean.npy"),
                    eng.region_batch_results(0, 0)[0, 0, 0])
        print(json.dumps(out), flush=True)
    del eng
    torch.cuda.empty_cache()
