"""Checkpoints: wall time, bytes and GB/s of pumitally_save_checkpoint at a batch end and mid-batch, of
pumitally_load_checkpoint and of pumitally_merge_checkpoint, device-resident, for
  - scores1: one score (the flux);
  - scores8_time16_collision_slabs64: 8 scores, 16 time bins, the collision estimator (events at the particles) and 64
    slab regions.
In the same run and the same directory (--dir), the plain sequential write and read of the same bytes with
numpy.tofile / numpy.fromfile, so that the engine's overhead over the file system shows; one move and one end_batch for
scale; and the device time of the merge kernel alone (torch.profiler around one more merge).  The page cache is not
dropped (that needs root): reads may come from memory, and a write is timed to its fsync.  Prints one JSON line per variant, with the card name and power limit.
Usage: python scripts/bench_checkpoint.py --dir DIR [--config c2] [--reps 3]"""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.mesh import kuhn_box
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

ap = argparse.ArgumentParser()
ap.add_argument("--dir", required=True, help="directory for the checkpoint files (removed afterwards)")
ap.add_argument("--config", default="c2")
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()
os.makedirs(args.dir, exist_ok=True)
dev = torch.device("cuda", 0)
card = torch.cuda.get_device_name(dev)
try:
    power = float(subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                          text=True, timeout=30).strip())
except Exception:
    power = None

cfg = CONFIGS[args.config]
cells = cfg["cells"]
n = cfg["particles"]
coords, t2v = kuhn_box(*cells)
E = len(t2v)
zc = coords[t2v].mean(axis=1)[:, 2]
slabs = np.minimum(((zc - zc.min()) / (zc.max() - zc.min()) * 64).astype(np.int32), 63)
VARIANTS = [("scores1", 1, 0, False, None), ("scores8_time16_collision_slabs64", 8, 16, True, slabs)]


def median(f, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def plain_rates(nbytes, reps):
    """sequential write (to fsync) and read of nbytes with numpy.tofile / fromfile, in the same directory"""
    a = np.ones(nbytes // 8)
    p = os.path.join(args.dir, "plain.bin")

    def w():
        with open(p, "wb") as f:
            a.tofile(f)
            f.flush()
            os.fsync(f.fileno())

    tw = median(w, reps)
    tr = median(lambda: np.fromfile(p, dtype=np.float64), reps)
    os.remove(p)
    return tw, tr


for label, ns, nt, coll, rmap in VARIANTS:
    def make():
        e = PumiTally.from_arrays(coords, t2v, n, device=0)
        e.set_scores(ns)
        if nt:
            e.set_time_bins(np.linspace(0.0, 16.0, nt + 1))
        e.set_collision_estimator(coll)
        e.set_batch_statistics(True)
        e.set_source_normalization(3)
        if rmap is not None:
            e.set_regions(rmap)
        return e

    eng = make()
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

    def move():
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        if nt:
            eng.move_device_timed(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), times.data_ptr(),
                                  speeds.data_ptr(), resp.data_ptr() if resp is not None else None, None, s)
        else:
            eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
        if coll:
            eng.tally_collisions_at_particles_device(collided, cw, resp, None, times if nt else None)
        torch.cuda.synchronize()

    t_move = median(move, 1)
    for _ in range(2):  # two batches folded: statistics with errors
        move()
        eng.end_batch()
    move()
    t_end = median(eng.end_batch, 1)
    end_path = os.path.join(args.dir, f"{label}_end.ckpt")
    mid_path = os.path.join(args.dir, f"{label}_mid.ckpt")
    t_save_end = median(lambda: eng.save_checkpoint(end_path), args.reps)
    b_end = os.path.getsize(end_path)
    move()
    t_save_mid = median(lambda: eng.save_checkpoint(mid_path), args.reps)
    b_mid = os.path.getsize(mid_path)
    other = make()
    t_load = median(lambda: other.load_checkpoint(end_path), args.reps)
    t_merge = median(lambda: other.merge_checkpoint(end_path), args.reps)
    # merge kernel alone: CUDA events on the default stream cannot see the engine's own stream, so time the kernel
    # with torch.profiler around one merge
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        other.merge_checkpoint(end_path)
        torch.cuda.synchronize()
    kern_us = sum(ev.device_time_total for ev in prof.key_averages() if "batch_merge_kernel" in ev.key)
    del other
    tw, tr = plain_rates(b_end, args.reps)
    os.remove(end_path)
    os.remove(mid_path)
    gb = lambda b, t: b / t / 1e9  # noqa: E731
    merge_bytes = 48 * (b_end // 16)  # 48 B per merged double (six 8-byte streams), about half the file's doubles
    print(json.dumps({
        "config": args.config, "variant": label, "card": card, "power_limit_w": power,
        "bytes_batch_end": b_end, "bytes_mid_batch": b_mid,
        "save_batch_end_s": t_save_end, "save_batch_end_gbs": gb(b_end, t_save_end),
        "save_mid_batch_s": t_save_mid, "save_mid_batch_gbs": gb(b_mid, t_save_mid),
        "load_s": t_load, "load_gbs": gb(b_end, t_load), "merge_s": t_merge, "merge_gbs": gb(b_end, t_merge),
        "plain_write_s": tw, "plain_write_gbs": gb(b_end, tw), "plain_read_s": tr, "plain_read_gbs": gb(b_end, tr),
        "save_vs_plain_write": tw / t_save_end,
        "merge_kernel_ms": kern_us / 1e3, "merge_kernel_gbs": merge_bytes / (kern_us * 1e-6) / 1e9 if kern_us else None,
        "move_s": t_move, "end_batch_s": t_end}), flush=True)
    del eng
    torch.cuda.empty_cache()
