"""Cost of cosine bins on the face currents: a device-resident plain move with face currents and C cosine bins (equal
bins over [0, 1]) against the same move with face currents and no cosine bins, one engine each, the two alternated move
by move in this process (same batches, same positions before every move), timed with per-move CUDA events.  Prints one
JSON line per C: ms per move of both and their ratio, the kernel that ran, the current block's bytes against the L2,
and the card name and power limit.
Usage: python scripts/bench_current_cosines.py [--config c2] [--cosines 1,8,64] [--steps 10] [--warmup 3]"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

ap = argparse.ArgumentParser()
ap.add_argument("--config", default="c2")
ap.add_argument("--cosines", default="1,8,64", help="comma-separated cosine-bin counts, 1..64")
ap.add_argument("--particles", type=int, default=0, help="override the config's particle count")
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--variant", type=int, default=-1)
args = ap.parse_args()
counts = [int(c) for c in args.cosines.split(",")]
if not all(1 <= c <= 64 for c in counts) or args.steps < 1:
    raise SystemExit("bench_current_cosines.py: --cosines must be 1..64 each and --steps at least 1")

cfg = CONFIGS[args.config]
cells = cfg["cells"]
spec = f"box:{cells[0]},{cells[1]},{cells[2]}"
n, steps, warmup = args.particles or cfg["particles"], args.steps, max(args.warmup, 0)
dev = torch.device("cuda", 0)
stream = torch.cuda.current_stream().cuda_stream
card = torch.cuda.get_device_name(dev)
try:
    power = float(subprocess.check_output(
        ["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], text=True, timeout=30).strip())
except Exception:
    power = None
l2 = torch.cuda.get_device_properties(dev).L2_cache_size


def new_engine(C):
    e = PumiTally.from_spec(spec, n, device=0)
    e.set_option("variant", args.variant)  # -1 = the engine's own choice for this mesh
    e.set_face_currents(True)
    if C:
        e.set_current_cosine_bins(np.linspace(0.0, 1.0, C + 1))
    return e


for C in counts:
    wl = SyntheticWorkload(box=tuple(float(c) for c in cells), num_particles=n, mean_length=cfg["mean_length"],
                           mu_min=cfg["mu_min"], backend="torch", device=dev)
    init = wl.initial_positions().contiguous()
    mu, base = new_engine(C), new_engine(0)
    for e in (mu, base):
        e.copy_initial_position_device(init.data_ptr(), stream)
    ms = {"cosines": 0.0, "no_cosines": 0.0}
    for k in range(warmup + steps):
        o, d, f, w = (x.contiguous() for x in wl.next_step())
        for name, e in (("cosines", mu), ("no_cosines", base)):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            e.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), stream)
            ev1.record()
            torch.cuda.synchronize()
            if k >= warmup:
                ms[name] += ev0.elapsed_time(ev1)
    E = mu.num_elements
    # the sums agree: every crossing lands in one of the bins of [0, 1]
    a, b = mu.face_current_results(0).sum(axis=2), base.face_current_results(0)
    agree = bool(np.allclose(a, b, rtol=1e-12, atol=1e-12 * np.abs(b).max()))
    out = {"config": args.config, "particles": n, "steps": steps, "cosine_bins": C, "move": "plain, device pointers",
           "timing": "per-move CUDA events, moves with and without cosine bins alternated on the same batches",
           "cosines_ms_per_move": ms["cosines"] / steps, "no_cosines_ms_per_move": ms["no_cosines"] / steps,
           "ratio": ms["cosines"] / ms["no_cosines"], "variant": mu.get_option("variant"),
           "walk_blocks_per_sm": {"cosines": mu.get_option("walk_blocks_per_sm"),
                                  "no_cosines": base.get_option("walk_blocks_per_sm")},
           "sums_agree": agree,
           "byte_model": {"current_block_bytes": C * E * 4 * 8, "no_cosine_block_bytes": E * 4 * 8, "l2_bytes": l2},
           "card": card, "power_limit_w": power}
    print(json.dumps(out), flush=True)
    del mu, base
