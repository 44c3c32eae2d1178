"""Experiment: walk-kernel time for random vs spatially sorted particle order, per variant.
Usage: python scripts/exp_sorted.py "<mode>:<variant> ..."   e.g. "random:4 sorted_cell:4 random:16" """
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pumiumtally_b200.tally import PumiTally
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload

cfg = CONFIGS["c2"]; cells = cfg["cells"]; n = cfg["particles"]
box = tuple(float(c) for c in cells)
dev = torch.device("cuda", 0)
runs = (sys.argv[1] if len(sys.argv) > 1 else "random:4 sorted_cell:4").split()
for run in runs:
    mode, variant = run.split(":"); variant = int(variant)
    wl = SyntheticWorkload(box=box, num_particles=n, mean_length=cfg["mean_length"], backend="torch", device=dev)
    init = wl.initial_positions()
    o, d, f, w = wl.next_step()
    if mode != "random":
        c = init.floor().long()
        key = (c[:, 2] * cells[1] + c[:, 1]) * cells[0] + c[:, 0]
        perm = torch.argsort(key)
        init, o, d, f, w = (x[perm].contiguous() for x in (init, o, d, f, w))
    eng = PumiTally.from_spec(f"box:{cells[0]},{cells[1]},{cells[2]}", n, device=0)
    eng.set_option("variant", variant)
    s = torch.cuda.current_stream().cuda_stream
    eng.copy_initial_position_device(init.contiguous().data_ptr(), s)
    torch.cuda.synchronize()
    st0 = eng.stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    eng.move_device(o.data_ptr(), d.data_ptr(), f.data_ptr(), w.data_ptr(), s)
    e1.record(); torch.cuda.synchronize()
    st1 = eng.stats()
    segs = st1["segments"] - st0["segments"]
    ms = e0.elapsed_time(e1)
    print(json.dumps({"mode": mode, "variant": variant, "ms": round(ms, 3), "gseg_s": round(segs / ms / 1e6, 2),
                      "frac": round((128 * segs + 89 * (st1["tracks"] - st0["tracks"])) / (ms * 1e-3) / 3350e9, 3)}), flush=True)
    del eng
