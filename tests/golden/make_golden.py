"""Regenerates the committed golden fixtures.

t1_known_answers.json is transcribed from the reference's own known-answer test
(test/test_pumi_tally_impl_methods.cpp of the reference; line numbers inside the file) -- it is not
generated, and neither is reference_facade_symbols.json: the undefined symbols of the
tests/test_abi_symbols.py translation unit compiled against the reference's PumiTally.h.  c1_oracle.npz is produced here by the CPU oracle (oracle/umtally_oracle.c), which is
pinned against t1_known_answers.json and the brute-force integrator by tests/test_oracle_golden.py.

    python tests/golden/make_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle.oracle import OraclePumiTally  # noqa: E402
from pumiumtally_b200.mesh import kuhn_box  # noqa: E402
from pumiumtally_b200.workload import CONFIGS, SyntheticWorkload  # noqa: E402


def c1_case(steps=3):
    cfg = CONFIGS["c1"]
    coords, t2v = kuhn_box(*cfg["cells"])
    n = cfg["particles"]
    wl = SyntheticWorkload(box=tuple(float(c) for c in cfg["cells"]), num_particles=n, mean_length=cfg["mean_length"])
    return coords, t2v, n, wl, steps


def main():
    coords, t2v, n, wl, steps = c1_case()
    orc = OraclePumiTally(coords, t2v, n, per_particle=False)  # reference-shaped schedule
    orc.CopyInitialPosition(wl.initial_positions().reshape(-1))
    elem_after_init = orc.elem_ids
    for _ in range(steps):
        o, d, f, w = wl.next_step()
        orc.MoveToNextLocation(o.reshape(-1), d.reshape(-1), f, w)
    np.savez_compressed(os.path.join(HERE, "c1_oracle.npz"), flux=orc.flux, elem_after_init=elem_after_init,
                        elem_final=orc.elem_ids, positions_final=orc.positions, n_segments=orc.n_segments,
                        n_tracks=orc.n_tracks, steps=steps)
    print("wrote c1_oracle.npz:", orc.n_segments, "segments, flux sum", orc.flux.sum())


if __name__ == "__main__":
    main()
