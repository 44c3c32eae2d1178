"""Instruction shape of the binned walk's cooperative record fetch (CPU only: walk_kernels.cu cross-compiled for
sm_90a).

coop_plane_step() issues a warp's record copies as one run: the (element, face) slots of a lane group are read with
four 128-bit shared loads, and each of the eight copies goes out under a predicate, not behind a branch.  With the
slots read one round at a time behind two divergent branches, the fetch of the plain binned kernel (variant 16) took
332 instruction slots from the slot store to the wait; these tests keep it a straight run well under that."""
import os
import re
import subprocess

import pytest

from pumiumtally_b200 import build as pbuild

# walk_persist_kernel<128, kFetchCoopL1, 5, 8, 1 (gather), NS 0, TM false, MO false>: variant 16's plain kernel
PLAIN_V16 = "19walk_persist_kernelILi128ELi5ELi5ELi8ELi1ELi0ELb0ELb0E"
# slots from the store of the (element, face) slot to the DEPBAR of cp.async.wait_all, fast path
SPAN_BUDGET = 140
_PRED = r"(?:@!?U?P\w+\s+)?"


@pytest.fixture(scope="module")
def fetch(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("sass_coop") / "walk_kernels.o")
    subprocess.run([pbuild._nvcc(), *pbuild.NVCC_FLAGS, "-c", os.path.join(pbuild.CSRC, "walk_kernels.cu"), "-o", out],
                   check=True, capture_output=True)
    cuobjdump = os.path.join(os.path.dirname(pbuild._nvcc()), "cuobjdump")
    text = subprocess.run([cuobjdump, "-sass", out], check=True, capture_output=True, text=True).stdout
    bodies = [f for f in text.split("Function : ")[1:] if PLAIN_V16 in f.split("\n", 1)[0]]
    assert len(bodies) == 1, "plain variant-16 kernel not found"
    ins = [(int(a, 16), t.strip()) for a, t in re.findall(r"^\s+/\*([0-9a-f]{4,})\*/\s+([^;]*);", bodies[0], re.M)]
    copies = [i for i, (_, t) in enumerate(ins) if re.match(_PRED + r"LDGSTS\.E\.128 ", t)]
    return ins, copies


def test_eight_predicated_record_copies(fetch):
    ins, copies = fetch
    assert len(copies) == 8, [ins[i][1] for i in copies]  # one per round; the fetch is not duplicated


def test_copies_are_not_behind_per_round_branches(fetch):
    ins, copies = fetch
    flow = [i for i in range(copies[0], copies[-1] + 1) if re.match(_PRED + r"(BRA|BSSY|BSYNC|WARPSYNC)", ins[i][1])]
    # no divergent region opens or closes among the copies: the only branches are the exit before the last round
    # (at most 28 active lanes), after the seventh copy, and they jump past the eighth
    assert all(re.match(_PRED + r"BRA ", ins[i][1]) for i in flow), [ins[i][1] for i in flow]
    assert all(i > copies[-2] for i in flow), [ins[i][1] for i in flow]
    assert all(int(ins[i][1].split()[-1], 16) > ins[copies[-1]][0] for i in flow), [ins[i][1] for i in flow]


def test_fetch_span_within_budget(fetch):
    ins, copies = fetch
    store = max(i for i in range(copies[0]) if re.match(_PRED + r"STS\.64 ", ins[i][1]))
    wait = min(i for i in range(copies[-1], len(ins)) if re.match(_PRED + r"DEPBAR", ins[i][1]))
    slot_reads = [t for _, t in ins[store:copies[0]] if re.match(_PRED + r"LDS\.128 ", t)]
    assert len(slot_reads) == 4, slot_reads
    assert wait - store + 1 <= SPAN_BUDGET, wait - store + 1
