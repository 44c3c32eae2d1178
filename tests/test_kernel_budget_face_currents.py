"""Register budget of the persistent walk kernels with face currents (CPU only: ptxas reports it at compile time).

walk_kernels.cu is compiled for sm_90a with -Xptxas -v.  Every face-current instantiation of the product kernels
(streaming 8, binned 16, packed 24; timed and moments on or off) must be in the report, under its own name
walk_persist_current_kernel, and must spill no more than it did when it was added: a crossing costs one more
reduction, and its weight lives in a shared-memory lane slot, not in a register."""
import os
import re
import subprocess

import pytest

from pumiumtally_b200 import build as pbuild

PRODUCT = {(1, 0): 8, (5, 1): 16, (1, 2): 24}

# spill bytes (stores, loads) when the face currents were added: (variant, timed, moments) -> limit
SPILL_LIMIT = {
    (8, False, False): (0, 0), (8, False, True): (0, 0), (8, True, False): (28, 44), (8, True, True): (76, 100),
    (16, False, False): (16, 24), (16, False, True): (16, 24), (16, True, False): (20, 28), (16, True, True): (28, 40),
    (24, False, False): (16, 24), (24, False, True): (16, 24), (24, True, False): (40, 52), (24, True, True): (32, 48),
}

KERNEL = re.compile(r"walk_persist_current_kernelILi128ELi(\d+)ELi(\d+)ELi8ELi(\d+)ELi(\d+)ELb([01])ELb([01])E")


@pytest.fixture(scope="module")
def budget(tmp_path_factory):
    out = tmp_path_factory.mktemp("budget")
    cmd = [pbuild._nvcc(), *pbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(pbuild.CSRC, "walk_kernels.cu"),
           "-o", str(out / "walk_kernels.o")]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True)
    text = log.stdout + log.stderr
    found = {}
    for block in re.split(r"Compiling entry function '", text)[1:]:
        m = KERNEL.search(block.split("'", 1)[0])
        if not m:
            continue
        fetch, minb, staging, ns, tm, mo = (int(g) for g in m.groups())
        variant = PRODUCT.get((fetch, staging))
        if variant is None:
            continue
        s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        r = re.search(r"Used (\d+) registers", block)
        found[(variant, bool(tm), bool(mo))] = dict(ns=ns, minb=minb, regs=int(r.group(1)), stack=int(s.group(1)),
                                                    stores=int(s.group(2)), loads=int(s.group(3)))
    return found


def test_every_current_instantiation_reported(budget):
    assert sorted(budget) == sorted(SPILL_LIMIT)
    for k in budget.values():
        assert k["ns"] == 8


@pytest.mark.parametrize("key", sorted(SPILL_LIMIT), ids=lambda k: f"v{k[0]}-timed{int(k[1])}-moments{int(k[2])}")
def test_current_instantiation_spills_no_more_than_when_added(budget, key):
    k = budget[key]
    stores, loads = SPILL_LIMIT[key]
    assert k["stores"] <= stores and k["loads"] <= loads, f"{key}: {k} against ({stores}, {loads})"
    # the launch bound still holds the blocks per SM it promises: 65536 registers / (MINB * 128 lanes)
    assert k["regs"] <= 65536 // (k["minb"] * 128), k
