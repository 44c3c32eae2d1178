"""Register budget of the detector void's kernels (CPU only: ptxas reports it at compile time).

detector_kernels.cu is compiled for sm_90a with -Xptxas -v.  The two void kernels (located, at the particles), each with
the shared-memory and the warp aggregation, must be in the report with no stack frame and no spills.  Their register
counts are pinned: the entry search shares the walk's registers (one search site in detector_ray<true>), and a change
in either shows here first.  __launch_bounds__(128, 3) lets them take up to 170 registers rather than spill, three 128-thread blocks per SM."""
import os
import re
import subprocess

import pytest

from pumiumtally_b200 import build as pbuild

KERNEL = re.compile(r"detect_(located|particles)_void_kernelILb([01])E")
REGISTERS = {"located": 142, "particles": 144}


@pytest.fixture(scope="module")
def budget(tmp_path_factory):
    out = tmp_path_factory.mktemp("budget_void")
    cmd = [pbuild._nvcc(), *pbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(pbuild.CSRC, "detector_kernels.cu"),
           "-o", str(out / "detector_kernels.o")]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True)
    found = {}
    for block in re.split(r"Compiling entry function '", log.stdout + log.stderr)[1:]:
        m = KERNEL.search(block.split("'", 1)[0])
        if not m:
            continue
        s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        r = re.search(r"Used (\d+) registers", block)
        found[(m.group(1), m.group(2) == "1")] = tuple(int(g) for g in s.groups()) + (int(r.group(1)),)
    return found


KEYS = [(k, s) for k in ("located", "particles") for s in (False, True)]


def test_every_void_kernel_reported(budget):
    assert sorted(budget) == sorted(KEYS)


@pytest.mark.parametrize("key", KEYS, ids=lambda k: f"{k[0]}-smem{int(k[1])}")
def test_void_kernel_has_no_stack_no_spills_and_its_registers(budget, key):
    assert budget[key] == (0, 0, 0, REGISTERS[key[0]]), budget[key]
