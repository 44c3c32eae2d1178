"""Register budget of the point-detector kernels (CPU only: ptxas reports it at compile time).

detector_kernels.cu is compiled for sm_90a with -Xptxas -v.  Both kernels (located, at the particles), each with the
shared-memory and the warp aggregation, must be in the report with no stack frame and no spills."""
import os
import re
import subprocess

import pytest

from pumiumtally_b200 import build as pbuild

KERNEL = re.compile(r"detect_(located|particles)_kernelILb([01])E")


@pytest.fixture(scope="module")
def budget(tmp_path_factory):
    out = tmp_path_factory.mktemp("budget")
    cmd = [pbuild._nvcc(), *pbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(pbuild.CSRC, "detector_kernels.cu"),
           "-o", str(out / "detector_kernels.o")]
    log = subprocess.run(cmd, check=True, capture_output=True, text=True)
    found = {}
    for block in re.split(r"Compiling entry function '", log.stdout + log.stderr)[1:]:
        m = KERNEL.search(block.split("'", 1)[0])
        if not m:
            continue
        s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        found[(m.group(1), m.group(2) == "1")] = tuple(int(g) for g in s.groups())
    return found


def test_every_detector_kernel_reported(budget):
    assert sorted(budget) == sorted((k, s) for k in ("located", "particles") for s in (False, True))


@pytest.mark.parametrize("key", [(k, s) for k in ("located", "particles") for s in (False, True)],
                         ids=lambda k: f"{k[0]}-smem{int(k[1])}")
def test_detector_kernel_has_no_stack_and_no_spills(budget, key):
    assert budget[key] == (0, 0, 0), budget[key]
