"""The binning key's arithmetic in the SASS of bin_count_kernel (CPU only: bin_kernels.cu cross-compiled for sm_90a).

tests/test_gpu_bin_kernels.py compares every key with numpy's float64 arithmetic, which rounds each operation on its
own.  That holds only while the kernel's key arithmetic is unfused: (x - x0) * inv_h and 0.5 * (x + mx) as a DADD
and a DMUL each.  The only DFMAs allowed are those of all_finite, whose products are 0 * v: +-0 or NaN, so fusing them
cannot change the outcome."""
import os
import re
import subprocess

import pytest

from pumiumtally_b200 import build as pbuild


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("sass_bin") / "bin_kernels.o")
    subprocess.run([pbuild._nvcc(), *pbuild.NVCC_FLAGS, "-c", os.path.join(pbuild.CSRC, "bin_kernels.cu"), "-o", out],
                   check=True, capture_output=True)
    cuobjdump = os.path.join(os.path.dirname(pbuild._nvcc()), "cuobjdump")
    text = subprocess.run([cuobjdump, "-sass", out], check=True, capture_output=True, text=True).stdout
    return {f.split("\n", 1)[0].strip(): f for f in text.split("Function : ")[1:]}


def _instructions(body, op):
    return re.findall(rf"^\s+/\*[0-9a-f]+\*/\s+(?:@!?P\w+\s+)?({op}\S*)\s+([^;]*);", body, re.M)


def test_bin_count_kernel_fuses_nothing_but_the_finiteness_test(sass):
    names = [n for n in sass if "bin_count_kernel" in n]
    assert len(names) == 1, list(sass)
    body = sass[names[0]]
    dfma = _instructions(body, "DFMA")
    assert len(dfma) == 2, dfma  # all_finite(mx, my, mz): 0 * my, then 0 * mx + _ and 0 * mz + _
    for _, ops in dfma:
        assert "RZ" in [o.strip() for o in ops.split(",")[1:3]], ops  # a multiplicand is zero
    assert len(_instructions(body, "DMUL")) == 1 + 3 + 3  # 0 * my, 0.5 * (x + mx), f * inv_h
    assert len(_instructions(body, "DADD")) == 3 + 3  # x + mx, x - x0
    assert len(_instructions(body, r"F2I\.F64\.TRUNC")) == 3
