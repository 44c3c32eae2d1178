"""Register budget of the persistent walk kernels (CPU only: ptxas reports it at compile time).

walk_kernels.cu is compiled for sm_90a with -Xptxas -v.  The plain product persistent kernels (streaming 8,
binned 16, packed 24) must not spill: their crossing loop is bound by the L1TEX pipe, and spill traffic goes
through the same pipe and takes L1 from the tet records.  Their scored, timed and moment instantiations may
spill a little (the score loop's address arithmetic), but never more than they did before the scheduling
state moved to shared memory (DESIGN section 4.7)."""
import os
import re
import subprocess

import pytest

from pumiumtally_b200 import build as pbuild

# (fetch mode, staging) -> product variant: walk_persist_kernel<128, FETCH, MINB, 8, STAGING, NS, TM, MO>
PRODUCT = {(1, 0): 8, (5, 1): 16, (1, 2): 24}

# spill bytes (stores, loads) of the scored, timed and moment instantiations before the change:
# (variant, timed, moments) -> limit
SPILL_LIMIT = {
    (8, False, False): (100, 132), (8, False, True): (92, 132), (8, True, False): (140, 212), (8, True, True): (160, 196),
    (16, False, False): (104, 136), (16, False, True): (96, 140), (16, True, False): (136, 196), (16, True, True): (156, 212),
    (24, False, False): (80, 120), (24, False, True): (88, 128), (24, True, False): (112, 156), (24, True, True): (132, 180),
}

KERNEL = re.compile(r"walk_persist_kernelILi128ELi(\d+)ELi(\d+)ELi8ELi(\d+)ELi(\d+)ELb([01])ELb([01])E")


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
        found[(variant, ns, bool(tm), bool(mo))] = dict(minb=minb, regs=int(r.group(1)), stack=int(s.group(1)),
                                                        stores=int(s.group(2)), loads=int(s.group(3)))
    return found


def test_every_product_instantiation_reported(budget):
    for v in PRODUCT.values():
        assert (v, 0, False, False) in budget, f"variant {v}: plain kernel not found in the ptxas report"
        for (lv, tm, mo) in SPILL_LIMIT:
            if lv == v:
                assert (v, 8, tm, mo) in budget, f"variant {v} timed={tm} moments={mo}: not found"


@pytest.mark.parametrize("variant", sorted(PRODUCT.values()))
def test_plain_product_kernel_does_not_spill(budget, variant):
    k = budget[(variant, 0, False, False)]
    assert k["stores"] == 0 and k["loads"] == 0 and k["stack"] == 0, f"variant {variant}: {k}"
    # the launch bound still holds the blocks per SM it promises: 65536 registers / (MINB * 128 lanes)
    assert k["regs"] <= 65536 // (k["minb"] * 128), k


@pytest.mark.parametrize("key", sorted(SPILL_LIMIT), ids=lambda k: f"v{k[0]}-timed{int(k[1])}-moments{int(k[2])}")
def test_tallied_instantiation_spills_no_more_than_before(budget, key):
    variant, tm, mo = key
    k = budget[(variant, 8, tm, mo)]
    stores, loads = SPILL_LIMIT[key]
    assert k["stores"] <= stores and k["loads"] <= loads, f"{key}: {k} against ({stores}, {loads})"
