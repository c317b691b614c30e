"""The issue-path discipline of DESIGN 5 ("The issue path") as a regression test on the BUILT library: in the product
kernels no TMA instruction may sit in one of the per-instruction issue loops ptxas builds around them when they are
not behind elect.sync (`R2UR.BROADCAST` of operands, `BRA.U.ANY` back-edges), and the Hopper warpgroup-MMA and TMA
opcodes must be there at all.  Needs only cuobjdump (no GPU)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "openibl_b200", "lib", "libiblb200.so")

PRODUCT_KERNELS = ("conv3x3_tc_kernel", "conv1_fused_tc_kernel", "conv1_1_tc_kernel", "netvlad_tc_kernel", "gemm_f16_top16_kernel",
                   "gemm_tc_kernel", "conv_wgrad_tc_kernel")
NO_TMA = ("conv1_1_tc_kernel",)   # builds its operands in shared memory (a 3-channel row is too short for TMA)


@pytest.fixture(scope="module")
def sass_counts():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is missing")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600).stdout
    counts, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            counts.setdefault(fn, {})
            continue
        if fn is None:
            continue
        for op in ("HGMMA", "UTMALDG", "R2UR.BROADCAST", "BRA.U.ANY"):
            if re.search(r"\b" + re.escape(op), line):
                counts[fn][op] = counts[fn].get(op, 0) + 1
    return counts


def test_product_kernels_are_wgmma_tma_code(sass_counts):
    for name in PRODUCT_KERNELS:
        variants = {k: v for k, v in sass_counts.items() if name in k}
        assert variants, f"{name} is not in the library"
        for k, c in variants.items():
            assert c.get("HGMMA", 0) > 0 and (name in NO_TMA or c.get("UTMALDG", 0) > 0), (k, c)


def test_no_per_instruction_issue_loops_in_product_kernels(sass_counts):
    for name in PRODUCT_KERNELS:
        for k, c in sass_counts.items():
            if name in k:
                assert c.get("BRA.U.ANY", 0) == 0, (k, c)
                assert c.get("R2UR.BROADCAST", 0) <= 1, (k, c)
