"""The fused conv1 kernel holds conv1_2's 128 accumulator registers and its weight fragments next to conv1_1's passes
within the 168 registers it is compiled for: a spill would put local-memory traffic into the loop that feeds the tensor
cores.  Reads the resource usage of the BUILT library with cuobjdump (no GPU)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "openibl_b200", "lib", "libiblb200.so")


def test_conv1_fused_kernel_does_not_spill():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is missing")
    out = subprocess.run([exe, "-res-usage", LIB], capture_output=True, text=True, timeout=600).stdout
    usage = re.findall(r"Function (\S*conv1_fused_tc_kernel\S*):\s*\n\s*(REG:.*)", out)
    assert usage, "conv1_fused_tc_kernel is not in the library"
    for name, line in usage:
        fields = dict(re.findall(r"(\w+):(\d+)", line))
        assert fields["STACK"] == "0" and fields["LOCAL"] == "0", (name, line)
