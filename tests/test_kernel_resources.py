"""The tensor-core layer kernels keep their working set in registers: no instantiation of tc_conv3x3_kernel has a stack
frame (spilled accumulators cost local-memory traffic on every tap and every epilogue)."""
import re
import shutil
import subprocess

import pytest


def test_tc_layer_kernels_have_no_stack_frame(w2x):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    r = subprocess.run(["cuobjdump", "-res-usage", w2x.lib_path()], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump could not read the library")
    found = re.findall(r"Function (\S*tc_conv3x3_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", r.stdout)
    assert len(found) == 36, len(found)                   # 9 shapes x (plain, fused last layer) x (f16x3, f16 + 2 x e4m3)
    stacked = [(name, int(stack)) for name, _, stack in found if int(stack) != 0]
    assert not stacked, stacked
