"""The correlation build keeps its accumulators and epilogue values in registers: any local memory
(spill slots or stack) puts L2 round trips inside the per-tile loop of an HBM-write-bound kernel."""
import re
import shutil
import subprocess

import pytest


def test_corr_build_tc_kernel_uses_no_local_memory():
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout
    lines = out.splitlines()
    idx = [i for i, l in enumerate(lines) if "Function" in l and "corr_build_tc_kernel" in l]
    assert len(idx) == 1, "expected one corr_build_tc_kernel in the library, found %d" % len(idx)
    usage = lines[idx[0] + 1]
    assert re.search(r"\bSTACK:0\b", usage), usage
    assert re.search(r"\bLOCAL:0\b", usage), usage
