"""The encoder kernels keep their accumulators and staged operands in registers: no spill slots or stack frames."""
import re
import shutil
import subprocess

import pytest


def test_encoder_kernels_use_no_local_memory():
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout
    lines = out.splitlines()
    idx = [i for i, l in enumerate(lines) if "Function" in l and "encoder_" in l and "_kernel" in l]
    assert len(idx) >= 6, "encoder kernels not found in the library"
    for i in idx:
        usage = lines[i + 1]
        assert re.search(r"\bSTACK:0\b", usage), (lines[i], usage)
        assert re.search(r"\bLOCAL:0\b", usage), (lines[i], usage)
