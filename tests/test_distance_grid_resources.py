"""The banded frame-distance grid kernel (goslam_frame_distance_grid) keeps everything in registers and shared memory:
no stack frame, no local memory and no local loads or stores in its sm_90a SASS.  Its row search and both pair
distances are straight-line integer and float code; a spill there would be paid once per frame pair."""
import re
import shutil
import subprocess

import pytest

KERNEL = "frame_distance_grid_kernel"


def _cuobjdump(flag):
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    return subprocess.run(["cuobjdump", flag, _lib.lib_path()], capture_output=True, text=True).stdout


def test_grid_kernel_has_no_stack_or_local_memory():
    lines = _cuobjdump("-res-usage").splitlines()
    idx = [i for i, l in enumerate(lines) if "Function" in l and KERNEL in l]
    assert len(idx) == 1, idx
    usage = lines[idx[0] + 1]
    stack = re.search(r"\bSTACK:(\d+)\b", usage)
    local = re.search(r"\bLOCAL:(\d+)\b", usage)
    assert stack and local, usage
    assert int(stack.group(1)) == 0 and int(local.group(1)) == 0, usage


def test_grid_kernel_issues_no_local_loads_or_stores():
    parts = re.split(r"\n\s*Function : ", _cuobjdump("-sass"))[1:]
    bodies = [p.partition("\n")[2] for p in parts if KERNEL in p.partition("\n")[0]]
    assert len(bodies) == 1
    ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)", bodies[0])
    assert ops, "no SASS parsed"
    local = [o for o in ops if o.split(".")[0] in ("LDL", "STL")]
    assert not local, len(local)
