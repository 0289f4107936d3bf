"""The bundle-adjustment kernels keep their per-pixel reductions in registers: the 32-value warp
transpose-reduction and the Schur flush index their arrays with compile-time constants only, so the
linearise and system kernels have no stack frame and never touch local memory (LDL / STL).

The cooperative kernel also retracts the poses, and CUDA's sinf / cosf keep a 28-byte scratch array
for their Payne-Hanek slow path (|x| > 105615, never reached by a pose increment).  That array is the
only stack the kernel may have; the reductions used to put 288 bytes there."""
import re
import shutil
import subprocess

import pytest

NO_STACK = ("ba_linearize_kernel", "ba_system_kernel")
PERSISTENT = "ba_persistent_kernel"
TRIG_SLOW_PATH_STACK = 32


def _cuobjdump(flag):
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    return subprocess.run(["cuobjdump", flag, _lib.lib_path()], capture_output=True, text=True).stdout


def _usage(kernel):
    lines = _cuobjdump("-res-usage").splitlines()
    idx = [i for i, l in enumerate(lines) if "Function" in l and kernel in l]
    assert len(idx) == 1, idx
    usage = lines[idx[0] + 1]
    stack = re.search(r"\bSTACK:(\d+)\b", usage)
    local = re.search(r"\bLOCAL:(\d+)\b", usage)
    assert stack and local, usage
    return int(stack.group(1)), int(local.group(1)), usage


@pytest.mark.parametrize("kernel", NO_STACK)
def test_ba_kernel_has_no_stack_or_local_memory(kernel):
    stack, local, usage = _usage(kernel)
    assert stack == 0 and local == 0, usage


@pytest.mark.parametrize("kernel", NO_STACK)
def test_ba_kernel_issues_no_local_loads_or_stores(kernel):
    parts = re.split(r"\n\s*Function : ", _cuobjdump("-sass"))[1:]
    bodies = [p.partition("\n")[2] for p in parts if kernel in p.partition("\n")[0]]
    assert len(bodies) == 1
    ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)", bodies[0])
    local = [o for o in ops if o.split(".")[0] in ("LDL", "STL")]
    assert not local, (kernel, len(local))


def test_persistent_kernel_stack_is_only_the_trig_slow_path():
    stack, local, usage = _usage(PERSISTENT)
    assert stack <= TRIG_SLOW_PATH_STACK and local == 0, usage
