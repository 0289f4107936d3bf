"""The tiled correlation build writes its pyramid through the TMA engine: the consumer warpgroups stage the
volume in shared memory (stmatrix / STS) and issue no global stores of their own, and every shared-memory
access is shared-typed (no generic LD.E / ST.E, which cost an address-space check per access)."""
import re
import shutil
import subprocess

import pytest


def _functions(text):
    """{function name: its SASS} from `cuobjdump -sass`."""
    out = {}
    for part in re.split(r"\n\s*Function : ", text)[1:]:
        name, _, body = part.partition("\n")
        out[name.strip()] = body
    return out


def _opcodes(body):
    return re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)", body)


@pytest.fixture(scope="module")
def build_kernels():
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.lib_path()], capture_output=True, text=True).stdout
    fns = {k: v for k, v in _functions(sass).items() if "corr_build_tc_kernel" in k}
    assert len(fns) == 1, sorted(fns)          # one kernel, one (tiled) output layout
    return fns


def test_corr_build_is_one_instance_without_local_memory():
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    lines = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout.splitlines()
    idx = [i for i, l in enumerate(lines) if "Function" in l and "corr_build_tc_kernel" in l]
    assert len(idx) == 1
    for i in idx:
        assert re.search(r"\bSTACK:0\b", lines[i + 1]) and re.search(r"\bLOCAL:0\b", lines[i + 1]), lines[i + 1]


def test_corr_build_stores_only_through_tma(build_kernels):
    (body,) = build_kernels.values()
    ops = [o.split(".")[0] for o in _opcodes(body)]
    assert "UTMASTG" in ops and "STSM" in ops
    assert "STG" not in ops


def test_corr_build_has_no_generic_shared_memory_access(build_kernels):
    for name, body in build_kernels.items():
        ops = _opcodes(body)
        generic = [o for o in ops if o in ("LD", "ST") or o.startswith(("LD.", "ST."))]
        assert not generic, (name, generic[:5])
