"""CPU checks of the trajectory-evaluation entry points (goslam_ape_workspace_bytes / goslam_ape_sim3): the workspace
query, argument validation before any CUDA call, the failure without a device, and the kernels' resources."""
import ctypes
import re
import shutil
import subprocess
import threading

import pytest

# every kernel but the one-thread Umeyama solve, whose indexed 3x3 arrays take stack slots as the ICP's do (no spills:
# ptxas -v reports none for any of them)
KERNELS = ("ape_init_kernel", "ape_keep_kernel", "ape_gather_kernel", "ape_mean_kernel", "ape_cov_kernel",
           "ape_error_kernel", "ape_moment_kernel", "ape_spread_kernel", "ape_result_kernel")


def test_workspace_is_zero_only_for_an_invalid_n(lib):
    sizes = [lib.goslam_ape_workspace_bytes(n) for n in (0, 1, 3, 6000, 10 ** 6, (1 << 31) - 1)]
    assert all(s > 0 for s in sizes) and sizes == sorted(sizes)
    assert sizes[-1] > 60 * ((1 << 31) - 1)                  # the per-row buffers of the largest call
    assert lib.goslam_ape_workspace_bytes(-1) == 0 and lib.goslam_ape_workspace_bytes(1 << 31) == 0


def test_arguments_are_checked_first(lib):
    p = ctypes.c_void_p(1 << 20)
    ws = lib.goslam_ape_workspace_bytes(4)
    assert lib.goslam_ape_sim3(p, p, -1, p, ws, p, p, None) == -1
    assert lib.goslam_ape_sim3(p, p, 1 << 31, p, ws, p, p, None) == -1
    assert lib.goslam_ape_sim3(p, p, 4, p, ws, None, p, None) == -1               # no out
    assert lib.goslam_ape_sim3(None, p, 4, p, ws, p, p, None) == -1               # no estimate
    assert lib.goslam_ape_sim3(p, p, 4, p, ws, p, None, None) == -1               # no errors
    assert lib.goslam_ape_sim3(p, p, 4, None, ws, p, p, None) == -3               # no workspace
    assert lib.goslam_ape_sim3(p, p, 4, p, ws - 1, p, p, None) == -3              # too small


def _has_cuda_device():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        return False


@pytest.mark.skipif(_has_cuda_device(), reason="checks the failure path without a CUDA device")
def test_without_a_device_a_valid_call_is_a_launch_error(lib):
    got = {}

    def run(n):   # the noted error is per thread: a fresh thread starts with none
        p = ctypes.c_void_p(1 << 20)
        got[n] = (lib.goslam_ape_sim3(p, p, n, p, lib.goslam_ape_workspace_bytes(n), p, p, None),
                  lib.goslam_last_cuda_error())
    for n in (0, 5, 10 ** 6):
        t = threading.Thread(target=run, args=(n,))
        t.start()
        t.join()
    for n, (rc, err) in got.items():
        assert rc == -2 and err, (n, rc, err)


def _cuobjdump(flag):
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    return subprocess.run(["cuobjdump", flag, _lib.lib_path()], capture_output=True, text=True).stdout


def test_kernels_have_no_stack_or_local_memory():
    lines = _cuobjdump("-res-usage").splitlines()
    for kernel in KERNELS:
        idx = [i for i, l in enumerate(lines) if "Function" in l and kernel in l]
        assert len(idx) == 1, (kernel, idx)
        usage = lines[idx[0] + 1]
        assert re.search(r"\bSTACK:0\b", usage) and re.search(r"\bLOCAL:0\b", usage), (kernel, usage)

