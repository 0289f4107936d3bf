"""CPU-side checks of the drop-in boundary: the C-ABI library loads without a GPU and exports
every symbol include/goslam_b200.h declares; host-only entry points behave."""
import ctypes
import os
import re

import numpy as np

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "goslam_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(goslam_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(lib):
    from goslam_b200 import _lib
    names = _declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), "library does not export %s" % n
        assert n in _lib.SIGNATURES, "ctypes binding missing for %s" % n
    assert sorted(_lib.SIGNATURES) == names, "binding declares symbols the header does not"


def test_identification(lib):
    assert lib.goslam_version() == 100
    assert lib.goslam_sm_arch() == 90
    assert lib.goslam_strerror(0) == b"ok"
    assert b"workspace" in lib.goslam_strerror(-3)
    assert lib.goslam_corr_index_backward() == -4 and lib.goslam_altcorr_backward() == -4


def test_library_has_no_torch_dependency():
    from goslam_b200 import _lib
    import subprocess
    out = subprocess.run(["ldd", _lib.lib_path()], capture_output=True, text=True).stdout
    assert "torch" not in out and "python" not in out and "libcuda.so" not in out, out


def test_sass_is_hopper_native():
    """HGMMA (wgmma) and UTMALDG (TMA loads) must be in the sm_90a SASS."""
    import shutil
    import subprocess
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        import pytest
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in sass or "SM90" in sass.upper()
    for mnem in ("HGMMA", "UTMALDG"):
        assert mnem in sass, mnem


def test_workspace_queries(lib):
    # BA: grows with edges and pixels, 0 on invalid shapes
    a = lib.goslam_ba_workspace_bytes(36, 8, 40, 80, 1, 8)
    b = lib.goslam_ba_workspace_bytes(72, 8, 40, 80, 1, 8)
    assert 0 < a < b
    assert lib.goslam_ba_workspace_bytes(36, 0, 40, 80, 1, 8) == 0
    assert lib.goslam_ba_workspace_bytes(36, 8, 40, 80, 1, 9) == 0        # t1 > num
    assert lib.goslam_ba_system_doubles(1, 8) == 42 * 42 + 42
    assert lib.goslam_corr_build_workspace_bytes(36, 128, 40, 80) >= 2 * 36 * 3200 * 128 * 2
    assert lib.goslam_neus_workspace_bytes(1 << 18, 72) > 0


def test_argument_validation_without_gpu(lib):
    """shape errors are rejected before any CUDA call."""
    null = ctypes.c_void_p(None)
    assert lib.goslam_corr_index_forward(null, 1, null, null, 2, 0, 4, 4, 4, 3, null) == -1
    assert lib.goslam_corr_index_forward(null, 1, null, null, 0, 4, 4, 4, 4, 3, null) == 0      # N == 0: no-op
    assert lib.goslam_frame_distance(null, null, null, null, null, null, 0, 4, 4, 0.3, null) == 0
    assert lib.goslam_altcorr_forward(null, null, null, null, 1, 1, 4, 4, 4, 4, 128, 2, null) == -1  # r != 3
    assert lib.goslam_ba(null, null, null, null, null, null, null, 0, null, null, 4, 8, 4, 4, 1, 8, 2,
                         1e-4, 0.1, 0, null, null, null, null, 0, null) == -1     # eta missing
    assert lib.goslam_ba(null, null, null, null, null, null, null, 0, null, null, 4, 8, 4, 4, 1, 8, 2,
                         1e-4, 0.1, 1, null, null, null, null, 0, null) == -3     # no workspace
    # a conv layer wider than the 1024-entry shared-memory bias vector (1152 = 6 x 192 and 1280 = 5 x 256 are otherwise
    # valid tilings) is rejected as a shape error, even with B = 0 (a library that accepted it returns 0 for the empty
    # batch, so this never reaches a device)
    from goslam_b200 import _lib
    for cout_pad in (1152, 1280):
        d = _lib.ConvDesc()
        d.cin[0], d.cin_stride[0], d.n_in = 64, 64, 1
        d.taps, d.cout, d.cout_pad, d.out_scale, d.out_stride = 1, cout_pad, cout_pad, 1.0, cout_pad
        assert lib.goslam_conv2d_nhwc(ctypes.byref(d), 0, 8, 16, null) == -1, cout_pad


def test_hashgrid_layout_matches_oracle(lib):
    from goslam_b200 import neus
    from oracle import neus_oracle
    offs, ress, scales, total = neus.hashgrid_layout()
    metas, entries = neus_oracle.hashgrid_meta()
    assert total == 2 * entries == 12599920
    assert ress == [m["res"] for m in metas] == [16, 24, 34, 49, 71, 102, 148, 213, 308, 446, 646, 934, 1352, 1956, 2831, 4096]
    assert offs[:-1] == [2 * m["offset"] for m in metas]
    for s, m in zip(scales, metas):
        # BIT-exact: a 1-ulp difference in a level's scale moves samples on that level's cell faces into the
        # neighbouring cell, i.e. changes their normal (found with tests/tools/diag_render_parity.py)
        assert np.float32(s).tobytes() == np.float32(m["scale"]).tobytes(), (s, float(m["scale"]))


def test_header_is_plain_c_and_library_links_without_torch(tmp_path):
    """compile tests/c/abi_smoke.c as C99 against include/goslam_b200.h, link it to libgoslam_b200.so only,
    run it: host-only helpers answer, argument validation returns before any CUDA call."""
    import shutil
    import subprocess
    from goslam_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None or not os.path.exists(_lib.lib_path()):
        pytest.skip("gcc or the built library is missing")
    exe = str(tmp_path / "abi_smoke")
    libdir = os.path.dirname(_lib.lib_path())
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "c", "abi_smoke.c"), "-o", exe, "-L", libdir, "-lgoslam_b200",
                    "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "abi smoke ok" in out.stdout
