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


P = ctypes.c_void_p
_C_STRUCTS = {"goslam_neus_params": "NeusParams", "goslam_neus_out": "NeusOut", "goslam_neus_mlp_bwd_out": "NeusMlpBwdOut",
              "goslam_ba_peers": "BaPeers", "goslam_gru_weights": "GruWeights", "goslam_update_weights": "UpdateWeights",
              "goslam_conv_desc": "ConvDesc", "goslam_encoder_conv": "EncoderConv",
              "goslam_encoder_weights": "EncoderWeights"}


def _prototypes():
    """(return type, name, [parameter declarations]) of every prototype: a line-anchored scan of the header"""
    src = open(os.path.join(ROOT, "include", "goslam_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = []
    for m in re.finditer(r"^(int|size_t|int64_t|const char\*) (goslam_[a-z0-9_]+)\((.*?)\);", src, flags=re.M | re.S):
        params = [" ".join(p.split()) for p in m.group(3).split(",")]
        out.append((m.group(1), m.group(2), [] if params == ["void"] else params))
    return out


def _expected_type(decl):
    from goslam_b200 import _lib
    words = decl.replace("*", " * ").split()
    if decl in ("int", "size_t", "int64_t", "const char*"):          # return types
        words = words + ["_"]
    words = [w for w in words[:-1] if w != "const"]
    if "*" not in words:
        return {"int": ctypes.c_int, "unsigned": ctypes.c_uint, "float": ctypes.c_float, "double": ctypes.c_double,
                "size_t": ctypes.c_size_t, "int64_t": ctypes.c_int64, "long long": ctypes.c_int64}[" ".join(words)]
    if words == ["char", "*"]:
        return ctypes.c_char_p
    if words[0] in _C_STRUCTS and words[1:] == ["*"]:
        return ctypes.POINTER(getattr(_lib, _C_STRUCTS[words[0]]))
    return P


def test_every_prototype_is_bound_with_its_header_types(lib):
    protos = _prototypes()
    assert len(protos) == len(_declared_symbols())
    for ret, name, params in protos:
        fn = getattr(lib, name)
        assert fn.restype == _expected_type(ret), name
        assert fn.argtypes == [_expected_type(p) for p in params], name


def test_derived_signatures_written_out():
    from goslam_b200 import _lib
    sigs = _lib.parse_header(open(_lib.HEADER).read())
    i, f, d, z, i64 = ctypes.c_int, ctypes.c_float, ctypes.c_double, ctypes.c_size_t, ctypes.c_int64
    assert sigs["goslam_ba"] == (i, [P] * 7 + [i] + [P] * 2 + [i] * 7 + [f, f, i] + [P] * 3 + [P, z, P], True)
    assert sigs["goslam_neus_forward"] == (i, [ctypes.POINTER(_lib.NeusParams)] + [P] * 4 + [i, i] +
                                           [ctypes.POINTER(_lib.NeusOut), P, z, P], True)
    assert sigs["goslam_mapping_rays"] == (i, [P, z, i, i, i, P, P, i64, i, P, P, P, d, d, d, d, P, P, P, P, i64, P],
                                           True)
    assert sigs["goslam_ape_sim3"] == (i, [P, P, i64, P, z, P, P, P], True)
    assert sigs["goslam_neus_composite_backward"][1][14:18] == [i64, i64, i, i]          # long long
    assert sigs["goslam_strerror"] == (ctypes.c_char_p, [i], False)
    assert sigs["goslam_ape_workspace_bytes"] == (z, [i64], False)
    assert sigs["goslam_peer_alloc"] == (i, [z, P, P], False)


def test_unknown_c_type_is_an_error():
    from goslam_b200 import _lib
    with pytest.raises(ValueError, match="goslam_probe"):
        _lib.parse_header("int goslam_probe(const float* x, struct unknown u, void* stream);")
    with pytest.raises(ValueError, match="goslam_probe_ret"):
        _lib.parse_header("half goslam_probe_ret(int n);")


def test_structures_match_the_c_layout(tmp_path):
    """sizeof and every field's offsetof of each C struct, from a C99 program compiled against the header"""
    import shutil
    import subprocess
    from goslam_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc is missing")
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "goslam_b200.h"', "int main(void) {"]
    for cname, pyname in _C_STRUCTS.items():
        lines.append('  printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for field, _ in getattr(_lib, pyname)._fields_:
            cfield = "in" if field == "inp" else field
            lines.append('  printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, field, cname, cfield))
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", str(tmp_path / "layout")
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src),
                    "-o", exe], check=True)
    got = dict(line.split() for line in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    want = {}
    for cname, pyname in _C_STRUCTS.items():
        cls = getattr(_lib, pyname)
        want[cname] = str(ctypes.sizeof(cls))
        for field, _ in cls._fields_:
            want["%s.%s" % (cname, field)] = str(getattr(cls, field).offset)
    assert got == want
    assert {c: int(got[c]) for c in _C_STRUCTS} == {
        "goslam_neus_params": 96, "goslam_neus_out": 120, "goslam_neus_mlp_bwd_out": 80, "goslam_ba_peers": 216,
        "goslam_gru_weights": 64, "goslam_update_weights": 240, "goslam_conv_desc": 168, "goslam_encoder_conv": 16,
        "goslam_encoder_weights": 320}


def test_call_rejects_a_cpu_tensor_before_the_library(monkeypatch):
    import torch
    from goslam_b200 import _lib

    class Unreachable:
        def __getattr__(self, name):
            def fn(*args):
                raise AssertionError("%s reached the library" % name)
            return fn
    monkeypatch.setattr(_lib, "_LIB", Unreachable())
    cpu = torch.zeros(4, 7)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.call("iproj", cpu, cpu, cpu, cpu, 1, 1, 1)
    with pytest.raises(RuntimeError, match="CUDA"):
        _lib.call("frame_distance", None, None, None, None, None, cpu, 0, 4, 4, 0.3)


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


def test_ba_and_neus_workspace_queries(lib):
    # BA: grows with edges and pixels, 0 on invalid shapes
    a = lib.goslam_ba_workspace_bytes(36, 8, 40, 80, 1, 8)
    b = lib.goslam_ba_workspace_bytes(72, 8, 40, 80, 1, 8)
    assert 0 < a < b
    assert lib.goslam_ba_workspace_bytes(36, 0, 40, 80, 1, 8) == 0
    assert lib.goslam_ba_workspace_bytes(36, 8, 40, 80, 1, 9) == 0        # t1 > num
    assert lib.goslam_ba_system_doubles(1, 8) == 42 * 42 + 42
    assert lib.goslam_neus_workspace_bytes(1 << 18, 72) > 0


def test_argument_validation_without_gpu(lib):
    """shape errors are rejected before any CUDA call."""
    null = ctypes.c_void_p(None)
    assert lib.goslam_corr_index_forward(null, 1, null, null, 2, 0, 4, 4, 4, 3, null) == -1
    assert lib.goslam_corr_index_forward(null, 1, null, null, 0, 4, 4, 4, 4, 3, null) == 0      # N == 0: no-op
    assert lib.goslam_corr_build(null, null, 2, null, 4, 1, 128, 40, 80, null) == -1              # dtype neither f16 nor f32
    assert lib.goslam_corr_build(null, null, 1, null, 4, 1, 128, 4, 80, null) == -1               # level 3 of h = 4 is empty
    assert lib.goslam_corr_build(null, null, 0, null, 4, 0, 128, 40, 80, null) == 0               # N == 0: no-op
    assert lib.goslam_corr_pool_build(null, 8, 1, null, null, null, null, 4, 1, 128, 40, 160, null) == -1  # w > 128
    assert lib.goslam_frame_distance(null, null, null, null, null, null, 0, 4, 4, 0.3, null) == 0
    # the per-pixel geometry entries put edges (frames for iproj) on grid.y: more than 65535 is a shape error,
    # not a failed launch; 65535 itself passes validation (null stream / pointers never reach a device at K = 0)
    for K in (65536, 1 << 30):
        assert lib.goslam_reproject(null, null, null, null, null, null, null, K, 4, 4, null) == -1
        assert lib.goslam_reproject_motion(null, null, null, null, null, null, null, null, null, K, 4, 4, null) == -1
        assert lib.goslam_projmap(null, null, null, null, null, null, null, K, 4, 4, null) == -1
        assert lib.goslam_depth_filter(null, null, null, null, null, null, K, 8, 4, 4, null) == -1
        assert lib.goslam_iproj(null, null, null, null, K, 4, 4, null) == -1
    assert lib.goslam_reproject(null, null, null, null, null, null, null, 0, 4, 4, null) == 0
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


def _has_cuda_device():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        return False


@pytest.mark.skipif(_has_cuda_device(), reason="checks the failure path without a CUDA device")
def test_setup_failure_is_launch_error_with_cuda_error(lib):
    """valid calls whose first CUDA work is per-device setup (function attributes, constant memory, the tensor-map
    encoder) fail as GOSLAM_ELAUNCH and name the CUDA error behind it, as every other failed launch does."""
    import threading
    from goslam_b200 import _lib
    p = ctypes.c_void_p(1 << 20)                       # never dereferenced: nothing reaches a device
    pyramid = (ctypes.c_void_p * 4)(*[1 << 20] * 4)   # host array of (16-byte aligned) device pointers
    conv = _lib.ConvDesc()
    conv.inp[0], conv.cin[0], conv.cin_stride[0], conv.n_in = p, 64, 64, 1
    conv.weight, conv.bias, conv.out = p, p, p
    conv.taps, conv.cout, conv.cout_pad, conv.out_scale, conv.out_stride = 1, 64, 64, 1.0, 64
    ba_ws = lib.goslam_ba_workspace_bytes(1, 2, 4, 4, 1, 2)
    neus = _lib.NeusParams(p, p, p, p, p)
    neus_out = _lib.NeusOut(*[p] * 15)
    mlp_out = _lib.NeusMlpBwdOut(*[p] * 10)
    calls = {
        "altcorr_forward": lambda: lib.goslam_altcorr_forward(p, p, p, p, 1, 1, 8, 8, 8, 8, 128, 3, None),
        "altcorr_pyramid": lambda: lib.goslam_altcorr_pyramid(pyramid, 4, p, p, p, p, 1, 16, 16, 128, 3, None),
        "conv2d_nhwc": lambda: lib.goslam_conv2d_nhwc(ctypes.byref(conv), 1, 8, 16, None),
        "corr_pool_build": lambda: lib.goslam_corr_pool_build(p, 2, 1, p, p, p, pyramid, 4, 1, 128, 32, 32, None),
        "ba": lambda: lib.goslam_ba(p, p, p, p, p, p, None, 0, p, p, 1, 2, 4, 4, 1, 2, 1, 1e-4, 0.1, 1, None, None,
                                    None, p, ba_ws, None),
        "neus_forward": lambda: lib.goslam_neus_forward(ctypes.byref(neus), p, p, p, p, 1, 8, ctypes.byref(neus_out), p,
                                                        lib.goslam_neus_workspace_bytes(1, 8), None),
        "neus_mlp_backward": lambda: lib.goslam_neus_mlp_backward(ctypes.byref(neus), *[p] * 10, 1, 8,
                                                                  ctypes.byref(mlp_out), None),
        "neus_grid_backward": lambda: lib.goslam_neus_grid_backward(ctypes.byref(neus), p, p, p, p, None, 0, 1, 8, p,
                                                                    None, p, p, p, None),
        "neus_sdf_grid": lambda: lib.goslam_neus_sdf_grid(ctypes.byref(neus), p, p, p, 2, 2, 2, p, None),
        "neus_vertex_color": lambda: lib.goslam_neus_vertex_color(ctypes.byref(neus), p, 1, p, None),
    }
    got = {}

    def run(name):   # the noted error is per thread: a fresh thread starts with none
        got[name] = (calls[name](), lib.goslam_last_cuda_error())
    for name in calls:
        t = threading.Thread(target=run, args=(name,))
        t.start()
        t.join()
    for name, (rc, err) in got.items():
        assert rc == -2 and err, (name, rc, err)


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
