"""CPU checks of the rendering metrics (csrc/render_eval.cu, goslam_b200.render_eval, oracle/render_eval_oracle.py):
  - the float64 oracle against an independent formulation: scipy.signal.correlate2d with the 11 x 11 outer-product
    window for SSIM, direct sums for PSNR and depth L1;
  - the new prototypes bind through the header;
  - argument and workspace refusals before anything reaches CUDA, and the workspace size at several shapes;
  - no stack, local memory or spills in the new kernels;
  - RenderMetrics' means and its fixed text."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
from scipy import signal

from oracle import render_eval_oracle as ro

EINVAL, EWORKSPACE, ELAUNCH = -1, -3, -2
KERNELS = ("render_metrics_tile_kernel", "render_metrics_reduce_kernel")
NEW_ENTRIES = ("goslam_render_metrics_workspace_bytes", "goslam_render_metrics")


def _scipy_ssim(x, y):
    """SSIM of one channel pair [H, W]: 2-D 'valid' correlation with the outer product of the normalised 1-D window"""
    i = np.arange(11, dtype=np.float64)
    g = np.exp(-(i - 5.0) ** 2 / 4.5)
    g /= g.sum()
    w = np.outer(g, g)
    f = lambda a: signal.correlate2d(a, w, mode="valid")   # noqa: E731
    mx, my = f(x), f(y)
    vx, vy, cxy = f(x * x) - mx ** 2, f(y * y) - my ** 2, f(x * y) - mx * my
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    return ((2 * mx * my + c1) * (2 * cxy + c2) / ((mx ** 2 + my ** 2 + c1) * (vx + vy + c2))).mean()


def _frame(rng, H, W, kind):
    gt = rng.random((3, H, W))
    if kind == "noisy":
        color = np.clip(gt.transpose(1, 2, 0) + 0.05 * rng.standard_normal((H, W, 3)), 0, 1)
    elif kind == "constant":
        gt = np.full((3, H, W), 0.3)
        color = np.full((H, W, 3), 0.7)
    else:   # smooth: gradients, where SSIM is sensitive to the variance terms
        yy, xx = np.mgrid[0:H, 0:W] / max(H, W)
        gt = np.stack([xx, yy, 0.5 * (xx + yy)])
        color = (gt + 0.01 * np.sin(7 * xx + 3 * yy)).transpose(1, 2, 0)
    return color.reshape(H * W, 3), gt


@pytest.mark.parametrize("H,W", [(11, 11), (12, 19), (33, 40)])
@pytest.mark.parametrize("kind", ["noisy", "constant", "smooth"])
def test_oracle_matches_an_independent_formulation(H, W, kind):
    rng = np.random.default_rng(H * 100 + W)
    color, gt = _frame(rng, H, W, kind)
    planar = color.reshape(H, W, 3).transpose(2, 0, 1)
    want_ssim = np.mean([_scipy_ssim(planar[c], gt[c]) for c in range(3)])
    assert abs(ro.ssim(color, gt, H, W) - want_ssim) <= 1e-12
    mse = np.sum((planar - gt) ** 2) / (3 * H * W)
    assert abs(ro.psnr(color, gt, H, W) - 10 * np.log10(1.0 / mse)) <= 1e-9
    assert ro.psnr(gt.transpose(1, 2, 0).reshape(-1, 3), gt, H, W) == np.inf
    assert ro.ssim(gt.transpose(1, 2, 0).reshape(-1, 3), gt, H, W) == pytest.approx(1.0, abs=1e-12)


def test_oracle_depth_l1_counts_only_valid_pixels():
    rng = np.random.default_rng(4)
    d = rng.random(200) * 3
    g = rng.random(200) * 3
    g[:10] = 0.0
    g[10:15] = np.nan
    g[15:20] = np.inf
    g[20:25] = -1.0
    m = np.ones(200, np.uint8)
    m[25:40] = 0
    want = [abs(a - b) for a, b, k in zip(d, g, m) if np.isfinite(b) and b > 0 and k]
    got, n = ro.depth_l1(d, g, m)
    assert n == len(want) == 160 and abs(got - sum(want) / len(want)) <= 1e-15
    got, n = ro.depth_l1(d, g)
    assert n == 175
    got, n = ro.depth_l1(d, np.zeros(200))
    assert n == 0 and np.isnan(got)


def test_gaussian_window_is_the_documented_one():
    g = ro.gaussian_window()
    i = np.arange(11)
    assert np.allclose(g, np.exp(-(i - 5) ** 2 / 4.5) / np.exp(-(i - 5) ** 2 / 4.5).sum(), rtol=0, atol=1e-17)
    assert g[5] == g.max() and np.array_equal(g, g[::-1])


# ----------------------------------------------------------------------------- C entries
def test_new_prototypes_bind_through_the_header(lib):
    from goslam_b200 import _lib
    for name in NEW_ENTRIES:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
        assert getattr(lib, name).restype == _lib.SIGNATURES[name][0]
    assert "goslam_render_metrics" in _lib._TAKES_STREAM


def _bytes(K, H, W):
    """the layout: one 256-byte aligned block of 4 f64 partials per (frame, 16 x 32 tile of SSIM positions)"""
    tiles = -(-(H - 10) // 16) * -(-(W - 10) // 32)
    n = 4 * 8 * max(K, 1) * tiles
    return -(-n // 256) * 256


def test_workspace_size(lib):
    ws = lib.goslam_render_metrics_workspace_bytes
    for K, H, W in [(0, 11, 11), (1, 11, 11), (3, 31, 32), (17, 33, 65), (1, 26, 42), (1, 27, 43), (100, 320, 640),
                    (300, 240, 320), (5, 480, 640), (65536, 11, 11)]:
        assert ws(K, H, W) == _bytes(K, H, W), (K, H, W)
    assert ws(100, 320, 640) == 100 * 20 * 20 * 32            # 20 x 20 tiles of 16 x 32 over 310 x 630
    for K, H, W in [(-1, 20, 20), (1, 10, 20), (1, 20, 10), (1, 0, 0), (1, 65536, 65536)]:
        assert ws(K, H, W) == 0, (K, H, W)


def test_arguments_and_workspace_are_checked_first(lib):
    p = ctypes.c_void_p(1 << 20)
    K, H, W = 2, 20, 30
    need = lib.goslam_render_metrics_workspace_bytes(K, H, W)

    def call(K=K, H=H, W=W, ws=p, nb=need, **null):
        a = {n: (None if n in null else p) for n in ("color", "depth", "gt_color", "gt_depth", "mask", "psnr", "ssim",
                                                      "depth_l1", "depth_count")}
        return lib.goslam_render_metrics(a["color"], a["depth"], a["gt_color"], a["gt_depth"], a["mask"], K, H, W, ws,
                                         nb, a["psnr"], a["ssim"], a["depth_l1"], a["depth_count"], None)

    assert call(K=-1) == EINVAL
    assert call(H=10) == EINVAL and call(W=10) == EINVAL and call(H=10, W=10) == EINVAL
    assert call(H=65536, W=65536) == EINVAL
    for name in ("color", "depth", "gt_color", "gt_depth", "psnr", "ssim", "depth_l1", "depth_count"):
        assert call(**{name: True}) == EINVAL, name
    assert call(ws=None) == EWORKSPACE
    assert call(nb=need - 1) == EWORKSPACE
    assert call(K=0, ws=None, nb=0, color=True, psnr=True) == 0          # nothing to do, nothing touched


def _has_cuda_device():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        return False


@pytest.mark.skipif(_has_cuda_device(), reason="passes dummy device pointers: checked only without a CUDA device")
def test_without_a_device_a_valid_call_is_a_launch_error(lib):
    import threading
    got = []

    def run():
        p = ctypes.c_void_p(1 << 20)
        need = lib.goslam_render_metrics_workspace_bytes(2, 20, 30)
        got.append(lib.goslam_render_metrics(p, p, p, p, None, 2, 20, 30, p, need, p, p, p, p, None))
        got.append(lib.goslam_last_cuda_error())
    t = threading.Thread(target=run)
    t.start()
    t.join()
    assert got[0] == ELAUNCH and got[1]


def test_kernels_use_no_stack_or_local_memory():
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    lines = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout.splitlines()
    for kernel in KERNELS:
        idx = [i for i, l in enumerate(lines) if "Function" in l and kernel in l]
        assert len(idx) == 1, (kernel, idx)
        usage = lines[idx[0] + 1]
        assert re.search(r"\bSTACK:0\b", usage) and re.search(r"\bLOCAL:0\b", usage), (kernel, usage)


def test_kernels_compile_without_spills_for_sm90a(tmp_path):
    from goslam_b200 import build
    nvcc = build._nvcc()
    src = os.path.join(build.CSRC, "render_eval.cu")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "render_eval.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    seen = 0
    for b in re.split(r"ptxas info\s+: Compiling entry function", r.stderr):
        head = b.splitlines()[0] if b else ""
        if any(k in head for k in KERNELS):
            seen += 1
            assert "0 bytes spill stores, 0 bytes spill loads" in b and "0 bytes stack frame" in b, b
    assert seen == len(KERNELS)


# ----------------------------------------------------------------------------- Python layer
def test_render_metrics_means_and_text():
    from goslam_b200 import render_eval
    r = render_eval.RenderMetrics(np.array([20.0, 30.0, 40.0]), np.array([0.5, 0.7, 0.9]),
                                  np.array([0.1, np.nan, 0.3]), np.array([10, 0, 5], np.int64))
    assert r.stats == {"psnr": 30.0, "ssim": pytest.approx(0.7), "depth_l1": pytest.approx(0.2), "depth_views": 2}
    assert r.pretty_str() == ("Rendering metrics (3 views)\n\n"
                              "        psnr\t30.000000\n"
                              "        ssim\t0.700000\n"
                              "    depth_l1\t0.200000\n"
                              " depth_views\t2\n")
    mono = render_eval.RenderMetrics(np.array([25.0]), np.array([0.8]), np.array([np.nan]), np.array([0], np.int64))
    assert np.isnan(mono.stats["depth_l1"]) and mono.stats["depth_views"] == 0
    assert "    depth_l1\tnan\n" in mono.pretty_str()


def test_exported_from_the_package():
    import goslam_b200
    from goslam_b200 import render_eval
    for name in ("image_metrics", "keyframe_views", "eval_render", "RenderMetrics"):
        assert getattr(goslam_b200, name) is getattr(render_eval, name)
