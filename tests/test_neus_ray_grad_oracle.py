"""CPU: the closed form of the renderer's ray gradient (oracle/neus_ray_grad_oracle.py, what neus_ray_bwd_kernel
implements) against double-backward autograd in float64, the argument checks of the two new entry points, the
resources of the new kernel, and the restated quaternion / ray construction against tests/golden/neus_ray_grad.npz."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import neus_oracle as no
from oracle import neus_ray_grad_oracle as nro

EINVAL = -1
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "neus_ray_grad.npz")


def _autograd_ray_grads(ro, rd, z, inb, bound, enc, W, b, B, d_out, d_n, dE, d_tc):
    """dL/d rays of L = sum over the network's samples of d_out . out + d_n . normal + dE . (p B) + d_tc (d . normal),
    out = W [x | enc(u)] + b, normal = d out[0] / dp by autograd with create_graph (src/InstantNeuS.py:139-146)"""
    ro, rd = ro.clone().requires_grad_(True), rd.clone().requires_grad_(True)
    R, S = z.shape
    p = (ro[:, None, :] + rd[:, None, :] * z[..., None]).reshape(-1, 3)
    bt = torch.as_tensor(bound, dtype=torch.float64).reshape(3, 2)
    x = torch.clamp((p - bt[:, 0]) / (bt[:, 1] - bt[:, 0]) * 2.0 - 1.0, -1.0, 1.0)
    out = torch.cat([x, enc((x + 1.0) / 2.0)], dim=1) @ W.t() + b
    (nrm,) = torch.autograd.grad(out[:, 0].sum(), p, create_graph=True)
    dirs = rd[:, None, :].expand(R, S, 3).reshape(-1, 3)
    m = torch.as_tensor(inb.reshape(-1, 1), dtype=torch.float64)
    L = (m * (d_out * out)).sum() + (m * d_n * nrm).sum() + (m * dE * (p @ B)).sum() \
        + (m[:, 0] * d_tc * (dirs * nrm).sum(1)).sum()
    return torch.autograd.grad(L, (ro, rd))


@pytest.mark.parametrize("case", ["inside", "clamped", "out_of_bound", "fallback"])
def test_closed_form_matches_double_backward_autograd(case):
    """float64 on both sides: relative error ~1e-13.  'clamped': realtime_bound reaches beyond `bound` on x and z, so
    samples sit on clamped axes (no xyz / grid gradient along them); 'out_of_bound': a tight realtime_bound leaves most
    samples out of the network; 'fallback': nothing in bound and the first 100 samples of the call forced in."""
    torch.manual_seed({"inside": 1, "clamped": 2, "out_of_bound": 3, "fallback": 4}[case])
    dd = torch.float64
    R, S = 9, 24
    bound = [[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]]
    enc = nro.TorchHashGrid64()
    with torch.no_grad():
        offs = [m["offset"] * 2 for m in enc.metas]
        for l, m in enumerate(enc.metas):            # per-level amplitude ~ 1/res: O(1) input gradient per level
            n = m["size"] * 2
            enc.params[offs[l]:offs[l] + n] = torch.randn(n) * (0.5 / m["res"])
    ro = (torch.rand(R, 3, dtype=dd) - 0.5) * 1.0
    rd = torch.nn.functional.normalize(torch.randn(R, 3, dtype=dd), dim=1) * 1.3
    if case == "clamped":
        ro = ro * 4.0                                # start outside bound on some axes
    z = torch.sort(torch.rand(R, S, dtype=dd) * 3.0, dim=1).values
    p = (ro[:, None, :] + rd[:, None, :] * z[..., None]).numpy()
    rt = {"inside": [[-1.9, 1.9]] * 3, "clamped": [[-4.0, 4.0], [-2.0, 2.0], [-4.0, 4.0]],
          "out_of_bound": [[-0.5, 0.5]] * 3, "fallback": [[5.0, 6.0]] * 3}[case]
    rt = np.array(rt)
    inb = np.all((p > rt[:, 0]) & (p < rt[:, 1]), axis=-1)
    if case == "fallback":
        assert not inb.any()
        inb = (np.arange(R * S) < 100).reshape(R, S)
    if case == "clamped":
        x = (p - np.array(bound)[:, 0]) / 4.0 * 2 - 1
        assert (np.abs(x[inb]) > 1).any(axis=-1).sum() >= 10
    if case == "out_of_bound":
        assert 0 < inb.sum() < 0.5 * inb.size
    W = torch.randn(32, 35, dtype=dd) * 0.3
    b = torch.randn(32, dtype=dd) * 0.1
    B = torch.randn(3, 33, dtype=dd)
    n = R * S
    d_out, d_n = torch.randn(n, 32, dtype=dd), torch.randn(n, 3, dtype=dd)
    dE, d_tc = torch.randn(n, 33, dtype=dd), torch.randn(n, dtype=dd)
    want_o, want_d = _autograd_ray_grads(ro, rd, z, inb, bound, enc, W, b, B, d_out, d_n, dE, d_tc)
    # the closed form takes what the backward chain hands the kernel: d_enc = d_out W[:,3:], d_xyz = d_out W[:,:3], the
    # total dL/d normal (here d_n plus the true_cos path d_tc d) and d_tc for the direction's direct path
    dirs = rd[:, None, :].expand(R, S, 3).reshape(-1, 3)
    table = enc.params.detach().half().double().numpy().reshape(-1, 2)
    got_o, got_d = nro.ray_backward_closed_form(
        ro.numpy(), rd.numpy(), z.numpy(), inb, bound, table, W.numpy(), B.numpy(), (d_out @ W[:, 3:]).numpy(),
        (d_out @ W[:, :3]).numpy(), dE.numpy(), (d_n + d_tc[:, None] * dirs).numpy(), d_tc.numpy(), gy=W[0, 3:].numpy())
    for got, want in ((got_o, want_o.numpy()), (got_d, want_d.numpy())):
        assert np.abs(want).max() > 1e-3
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 1e-10, err


def test_second_order_term_is_the_mixed_partials():
    """with only dL/d normal non-zero the ray gradient is the SDF Hessian's mixed part: zero when d_grad is zero, and
    linear in d_grad"""
    rng = np.random.default_rng(0)
    R, S = 3, 8
    metas, total = no.hashgrid_meta()
    table = (rng.standard_normal((total, 2)) * 1e-2).astype(np.float16)
    args = dict(rays_o=np.zeros((R, 3)), rays_d=rng.standard_normal((R, 3)) * 0.3, z_mid=np.sort(rng.random((R, S)) * 2, 1),
                inb=np.ones((R, S), bool), bound=[[-2.0, 2.0]] * 3, table=table, w_sdf=rng.standard_normal((32, 35)),
                color_B=rng.standard_normal((3, 33)), d_enc=np.zeros((R * S, 32)), d_xyz=np.zeros((R * S, 3)),
                dE=np.zeros((R * S, 33)), d_true_cos=np.zeros(R * S))
    zo, zd = nro.ray_backward_closed_form(d_grad=np.zeros((R * S, 3)), **args)
    assert not zo.any() and not zd.any()
    g = rng.standard_normal((R * S, 3))
    o1, d1 = nro.ray_backward_closed_form(d_grad=g, **args)
    o2, d2 = nro.ray_backward_closed_form(d_grad=2.5 * g, **args)
    assert np.abs(o1).max() > 0
    np.testing.assert_allclose(o2, 2.5 * o1, rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(d2, 2.5 * d1, rtol=1e-12, atol=1e-300)


def test_pose_rays_match_the_reference_construction():
    """the restated quaternion_to_Rt + build_rays against what the reference produced from the same leaves"""
    if not os.path.exists(GOLDEN):
        pytest.skip("golden not generated")
    g = np.load(GOLDEN)
    cam = g["traj_cam"]
    px, py = torch.from_numpy(g["traj_px"]).double(), torch.from_numpy(g["traj_py"]).double()
    for f in range(g["traj_quadt0"].shape[0]):
        ro, rd = nro.pose_rays(torch.from_numpy(g["traj_quadt0"][f]).double(), px[f], py[f], *cam.tolist())
        np.testing.assert_allclose(ro.numpy(), g["traj_rays_o0"][f], rtol=0, atol=1e-6)
        np.testing.assert_allclose(rd.numpy(), g["traj_rays_d0"][f], rtol=0, atol=1e-6)


@pytest.fixture(scope="module")
def lib():
    from goslam_b200 import _lib
    return _lib.load()


def test_new_entry_points_reject_bad_arguments(lib):
    p = ctypes.c_void_p(16)
    from goslam_b200 import _lib
    prm = ctypes.byref(_lib.NeusParams())

    def ray(R=4, S=24, sample0=0, params=prm, ptr=p, d_rays_d=p, fallback=None, scale=None):
        return lib.goslam_neus_ray_backward(params, ptr, ptr, ptr, ptr, fallback, sample0, R, S, ptr, ptr, ptr, scale, ptr,
                                            ptr, ptr, d_rays_d, None)
    for kw in (dict(R=-1), dict(S=0), dict(S=129), dict(sample0=-1), dict(params=None), dict(ptr=None), dict(d_rays_d=None)):
        assert ray(**kw) == EINVAL, kw
    assert ray(R=0) == 0                                                    # nothing to do

    def comp(R=4, S=24, sample0=0, total=96, ptr=p):
        return lib.goslam_neus_composite_backward_ex(prm, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, None, None, None, None,
                                                     None, total, sample0, R, S, ptr, ptr, ptr, ptr, None, None)
    for kw in (dict(R=-1), dict(S=0), dict(S=129), dict(sample0=-1), dict(total=95), dict(ptr=None)):
        assert comp(**kw) == EINVAL, kw
    assert comp(R=0, total=0) == 0


def test_ray_kernel_uses_no_local_memory():
    """sm_90a: the ray backward keeps its per-level corners and per-ray sums in registers (no stack frame, no spills)"""
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    lines = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout.splitlines()
    idx = [i for i, l in enumerate(lines) if "Function" in l and "neus_ray_bwd_kernel" in l]
    assert len(idx) == 1, idx
    usage = lines[idx[0] + 1]
    assert re.search(r"\bSTACK:0\b", usage) and re.search(r"\bLOCAL:0\b", usage), usage


def test_ray_kernel_compiles_without_spills_for_sm90a(tmp_path):
    """cross-compile csrc/neus.cu for sm_90a and read ptxas' report for the ray backward: no spill stores or loads"""
    from goslam_b200 import build
    nvcc = build._nvcc()
    src = os.path.join(build.CSRC, "neus.cu")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "neus.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stderr.splitlines()
    idx = [i for i, l in enumerate(lines) if "Function properties" in l and "neus_ray_bwd_kernel" in l]
    assert len(idx) == 1, idx
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", lines[idx[0] + 1]), lines[idx[0] + 1]
