"""CPU checks of camera refinement in mapping (mapping.BA): the float64 closed form of the pose-ray backward
(oracle/refine_oracle.py) against double-precision autograd through neus_ray_grad_oracle.pose_rays; the
matrix-to-quaternion restatement on every Shepperd branch; the restated BA schedule against the reference's own
Mapper.__call__ (tests/golden/mapping_refine.npz); the new C entries' argument checks without a device, and their
kernels' resources."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import mapping_oracle as mo
from oracle import neus_ray_grad_oracle as nro
from oracle import refine_oracle as ro

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mapping_refine.npz")
EINVAL, EWORKSPACE = -1, -3
NEW_ENTRIES = ("goslam_mapping_c2w_to_quadt", "goslam_mapping_pose_rays", "goslam_mapping_pose_rays_backward")


# ----------------------------------------------------------------------------- closed form
def _autograd_case(rows, seed, unit=False):
    """(quadt [n,7] f64 leaf, dirs, rays of every entry through pose_rays, upstream gradients)"""
    g = torch.Generator().manual_seed(seed)
    n = len(rows)
    q = torch.randn(n, 7, generator=g, dtype=torch.float64)
    q[:, :4] *= 1.0 if unit else (0.5 + torch.rand(n, 1, generator=g, dtype=torch.float64))    # |q| off the sphere
    if unit:
        q[:, :4] /= q[:, :4].norm(dim=1, keepdim=True)
    q.requires_grad_(True)
    fx, fy, cx, cy = 20.5, 19.25, 11.3, 7.6
    px = [torch.randint(0, 24, (r,), generator=g).double() for r in rows]
    py = [torch.randint(0, 16, (r,), generator=g).double() for r in rows]
    ro_, rd_ = [], []
    for e in range(n):
        o, d = nro.pose_rays(q[e], px[e], py[e], fx, fy, cx, cy)
        ro_.append(o)
        rd_.append(d)
    rays_o, rays_d = torch.cat(ro_), torch.cat(rd_)
    go = torch.randn(rays_o.shape, generator=g, dtype=torch.float64)
    gd = torch.randn(rays_d.shape, generator=g, dtype=torch.float64)
    dirs = torch.cat([torch.stack([(x - cx) / fx, (y - cy) / fy, torch.ones_like(x)], -1) for x, y in zip(px, py)])
    return q, dirs, rays_o, rays_d, go, gd


@pytest.mark.parametrize("rows,unit", [([5, 7, 3], False), ([5, 0, 9, 0], False), ([1, 12], True), ([0], False),
                                       ([40, 40, 21], False)])
def test_closed_form_matches_double_autograd(rows, unit):
    q, dirs, rays_o, rays_d, go, gd = _autograd_case(rows, seed=len(rows) * 7 + sum(rows), unit=unit)
    if sum(rows) > 0:
        (rays_o * go).sum().add((rays_d * gd).sum()).backward()
        want = q.grad.numpy()
    else:
        want = np.zeros((len(rows), 7))
    got = ro.pose_ray_backward(q.detach().numpy(), dirs.numpy(), rows, go.numpy(), gd.numpy())
    for e in range(len(rows)):
        scale = max(np.linalg.norm(want[e]), 1e-300)
        assert np.linalg.norm(got[e] - want[e]) <= 1e-10 * scale or rows[e] == 0, (e, got[e], want[e])
        if rows[e] == 0:
            assert np.all(got[e] == 0.0)


def test_closed_form_gives_duplicate_entries_their_own_gradients():
    """a frame listed twice has two leaves with the same value but different rows: different gradients, each the
    autograd one"""
    rows = [6, 6]
    q, dirs, rays_o, rays_d, go, gd = _autograd_case(rows, seed=3)
    with torch.no_grad():
        q[1] = q[0]
    q.grad = None
    rays_o = torch.cat([nro.pose_rays(q[e], torch.zeros(6, dtype=torch.float64), torch.zeros(6, dtype=torch.float64),
                                      1.0, 1.0, 0.0, 0.0)[0] for e in range(2)])
    rd = [(dirs[6 * e:6 * e + 6] @ nro.quat_to_rotation(q[e:e + 1, :4])[0].t()) for e in range(2)]
    ((rays_o * go).sum() + (torch.cat(rd) * gd).sum()).backward()
    got = ro.pose_ray_backward(q.detach().numpy(), dirs.numpy(), rows, go.numpy(), gd.numpy())
    np.testing.assert_allclose(got, q.grad.numpy(), rtol=1e-10, atol=1e-12)
    assert np.abs(got[0] - got[1]).max() > 1e-3


def test_gradient_is_orthogonal_to_q():
    """quad2rotation is invariant under q -> c q, so dL/dq . q = 0 for any upstream gradient"""
    q, dirs, _, _, go, gd = _autograd_case([9, 4], seed=11)
    got = ro.pose_ray_backward(q.detach().numpy(), dirs.numpy(), [9, 4], go.numpy(), gd.numpy())
    qn = q.detach().numpy()
    for e in range(2):
        assert abs(got[e, :4] @ qn[e, :4]) <= 1e-12 * np.linalg.norm(got[e, :4]) * np.linalg.norm(qn[e, :4])


# ----------------------------------------------------------------------------- matrix to quaternion
def _rot(axis, ang):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def test_matrix_to_quaternion_round_trips_on_every_branch():
    rs = np.random.RandomState(2)
    mats = [np.eye(3), _rot([1, 0, 0], np.pi), _rot([0, 1, 0], np.pi), _rot([0, 0, 1], np.pi),
            _rot([1, 1, 0], np.pi), _rot([0.3, -0.2, 0.9], np.pi)]
    for axis in ([1, 0.01, 0.02], [0.01, 1, -0.02], [0.02, 0.01, 1], [0.4, -0.7, 0.5]):
        for eps in (1e-6, 3e-7, 1e-9, 0.0):
            mats.append(_rot(axis, np.pi - eps))
            mats.append(_rot(axis, -(np.pi - eps)))
    mats += [_rot(rs.randn(3), rs.uniform(-np.pi, np.pi)) for _ in range(200)]
    R = np.stack(mats)
    q = ro.matrix_to_quaternion(R)
    assert np.all(q[:, 0] >= 0.0)
    np.testing.assert_allclose(np.linalg.norm(q, axis=1), 1.0, atol=1e-15)
    back = nro.quat_to_rotation(torch.from_numpy(q)).numpy()
    assert np.abs(back - R).max() <= 1e-12
    # every branch is taken: the trace, then each diagonal entry the largest
    tr = np.trace(R, axis1=1, axis2=2)
    d = np.stack([tr, R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]], 1)
    assert set(np.argmax(d, 1).tolist()) == {0, 1, 2, 3}


# ----------------------------------------------------------------------------- the schedule against the reference
def run_refine_oracle(g, device="cpu"):
    """RefineSchedule over the golden scene with the stand-in renderer and the golden's draws; per training iteration
    (call, rows, loss, leaves after the step or None)"""
    from goslam_b200 import lietorch
    S = mo.GOLDEN_SIZE
    video = mo.golden_video()
    net = ro.StubNet(device)
    opt = torch.optim.AdamW([{'params': net.get_training_parameters(), 'lr': 0.001},
                             {'params': net.get_volume_parameters(), 'lr': 0.01}],
                            betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    iters, calls, losses = [], [], []

    def step(sched, *a):
        mo.reference_optimize_map(sched, *a, losses=losses)
        gr = sched.optimizer.param_groups
        iters.append((len(calls), len(a[0]), float(losses[-1]),
                      torch.stack([q.detach() for q in gr[2]['params']]).cpu().numpy() if len(gr) > 2 else None))

    slam = mo.stub_slam(video, net, ro.StubRenderer(device), mo.GOLDEN_INTR, None)
    sched = ro.RefineSchedule(ro.refine_cfg(device), slam, lietorch.SE3, step, optimizer=opt)
    np.random.seed(S["seed"])
    torch.manual_seed(S["seed"])
    trained = []
    for cur, the_end in ro.REFINE_CALLS:
        video.filtered_id[0] = cur
        trained.append(sched(the_end=the_end))
        calls.append((len(opt.param_groups), [gr['lr'] for gr in opt.param_groups], sched.last_visit))
    return sched, iters, calls, trained


def test_refine_schedule_reproduces_reference_golden():
    g = np.load(GOLDEN)
    sched, iters, calls, trained = run_refine_oracle(g)
    assert [len(d) for d in sched.draws] == g["draw_sizes"].tolist()
    assert np.array_equal(torch.cat(sched.draws).numpy(), g["draws"])
    assert [c[0] for c in calls] == g["call_groups"].tolist()
    assert [c[2] for c in calls] == g["call_last_visit"].tolist()
    lr = np.array([c[1] + [np.nan] * (3 - len(c[1])) for c in calls])
    np.testing.assert_array_equal(lr, g["call_lr"])
    assert [i[0] for i in iters] == g["iter_call"].tolist()
    assert [i[1] for i in iters] == g["iter_rows"].tolist()
    assert np.all(np.abs(np.array([i[2] for i in iters]) - g["iter_loss"]) <= 1e-6 * np.maximum(1.0, np.abs(g["iter_loss"])))
    n_leaves = [0 if i[3] is None else len(i[3]) for i in iters]
    assert n_leaves == g["iter_n_leaves"].tolist()
    got = np.concatenate([i[3] for i in iters if i[3] is not None])
    want = g["iter_leaves"]
    sign = np.sign(np.sum(got[:, :4] * want[:, :4], axis=1, keepdims=True))   # each leaf's sign, fixed at creation
    assert np.all(sign != 0)
    assert np.abs(got[:, :4] * sign - want[:, :4]).max() <= 1e-6 and np.abs(got[:, 4:] - want[:, 4:]).max() <= 1e-6


def test_refine_golden_covers_the_scenario():
    g = np.load(GOLDEN)
    sched, iters, calls, trained = run_refine_oracle(g)
    groups = g["call_groups"].tolist()
    assert groups[:3] == [2, 2, 2] and all(n == 3 for n in groups[3:])     # no leaves before last_visit reaches 10
    assert g["call_last_visit"].tolist()[2] == 10 and g["call_the_end"][-1]
    first = groups.index(3)
    assert trained[first] == [False]                                       # the first camera call's batch: < 100 rays
    ba_calls = set(g["iter_call"][g["iter_n_leaves"] > 0].tolist())
    assert len(ba_calls) >= 3                                              # later calls replace the group and train it
    visits = [v for _, v in sched.log]
    assert any(len(v) != len(set(v)) for v in visits[first:])              # repeated frames among the leaves
    # within a call the visit iterations move the leaves; the unvisit iterations give them no gradient, so AdamW
    # leaves them exactly where they were
    at = 0
    per_iter = []
    for n in g["iter_n_leaves"]:
        per_iter.append(g["iter_leaves"][at:at + n])
        at += n
    c = g["iter_call"]
    moved = [np.abs(per_iter[i] - per_iter[i - 1]).max() for i in range(1, len(c))
             if c[i] == c[i - 1] and len(per_iter[i]) and len(per_iter[i - 1])]
    assert moved and max(moved) > 0 and min(moved) == 0


# ----------------------------------------------------------------------------- C entries
def test_new_prototypes_bind_through_the_header(lib):
    from goslam_b200 import _lib
    for name in NEW_ENTRIES:
        assert name in _lib.SIGNATURES
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
        assert getattr(lib, name).restype == _lib.SIGNATURES[name][0]


def test_new_entry_points_reject_bad_arguments(lib):
    ws = lib.goslam_mapping_snapshot_workspace_bytes
    p = ctypes.c_void_p(16)
    q2w = lib.goslam_mapping_c2w_to_quadt
    assert q2w(p, -1, p, None) == EINVAL
    assert q2w(None, 3, p, None) == EINVAL and q2w(p, 3, None, None) == EINVAL
    assert q2w(None, 0, None, None) == 0                                   # nothing to do
    arr = ctypes.c_int * 3

    def fwd(slots, counts, draw, n_draws=100, max_rays=1000, workspace=p, nbytes=1 << 20, F=2, H=8, quadt=p, out=p):
        return lib.goslam_mapping_pose_rays(workspace, ctypes.c_size_t(nbytes), F, H, 8, quadt, p, n_draws, 3,
                                            arr(*slots), arr(*counts), arr(*draw), 1.0, 1.0, 0.0, 0.0, out, p, p, p,
                                            max_rays, None)

    def bwd(slots, counts, draw, n_draws=100, max_rays=1000, workspace=p, nbytes=1 << 20, F=2, H=8, quadt=p, out=p,
            grads=p):
        return lib.goslam_mapping_pose_rays_backward(workspace, ctypes.c_size_t(nbytes), F, H, 8, quadt, p, n_draws, 3,
                                                     arr(*slots), arr(*counts), arr(*draw), 1.0, 1.0, 0.0, 0.0, grads,
                                                     grads, max_rays, out, None)

    for f in (fwd, bwd):
        assert f([0, 1, 1], [4, 4, 4], [0, 0, 0], F=0) == EINVAL              # no snapshot
        assert f([0, 1, 1], [4, 4, 4], [0, 0, 0], H=0) == EINVAL
        assert f([0, 1, 2], [4, 4, 4], [0, 0, 0]) == EINVAL                   # slot outside the snapshot
        assert f([0, 1, 1], [4, 65, 4], [0, 0, 0]) == EINVAL                  # N_f beyond H*W
        assert f([0, 1, 1], [4, 0, 4], [0, 2, 0]) == EINVAL                   # draws from an empty frame
        assert f([0, 1, 1], [4, 4, 4], [0, -1, 0]) == EINVAL
        assert f([0, 1, 1], [40, 40, 40], [0, 0, 0], max_rays=119) == EINVAL  # rays / gradients too short
        assert f([0, 1, 1], [40, 40, 40], [5, 5, 0], n_draws=9) == EINVAL     # draw buffer too short
        assert f([0, 1, 1], [40, 40, 40], [5, 5, 0], quadt=None) == EINVAL
        assert f([0, 1, 1], [40, 40, 40], [5, 5, 0], out=None) == EINVAL
        assert f([0, 1, 1], [40, 40, 40], [5, 5, 0], workspace=None) == EWORKSPACE
        assert f([0, 1, 1], [40, 40, 40], [5, 5, 0], nbytes=ws(2, 8, 8) - 1) == EWORKSPACE
    assert bwd([0, 1, 1], [40, 40, 40], [5, 5, 0], grads=None) == EINVAL
    assert fwd([0, 1, 1], [0, 0, 0], [0, 0, 0]) == 0                          # empty batch: no launch
    assert lib.goslam_mapping_pose_rays_backward(p, ctypes.c_size_t(1 << 20), 2, 8, 8, None, None, 0, 0, None, None,
                                                 None, 1.0, 1.0, 0.0, 0.0, None, None, 0, None, None) == 0  # no entries


def test_pose_ray_kernels_use_no_local_memory():
    from goslam_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    _lib.load()
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout
    lines = out.splitlines()
    found = 0
    for i, line in enumerate(lines):
        if re.search(r"ray_batch_kernelILb1E|pose_rays_backward_kernel|c2w_to_quadt_kernel", line):
            found += 1
            res = lines[i + 1]
            assert re.search(r"STACK:0\b", res) and re.search(r"LOCAL:0\b", res), (line, res)
    assert found == 3


def test_pose_ray_kernels_compile_without_spills_for_sm90a(tmp_path):
    from goslam_b200 import build
    nvcc = build._nvcc()
    src = os.path.join(build.CSRC, "mapping.cu")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "mapping.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    blocks = re.split(r"ptxas info\s+: Compiling entry function", r.stderr)
    seen = 0
    for b in blocks:
        if re.search(r"ray_batch_kernelILb1E|pose_rays_backward_kernel|c2w_to_quadt_kernel", b.splitlines()[0] if b else ""):
            seen += 1
            assert "0 bytes spill stores, 0 bytes spill loads" in b and "0 bytes stack frame" in b, b
    assert seen == 3


def test_refining_mapper_is_exported_and_mapper_still_refuses_refinement():
    import goslam_b200
    from goslam_b200 import mapping
    assert goslam_b200.RefiningMapper is mapping.RefiningMapper and issubclass(mapping.RefiningMapper, mapping.Mapper)
    S = mo.GOLDEN_SIZE
    video = mo.stub_video(4, 8, 8)
    with tempfile.TemporaryDirectory() as tmp:
        slam = mo.stub_slam(video, mo.StubNet(), None, mo.GOLDEN_INTR, tmp)
        cfg = ro.refine_cfg("cuda:0")
        with pytest.raises(NotImplementedError):
            mapping.Mapper(cfg, None, slam)
        with pytest.raises(RuntimeError, match="CUDA"):
            mapping.RefiningMapper(ro.refine_cfg("cpu"), None, slam)
        m = mapping.RefiningMapper(cfg, None, slam)                          # accepted, no device touched
        assert m.BA and len(m.optimizer.param_groups) == 2
