"""Camera refinement in mapping on the GPU (goslam_mapping_c2w_to_quadt, goslam_mapping_pose_rays,
goslam_mapping_pose_rays_backward through goslam_b200.mapping, and RefiningMapper):
  (1) c2w_to_quadt recovers every rotation, unit and w >= 0;
  (2) the pose-ray forward against the reference's quaternion_to_Rt + build_rays restated with torch ops on CUDA with the
      same generator state, at the golden, Replica and ScanNet sizes;
  (3) the backward against the float64 closed form, deterministic, independent of chunking, no host synchronisation;
  (4) the reference's refinement trajectory (tests/golden/neus_ray_grad.npz traj_*) through the new kernels;
  (5) RefiningMapper against the reference's own driver (tests/golden/mapping_refine.npz), equal to Mapper with
      refinement off, and end to end with the library's InstantNeuS and Renderer."""
import ctypes
import os
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle import mapping_oracle as mo
from oracle import neus_ray_grad_oracle as nro
from oracle import refine_oracle as ro

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
HERE = os.path.dirname(os.path.abspath(__file__))

SCENES = {   # name: (frames, H, W, pixels, window, intrinsics)
    "golden": (16, 16, 24, 140, 14, mo.GOLDEN_INTR),
    "replica": (22, 320, 640, 4400, 22, (320.0, 320.0, 319.5, 159.5)),
    "scannet": (22, 240, 320, 4400, 22, (289.8, 290.4, 158.3, 119.6)),
}


def make_video(name, seed=5):
    """frame 1 has no masked pixel, 2 has 3, 3 exactly 2 n_rays (all taken), 4 2 n_rays + 1 (drawn)"""
    n, H, W, pixels, window, _ = SCENES[name]
    video = mo.stub_video(n, H, W, DEV)
    g = torch.Generator().manual_seed(seed)
    video.pose_compensate[0] = mo.random_pose(g, 0.3)
    k = pixels // window
    mo.fill_frames(video, range(n), g, {1: 0, 2: 3, 3: 2 * k, 4: 2 * k + 1})
    return video


def frame_list(n, k, seed):
    rs = np.random.RandomState(seed)
    return [1, 2, 3, 4, 3] + list(rs.choice(n, k - 5))


def leaves_for(snap, fl, seed):
    """c2w_to_quadt of each entry's c2w, moved off the unit sphere and off the frame's pose (as AdamW moves them)"""
    from goslam_b200 import mapping
    q = mapping.c2w_to_quadt(snap.c2w[[snap.slot[int(f)] for f in fl]])
    g = torch.Generator().manual_seed(seed)
    noise = 0.05 * torch.randn(q.shape, generator=g)
    scale = 0.8 + 0.4 * torch.rand(len(fl), 1, generator=g)
    q = q + noise.to(DEV)
    q[:, :4] *= scale.to(DEV)
    return q.contiguous()


def ulp_err(got, want):
    norm = want.double().norm(dim=-1, keepdim=True)
    ulp = torch.pow(2.0, torch.floor(torch.log2(norm)) - 23)
    return ((got.double() - want.double()).abs() / ulp).max().item()


def _reference_batch(items, fl, quadt, n_rays, H, W, intr, rec):
    parts = [[], [], [], []]
    for e, f in enumerate(fl):
        image, depth, _, _, mask = items[int(f)]
        c2w = ro.quaternion_to_rt(quadt[e])
        for acc, t in zip(parts, mo.build_rays(n_rays, H, W, *intr, c2w, depth, image, DEV, mask, record=rec)):
            acc.append(t.float())
    return [torch.cat(p) for p in parts]


# ---- (1) ------------------------------------------------------------------------------------------------------------
def test_c2w_to_quadt_recovers_rotations():
    from goslam_b200 import lietorch, mapping
    g = torch.Generator().manual_seed(1)
    poses = torch.stack([mo.random_pose(g, 2.0) for _ in range(300)])
    c2w = lietorch.SE3(poses).inv().matrix().float()
    near = []                                              # rotations within 1e-6 of 180 degrees, every axis
    for axis in ([1, 0.01, 0.02], [0.01, 1, -0.02], [0.02, 0.01, 1], [0.4, -0.7, 0.5]):
        a = np.asarray(axis) / np.linalg.norm(axis)
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        for ang in (np.pi, np.pi - 1e-6, -(np.pi - 1e-6)):
            m = np.eye(4)
            m[:3, :3] = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K
            m[:3, 3] = a
            near.append(m)
    c2w = torch.cat([c2w, torch.tensor(np.stack(near), dtype=torch.float32), torch.eye(4)[None]]).to(DEV)
    q = mapping.c2w_to_quadt(c2w)
    assert q.shape == (len(c2w), 7) and q.dtype == torch.float32
    assert torch.all(q[:, 0] >= 0)
    assert torch.equal(q[:, 4:], c2w[:, :3, 3])
    R = nro.quat_to_rotation(q[:, :4].double())
    err = (R - c2w[:, :3, :3].double()).abs().max().item()
    print("max |quat_to_rotation(q) - R| = %.2e" % err)
    assert err <= 1e-6
    nrm = q[:, :4].double().norm(dim=1)
    assert ((nrm - 1.0).abs() <= 2 * 2.0 ** -23).all(), (nrm - 1).abs().max()
    assert torch.equal(mapping.c2w_to_quadt(c2w[5]), q[5])                 # a single [4,4]


# ---- (2) ------------------------------------------------------------------------------------------------------------
# rays_d bound: the kernel and torch compute R = quad2rotation(q) with the same f32 expressions, but torch's
# `(quad * quad).sum(-1)` may sum in another order and `2.0 / x` is a reciprocal times 2: each R entry may differ by
# up to 2 f32 ulps of 1, which moves a component of R dirs by at most 2^-22 (|dx| + |dy| + 1) <= 2^-22 sqrt(3) |dirs|,
# i.e. 4 sqrt(3) < 7 ulps of the ray's length (its ulp is at least 2^-24 of it); cuBLAS's unspecified summation order
# adds the 2 ulps test_gpu_mapping allows.  Hence 9.
RAYS_D_ULP = 9


@pytest.mark.parametrize("name", list(SCENES))
def test_pose_ray_batch_matches_reference_construction(name):
    from goslam_b200 import mapping
    from goslam_b200.depth_video import DepthVideo
    n, H, W, pixels, window, intr = SCENES[name]
    video = make_video(name)
    twin = make_video(name)
    snap = mapping.snapshot_frames(video, list(range(n)), 0.8)
    items = {f: DepthVideo.get_mapping_item(twin, f, DEV, decay=0.8) for f in range(n)}
    worst = 0.0
    for seed, k, n_rays in ((7, window, pixels // window), (8, 7, pixels // 7), (9, 90, pixels // 90), (10, 6, 0)):
        fl = frame_list(n, k, seed)                          # repeats, an empty frame, both branches; 90 > 64 entries
        quadt = leaves_for(snap, fl, seed)
        torch.cuda.manual_seed(seed)
        rec = []
        want = _reference_batch(items, fl, quadt, n_rays, H, W, intr, rec)
        state = torch.cuda.get_rng_state()
        torch.cuda.manual_seed(seed)
        b = mapping.build_pose_ray_batch(snap, fl, n_rays, intr, quadt)
        assert torch.equal(torch.cuda.get_rng_state(), state)
        assert torch.equal(b.draws, torch.cat(rec) if rec else b.draws[:0])
        assert torch.equal(b.rays_o, want[0]) and torch.equal(b.depth, want[2]) and torch.equal(b.color, want[3])
        e = ulp_err(b.rays_d, want[1])
        worst = max(worst, e)
        assert e <= RAYS_D_ULP, (seed, e)
        # the same draws as build_ray_batch: refinement does not move the random stream
        torch.cuda.manual_seed(seed)
        plain = mapping.build_ray_batch(snap, fl, n_rays, intr)
        assert torch.equal(plain.draws, b.draws) and torch.equal(plain.color, b.color)
    print("%s: rays_d within %.2f ulp of the ray length" % (name, worst))


# ---- (3) ------------------------------------------------------------------------------------------------------------
def _dirs_and_rows(snap, fl, n_rays, intr, draws):
    """the kernel's f32 directions per row (the forward under the identity leaf, exact) and the rows per entry"""
    from goslam_b200 import mapping
    eye = torch.zeros(len(fl), 7, device=DEV)
    eye[:, 0] = 1.0
    counts = [snap.counts[snap.slot[int(f)]] for f in fl]
    plan = mapping.plan_batch(counts, n_rays)
    _, dirs = _pose_forward(snap, fl, plan, draws, eye, intr)
    return dirs, plan


def _table(snap, fl, plan):
    arr = ctypes.c_int * len(fl)
    slots = [snap.slot[int(f)] for f in fl]
    counts = [snap.counts[s] for s in slots]
    return (len(fl), arr(*slots), arr(*counts), arr(*plan.draw))


def _pose_forward(snap, fl, plan, draws, quadt, intr):
    from goslam_b200 import _lib
    ro_ = torch.empty((plan.R, 3), device=DEV)
    rd = torch.empty((plan.R, 3), device=DEV)
    dep, col = torch.empty((plan.R,), device=DEV), torch.empty((plan.R, 3), device=DEV)
    _lib.call("mapping_pose_rays", snap.workspace, snap.workspace.numel(), len(snap.frames), snap.H, snap.W, quadt,
              draws, draws.numel(), *_table(snap, fl, plan), *intr, ro_, rd, dep, col, plan.R)
    return ro_, rd


def _pose_backward(snap, fl, plan, draws, quadt, intr, g_o, g_d):
    from goslam_b200 import _lib
    out = torch.full((len(fl), 7), float("nan"), device=DEV)
    _lib.call("mapping_pose_rays_backward", snap.workspace, snap.workspace.numel(), len(snap.frames), snap.H, snap.W,
              quadt, draws, draws.numel(), *_table(snap, fl, plan), *intr, g_o, g_d, plan.R, out)
    return out


@pytest.mark.parametrize("name", ["golden", "replica"])
def test_pose_backward_matches_float64_closed_form(name):
    from goslam_b200 import mapping
    n, H, W, pixels, window, intr = SCENES[name]
    video = make_video(name)
    snap = mapping.snapshot_frames(video, list(range(n)), 0.8)
    for seed, k, n_rays in ((3, window, pixels // window), (4, 90, pixels // 90), (5, 5, 0)):
        fl = frame_list(n, k, seed)
        quadt = leaves_for(snap, fl, seed).requires_grad_(True)
        torch.cuda.manual_seed(seed)
        b = mapping.build_pose_ray_batch(snap, fl, n_rays, intr, quadt)
        g = torch.Generator(device=DEV).manual_seed(seed)
        g_o = torch.randn(b.rays_o.shape, device=DEV, generator=g)
        g_d = torch.randn(b.rays_d.shape, device=DEV, generator=g)
        ((b.rays_o * g_o).sum() + (b.rays_d * g_d).sum()).backward()
        dirs, plan = _dirs_and_rows(snap, fl, n_rays, intr, b.draws)
        want = ro.pose_ray_backward(quadt.detach().cpu().numpy(), dirs.cpu().numpy(), plan.rows, g_o.cpu().numpy(),
                                    g_d.cpu().numpy())
        got = quadt.grad.cpu().numpy().astype(np.float64)
        assert quadt.grad.dtype == torch.float32
        worst = 0.0
        for e in range(len(fl)):
            nrm = np.linalg.norm(want[e])
            if plan.rows[e] == 0:
                assert np.all(got[e] == 0.0), e                          # N_f = 0: written, zero
                continue
            worst = max(worst, np.linalg.norm(got[e] - want[e]) / nrm)
            assert np.linalg.norm(got[e] - want[e]) <= 1e-5 * nrm, (e, got[e], want[e])
        print("%s seed %d: worst |d quadt - float64| / |d quadt| = %.2e" % (name, seed, worst))


def test_pose_backward_is_deterministic_chunk_independent_and_does_not_synchronise():
    from goslam_b200 import mapping
    n, H, W, pixels, window, intr = SCENES["replica"]
    video = make_video("replica")
    snap = mapping.snapshot_frames(video, list(range(n)), 0.8)
    fl = frame_list(n, 70, 12)
    n_rays = pixels // 70
    quadt = leaves_for(snap, fl, 12)
    torch.cuda.manual_seed(12)
    b = mapping.build_pose_ray_batch(snap, fl, n_rays, intr, quadt)
    plan = mapping.plan_batch([snap.counts[snap.slot[int(f)]] for f in fl], n_rays)
    g = torch.Generator(device=DEV).manual_seed(1)
    g_o = torch.randn(b.rays_o.shape, device=DEV, generator=g)
    g_d = torch.randn(b.rays_d.shape, device=DEV, generator=g)
    one = _pose_backward(snap, fl, plan, b.draws, quadt, intr, g_o, g_d)
    two = _pose_backward(snap, fl, plan, b.draws, quadt, intr, g_o, g_d)
    assert torch.equal(one, two)
    # the same 70 entries as three calls of 23, 1 and 46 entries (one launch each, other chunk boundaries)
    parts, e0, r0, d0 = [], 0, 0, 0
    for k in (23, 1, 46):
        sub = fl[e0:e0 + k]
        sp = mapping.plan_batch([snap.counts[snap.slot[int(f)]] for f in sub], n_rays)
        parts.append(_pose_backward(snap, sub, sp, b.draws[d0:d0 + sp.n_draws].contiguous(), quadt[e0:e0 + k].contiguous(),
                                    intr, g_o[r0:r0 + sp.R].contiguous(), g_d[r0:r0 + sp.R].contiguous()))
        e0, r0, d0 = e0 + k, r0 + sp.R, d0 + sp.n_draws
    assert torch.equal(torch.cat(parts), one)
    # autograd's backward is this kernel
    q = quadt.clone().requires_grad_(True)
    torch.cuda.manual_seed(12)
    b2 = mapping.build_pose_ray_batch(snap, fl, n_rays, intr, q)
    ((b2.rays_o * g_o).sum() + (b2.rays_d * g_d).sum()).backward()
    assert torch.equal(q.grad, one)
    # no host synchronisation in the forward or the backward
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            q.grad = None
            torch.cuda.manual_seed(12)                                     # host-side generator state
            b3 = mapping.build_pose_ray_batch(snap, fl, n_rays, intr, q)
            torch.autograd.backward([b3.rays_o, b3.rays_d], [g_o, g_d])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(q.grad, one)


# ---- (4) ------------------------------------------------------------------------------------------------------------
def test_reference_refinement_trajectory_through_the_pose_kernels():
    """neus_ray_grad.npz's 6-iteration refinement: rays from a snapshot of two full-mask frames through
    build_pose_ray_batch (all records, raster order) rather than pose_rays; the existing test's bounds"""
    from goslam_b200 import mapping
    import test_gpu_neus_ray_grad as t
    g = np.load(os.path.join(HERE, "golden", "neus_ray_grad.npz"))
    net = t._net(int(g["weights_seed"]), g["bound"].tolist(), g["rt_bound"])
    net_lr, grid_lr, cam_lr = g["traj_lr"].tolist()
    quadt = [torch.nn.Parameter(torch.from_numpy(q).to(DEV)) for q in g["traj_quadt0"]]
    opt = torch.optim.AdamW([{"params": net.get_training_parameters(), "lr": net_lr},
                             {"params": net.get_volume_parameters(), "lr": grid_lr}], betas=(0.9, 0.999), eps=1e-8,
                            weight_decay=0.01)
    opt.add_param_group({"params": quadt, "lr": cam_lr})
    train_params = net.get_training_parameters() + net.get_volume_parameters()
    cam = tuple(float(v) for v in g["traj_cam"])
    F, H, W = g["traj_depth"].shape
    video = mo.stub_video(F, H, W, DEV)
    video.images.copy_(torch.from_numpy(g["traj_color"]).permute(0, 3, 1, 2))
    video.disps_filtered.copy_(1.0 / torch.from_numpy(g["traj_depth"]))
    video.mask_filtered.fill_(1.0)
    snap = mapping.snapshot_frames(video, list(range(F)), 1.0)
    depth = torch.from_numpy(g["traj_depth"]).reshape(-1).to(DEV)
    color = torch.from_numpy(g["traj_color"]).reshape(-1, 3).to(DEV)
    S = 32
    n = F * H * W
    zv = torch.linspace(0.3, 3.4, S + 1)[:-1].reshape(1, S).repeat(n, 1).to(DEV)
    ds = torch.full((n, S), (3.4 - 0.3) / S, device=DEV)
    losses, leaves = [], []
    for it in range(g["traj_losses"].shape[0]):
        opt.zero_grad()
        with torch.enable_grad():
            b = mapping.build_pose_ray_batch(snap, list(range(F)), 0, cam, torch.stack(quadt))
            if it == 0:
                np.testing.assert_allclose(b.rays_d.detach().cpu().numpy(), g["traj_rays_d0"].reshape(-1, 3), atol=1e-6)
                assert torch.equal(b.color, color)
            out = net(b.rays_o, b.rays_d, zv, ds)
            total = t._loss(net, out, color, depth, False)
        total.backward()
        torch.nn.utils.clip_grad_norm_(train_params, max_norm=35.0)
        opt.step()
        losses.append(float(total.detach()))
        leaves.append(torch.stack([q.detach() for q in quadt]).cpu().numpy())
    want = g["traj_losses"]
    print("ours     :", " ".join("%.5f" % v for v in losses))
    print("reference:", " ".join("%.5f" % v for v in want))
    assert np.all(np.abs(np.array(losses) - want) <= 1e-2 * np.abs(want))
    dev_leaf = np.abs(np.stack(leaves) - g["traj_quadt"]).max(axis=(1, 2))
    print("max |quadt - reference| per iteration:", " ".join("%.2e" % v for v in dev_leaf))
    assert np.all(dev_leaf <= 1e-3), dev_leaf
    assert np.abs(g["traj_quadt"][-1] - g["traj_quadt0"]).max() > 1e-3


# ---- (5) ------------------------------------------------------------------------------------------------------------
def _golden_video_on_device():
    src = mo.golden_video()
    S = mo.GOLDEN_SIZE
    video = mo.stub_video(S["buffer"], S["ht"], S["wd"], DEV)
    for k in mo.INPUTS:
        getattr(video, k).copy_(getattr(src, k))
    return video


def _replay_draws(monkeypatch, mapping, g):
    """build_ray_batch / build_pose_ray_batch draw the recorded CPU torch.randint outputs in order"""
    sizes, flat = g["draw_sizes"].tolist(), torch.from_numpy(g["draws"])
    at = [0, 0]
    real = mapping._draw_batch

    def replay(snapshot, frame_list, n_rays):
        slots, counts, plan, draws = real(snapshot, frame_list, n_rays)
        pos = 0
        for d in plan.draw:
            if d > 0:
                assert sizes[at[0]] == d
                draws[pos:pos + d].copy_(flat[at[1]:at[1] + d])
                at[0] += 1
                at[1] += d
                pos += d
        return slots, counts, plan, draws

    monkeypatch.setattr(mapping, "_draw_batch", replay)
    return at


def _recording_mapper(cls, cfg, video, net, renderer, tmp, losses):
    mapper = cls(cfg, types.SimpleNamespace(), mo.stub_slam(video, net, renderer, mo.GOLDEN_INTR, tmp))
    iters, calls = [], []
    real = mapper.optimize_map

    def optimize_map(rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters):
        real(rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters)
        gr = optimizer.param_groups
        iters.append((len(calls), len(rays_o), losses[-1],
                      torch.stack([q.detach() for q in gr[2]['params']]).cpu().numpy() if len(gr) > 2 else None,
                      rays_o.detach().clone(), rays_d.detach().clone(), rays_depth.clone(), rays_color.clone()))

    mapper.optimize_map = optimize_map
    return mapper, iters, calls


def _loss_spy(monkeypatch):
    losses = []
    real_backward = torch.Tensor.backward

    def spy(self, *a, **k):
        if self.dim() == 0:
            losses.append(float(self.detach()))
        return real_backward(self, *a, **k)

    monkeypatch.setattr(torch.Tensor, "backward", spy)
    return losses


def test_refining_mapper_reproduces_reference_driver_golden(monkeypatch):
    from goslam_b200 import mapping
    g = np.load(os.path.join(HERE, "golden", "mapping_refine.npz"))
    at = _replay_draws(monkeypatch, mapping, g)
    losses = _loss_spy(monkeypatch)
    S = mo.GOLDEN_SIZE
    with tempfile.TemporaryDirectory() as tmp:
        mapper, iters, calls = _recording_mapper(mapping.RefiningMapper, ro.refine_cfg("cuda:0"),
                                                 _golden_video_on_device(), ro.StubNet(DEV), ro.StubRenderer(DEV), tmp,
                                                 losses)
        np.random.seed(S["seed"])
        torch.manual_seed(S["seed"])
        for cur, the_end in ro.REFINE_CALLS:
            mapper.video.filtered_id[0] = cur
            mapper(the_end=the_end)
            gr = mapper.optimizer.param_groups
            calls.append((len(gr), [x['lr'] for x in gr], mapper.last_visit))
    assert at[0] == len(g["draw_sizes"])
    assert [c[0] for c in calls] == g["call_groups"].tolist()
    assert [c[2] for c in calls] == g["call_last_visit"].tolist()
    np.testing.assert_array_equal(np.array([c[1] + [np.nan] * (3 - len(c[1])) for c in calls]), g["call_lr"])
    assert [i[0] for i in iters] == g["iter_call"].tolist() and [i[1] for i in iters] == g["iter_rows"].tolist()
    loss = np.array([i[2] for i in iters])
    lerr = (np.abs(loss - g["iter_loss"]) / np.abs(g["iter_loss"])).max()      # the zero-disparity pixels' depth
                                                                                # of 1e7 makes the losses large
    assert [0 if i[3] is None else len(i[3]) for i in iters] == g["iter_n_leaves"].tolist()
    got = np.concatenate([i[3] for i in iters if i[3] is not None])
    want = g["iter_leaves"]
    sign = np.sign(np.sum(got[:, :4] * want[:, :4], axis=1, keepdims=True))
    qerr = max(np.abs(got[:, :4] * sign - want[:, :4]).max(), np.abs(got[:, 4:] - want[:, 4:]).max())
    print("max |loss - reference| / |loss| %.2e, max |leaf - reference| %.2e" % (lerr, qerr))
    assert lerr <= 1e-4 and qerr <= 1e-5
    assert len(mapper.optimizer.state) == 2 + 14                          # the replaced groups' state was dropped


@pytest.mark.parametrize("ba", [False, True])
def test_refining_mapper_without_refinement_is_mapper(monkeypatch, ba):
    """BA off, or BA on over calls that end before last_visit reaches 10: the same batches and bit-identical network
    parameters as Mapper"""
    from goslam_b200 import mapping
    losses = _loss_spy(monkeypatch)
    schedule = [(1, False), (6, False), (10, True)] if ba else [(1, False), (6, False), (10, False), (11, False), (13, True)]
    runs = []
    for cls in (mapping.Mapper, mapping.RefiningMapper):
        cfg = ro.refine_cfg("cuda:0")
        cfg['mapping']['BA'] = ba and cls is mapping.RefiningMapper
        with tempfile.TemporaryDirectory() as tmp:
            net = ro.StubNet(DEV)
            mapper, iters, _ = _recording_mapper(cls, cfg, _golden_video_on_device(), net, ro.StubRenderer(DEV), tmp,
                                                 losses)
            np.random.seed(3)
            torch.manual_seed(3)
            for cur, the_end in schedule:
                mapper.video.filtered_id[0] = cur
                mapper(the_end=the_end)
            runs.append((iters, [p.detach().clone() for p in net.parameters()], len(mapper.optimizer.param_groups)))
    (a, pa, na), (b, pb, nb) = runs
    assert len(a) == len(b) > 5 and na == nb == 2
    for x, y in zip(a, b):
        assert x[:3] == y[:3] and x[3] is None and y[3] is None
        assert all(torch.equal(u, v) for u, v in zip(x[4:], y[4:]))
    assert all(torch.equal(u, v) for u, v in zip(pa, pb))


def test_refining_mapper_with_instant_neus_matches_reference_schedule(monkeypatch):
    import bench
    from goslam_b200 import lietorch, mapping
    import test_gpu_mapping as tm
    n, H, W, pixels, window, _ = SCENES["golden"]
    intr = (16.0, 16.0, 12.0, 8.0)
    video = tm.make_video("golden", seed=13, zero_frac=0.0, trans=0.4, pose=mo.exact_pose)
    video.pose_compensate[0] = mo.exact_pose(torch.Generator().manual_seed(3), 0.3)
    video.bound[0] = torch.tensor([[-2.0, 2.0]] * 3)
    cfg = mo.mapping_cfg("cuda:0", pixels, window, 1)
    cfg['mapping']['BA'] = True
    nets = [bench.make_renderer(DEV, 43)[0] for _ in range(2)]
    losses = {0: [], 1: []}
    real_backward = torch.Tensor.backward
    side = [0]

    def spy(self, *a, **k):
        if self.dim() == 0:
            losses[side[0]].append(float(self.detach()))
        return real_backward(self, *a, **k)

    monkeypatch.setattr(torch.Tensor, "backward", spy)
    tmp = tempfile.mkdtemp()
    v_ref = tm.clone_video(video)
    opt = torch.optim.AdamW([{'params': nets[1].get_training_parameters(), 'lr': 0.001},
                             {'params': nets[1].get_volume_parameters(), 'lr': 0.01}],
                            betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    sched = ro.RefineSchedule(cfg, mo.stub_slam(v_ref, nets[1], tm._renderer(H, W, intr), intr, tmp), lietorch.SE3,
                              lambda s, *a: mo.reference_optimize_map(s, *a), optimizer=opt)
    mapper = mapping.RefiningMapper(cfg, types.SimpleNamespace(), mo.stub_slam(video, nets[0], tm._renderer(H, W, intr),
                                                                               intr, tmp))
    for s, (runner, v) in enumerate(((sched, v_ref), (mapper, video))):
        side[0] = s
        np.random.seed(4)
        torch.manual_seed(4)
        for cur in (6, 10, 12, 13):
            v.filtered_id[0] = cur
            runner()
    a, b = np.array(losses[0]), np.array(losses[1])
    assert len(a) == len(b) > 10
    print("max relative loss difference %.2e" % (np.abs(a - b) / np.abs(b)).max())
    assert np.all(np.abs(a - b) <= 1e-4 * np.abs(b)), np.abs(a - b).max()
    assert len(mapper.optimizer.param_groups) == 3 and len(opt.param_groups) == 3
    ours = torch.stack([q.detach() for q in mapper.optimizer.param_groups[2]['params']])
    start = torch.stack(sched.calls[-1][2])
    assert (ours - start).abs().max() > 1e-4                                   # the leaves moved
