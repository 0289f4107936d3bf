"""GPU checks of the mapping hand-over and ray sampling (csrc/mapping.cu, goslam_b200.mapping, Renderer.render_img)
against the restatement of the reference (oracle/mapping_oracle.py) run on CUDA with the same generator state, at the
golden scene, Replica (320x640, 22 frames, 4,400 pixels) and ScanNet (240x320) sizes:
  - snapshot records bit-identical to DepthVideo.get_mapping_item's image / depth / mask / c2w, update_priority decays
    bit-identical (repeated frames included);
  - drawn indices identical, rays_o / depth / color bit-identical, rays_d within 2 ulp of the ray's length (torch's
    `@` is cuBLAS, whose summation order is not specified; the kernel's order is fixed);
  - no host synchronisation in the batch build;
  - the Mapper's call schedule equal to the restated one; training with the real InstantNeuS agrees in loss;
  - render_img equal to the chunked build_all_rays + render_batch_ray."""
import copy
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle import mapping_oracle as mo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

SCENES = {   # name: (frames, H, W, pixels, window, intrinsics)
    "golden": (16, 16, 24, 140, 14, mo.GOLDEN_INTR),
    "replica": (22, 320, 640, 4400, 22, (320.0, 320.0, 319.5, 159.5)),
    "scannet": (22, 240, 320, 4400, 22, (289.8, 290.4, 158.3, 119.6)),
}


def make_video(name, seed=5, **fill):
    n, H, W, _, _, _ = SCENES[name]
    video = mo.stub_video(n, H, W, DEV)
    g = torch.Generator().manual_seed(seed)
    video.pose_compensate[0] = mo.random_pose(g, 0.3)
    counts = {1: 0, 2: 3, 3: 2 * (SCENES[name][3] // SCENES[name][4]), 4: 2 * (SCENES[name][3] // SCENES[name][4]) + 1}
    mo.fill_frames(video, range(n), g, counts, **fill)
    return video


def clone_video(video):
    c = copy.copy(video)
    for k, v in vars(video).items():
        if torch.is_tensor(v):
            setattr(c, k, v.clone())
    from multiprocessing import Value
    c.mapping = Value("i", 0)
    return c


def ulp_check(got, want, n_ulp=2):
    """|got - want| <= n_ulp f32 ulps of the ray's length, per component"""
    norm = want.double().norm(dim=-1, keepdim=True)
    ulp = torch.pow(2.0, torch.floor(torch.log2(norm)) - 23)
    err = ((got.double() - want.double()).abs() / ulp).max().item()
    assert err <= n_ulp, "rays_d off by %.2f ulp" % err


def frame_list(n, k, seed):
    rs = np.random.RandomState(seed)
    return [1, 2, 3, 4, 3] + list(rs.choice(n, k - 5))


@pytest.mark.parametrize("name", list(SCENES))
def test_snapshot_matches_get_mapping_item(name):
    from goslam_b200 import mapping
    from goslam_b200.depth_video import DepthVideo
    n, H, W, _, _, intr = SCENES[name]
    video = make_video(name)
    twin = clone_video(video)
    frames = frame_list(n, 22, 1) + list(range(n))            # a visit list with repeats, then every frame
    snap = mapping.snapshot_frames(video, frames, 0.8)
    items = {}
    for f in frames:
        items[int(f)] = DepthVideo.get_mapping_item(twin, int(f), DEV, decay=0.8)
    torch.cuda.synchronize()
    assert torch.equal(video.update_priority.view(torch.int32), twin.update_priority.view(torch.int32))
    assert snap.frames == mapping.distinct_frames(frames)[0]
    for f in snap.frames:
        image, depth, c2w, _, mask = items[f]
        sel = mask.reshape(-1).bool()
        assert snap.count(f) == int(sel.sum())
        assert torch.equal(snap.c2w[snap.slot[f]], c2w), f
        b = mapping.build_ray_batch(snap, [f], 0, intr)                # n_rays = 0: every record in raster order
        assert torch.equal(b.color, image.reshape(-1, 3)[sel]) and torch.equal(b.depth, depth.reshape(-1)[sel]), f
        assert torch.equal(b.rays_o, c2w[:3, 3].reshape(1, 3).expand(len(b.rays_o), 3)), f


def test_randint_into_slices_consumes_philox_as_randint():
    torch.cuda.manual_seed(123)
    want = [torch.randint(n, (k,), device=DEV) for n, k in ((1000, 200), (37, 5), (204800, 4400), (3, 1))]
    state = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(123)
    buf = torch.empty(3 + 200 + 5 + 4400 + 1, dtype=torch.int64, device=DEV)
    at = 3
    for (n, k), w in zip(((1000, 200), (37, 5), (204800, 4400), (3, 1)), want):
        buf[at:at + k].random_(0, n)
        assert torch.equal(buf[at:at + k], w)
        at += k
    assert torch.equal(torch.cuda.get_rng_state(), state)


def test_direction_arithmetic_is_torchs():
    """torch's CUDA `(x - cx) / fx` with Python floats multiplies by the reciprocal taken in double and rounded to f32
    (not 1.0f / (float)fx, not a true division); with c2w = identity the kernel's rays_d are those directions"""
    from goslam_b200 import mapping
    H, W = 7, 1280
    eye = torch.eye(4, device=DEV)
    for fx, fy, cx, cy in ((320.0, 320.0, 319.5, 159.5), (289.8, 290.4, 158.3, 119.6), (20.5, 19.25, 11.3, 7.6),
                           (517.3, 516.5, 318.6, 255.3)):
        x = torch.arange(0, W, dtype=torch.float32, device=DEV)
        rcp = torch.tensor(np.float32(1.0 / fx), device=DEV)
        assert torch.equal((x - cx) / fx, (x - np.float32(cx)) * rcp)
        _, rd = mapping.all_rays(H, W, (fx, fy, cx, cy), eye)
        _, want = mo.build_all_rays(H, W, fx, fy, cx, cy, eye, DEV)
        assert torch.equal(rd, want.reshape(-1, 3))


@pytest.mark.parametrize("name", list(SCENES))
def test_ray_batch_matches_build_rays(name):
    from goslam_b200 import mapping
    from goslam_b200.depth_video import DepthVideo
    n, H, W, pixels, window, intr = SCENES[name]
    video = make_video(name)
    twin = clone_video(video)
    snap = mapping.snapshot_frames(video, list(range(n)), 0.8)
    items = {f: DepthVideo.get_mapping_item(twin, f, DEV, decay=0.8) for f in range(n)}
    for seed, k in ((7, window), (8, 7), (9, 90)):               # 90 entries: more than one launch's 64
        fl = frame_list(n, k, seed)
        n_rays = pixels // len(fl)
        torch.cuda.manual_seed(seed)
        rec, parts = [], [[], [], [], []]
        for f in fl:
            image, depth, c2w, _, mask = items[int(f)]
            for acc, t in zip(parts, mo.build_rays(n_rays, H, W, *intr, c2w, depth, image, DEV, mask, record=rec)):
                acc.append(t.float())
        want = [torch.cat(p) for p in parts]
        state = torch.cuda.get_rng_state()
        torch.cuda.manual_seed(seed)
        b = mapping.build_ray_batch(snap, fl, n_rays, intr)
        assert torch.equal(torch.cuda.get_rng_state(), state)
        assert torch.equal(b.draws, torch.cat(rec) if rec else b.draws[:0])
        assert torch.equal(b.rays_o, want[0]) and torch.equal(b.depth, want[2]) and torch.equal(b.color, want[3])
        ulp_check(b.rays_d, want[1])


def test_batch_build_does_not_synchronise():
    from goslam_b200 import mapping
    n, H, W, pixels, window, intr = SCENES["replica"]
    video = make_video("replica")
    snap = mapping.snapshot_frames(video, list(range(n)), 0.8)
    fl = frame_list(n, window, 3)
    mapping.build_ray_batch(snap, fl, pixels // window, intr)          # warm-up (library load)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            b = mapping.build_ray_batch(snap, fl, pixels // window, intr)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(b.rays_o) > 0


def _recording_pair(name, the_video):
    from goslam_b200 import lietorch, mapping
    n, H, W, pixels, window, intr = SCENES[name]
    cfg = mo.mapping_cfg("cuda:0", pixels, window, 2)
    ours, theirs = [], []
    tmp = tempfile.mkdtemp()
    v_ours, v_theirs = the_video, clone_video(the_video)
    slam = mo.stub_slam(v_ours, mo.StubNet(DEV), None, intr, tmp)
    mapper = mapping.Mapper(cfg, types.SimpleNamespace(), slam)
    mapper.optimize_map = lambda rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters: ours.append(
        (len(calls_ours), rays_o, rays_d, rays_depth, rays_color))
    sched = mo.MapperSchedule(cfg, mo.stub_slam(v_theirs, mo.StubNet(DEV), None, intr, tmp), lietorch.SE3,
                              lambda s, ro, rd, rc, de, opt, k: theirs.append((len(calls_theirs), ro, rd, de, rc)))
    calls_ours, calls_theirs = [], []
    return mapper, sched, v_ours, v_theirs, ours, theirs, calls_ours, calls_theirs


@pytest.mark.parametrize("name", ["golden", "replica"])
def test_mapper_schedule_matches_reference_schedule(name):
    n = SCENES[name][0]
    video = make_video(name, seed=9)
    mapper, sched, v_ours, v_theirs, ours, theirs, calls_ours, calls_theirs = _recording_pair(name, video)
    schedule = [(1, False), (6, False), (10, False), (11, False), (n, False), (n, True)]
    for runner, v, calls in ((sched, v_theirs, calls_theirs), (mapper, v_ours, calls_ours)):
        np.random.seed(21)
        torch.manual_seed(21)
        for cur, the_end in schedule:
            v.filtered_id[0] = cur
            runner(the_end=the_end)
            calls.append((v.update_priority.clone(), runner.last_visit, runner.init))
    assert len(ours) == len(theirs) and [o[0] for o in ours] == [t[0] for t in theirs]
    for o, t in zip(ours, theirs):
        assert torch.equal(o[1], t[1]) and torch.equal(o[3], t[3]) and torch.equal(o[4], t[4])
        ulp_check(o[2], t[2])
    for a, b in zip(calls_ours, calls_theirs):
        assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and a[1:] == b[1:]
    assert all(len(o[1]) >= 100 for o in ours)                      # batches under 100 rays are skipped


def _renderer(H, W, intr, ray_batch_size=5e3):
    from goslam_b200.render import Renderer
    fx, fy, cx, cy = intr
    cfg = {'rendering': {'N_samples': 24, 'N_surface': 48, 'lindisp': False, 'perturb': 1.0}}
    return Renderer(cfg, None, types.SimpleNamespace(H=H, W=W, fx=fx, fy=fy, cx=cx, cy=cy),
                    ray_batch_size=ray_batch_size)


def test_training_with_instant_neus_matches_reference_loop(monkeypatch):
    import bench
    from goslam_b200 import lietorch, mapping
    name = "golden"
    n, H, W, pixels, window, _ = SCENES[name]
    intr = (16.0, 16.0, 12.0, 8.0)          # with exact rotations: exact ray directions, the same batches on both sides
    video = make_video(name, seed=13, zero_frac=0.0, trans=0.4, pose=mo.exact_pose)
    video.pose_compensate[0] = mo.exact_pose(torch.Generator().manual_seed(3), 0.3)
    video.bound[0] = torch.tensor([[-2.0, 2.0]] * 3)
    cfg = mo.mapping_cfg("cuda:0", pixels, window, 1)
    nets = [bench.make_renderer(DEV, 43)[0] for _ in range(2)]
    trained = nets[0].trainable_tensors()                     # the ones the renderer backward has gradients for
    start = [p.detach().clone() for p in trained]
    losses = {0: [], 1: []}
    real_backward = torch.Tensor.backward
    side = [0]

    def spy(self, *a, **k):
        if self.dim() == 0:
            losses[side[0]].append(float(self.detach()))
        return real_backward(self, *a, **k)

    monkeypatch.setattr(torch.Tensor, "backward", spy)
    tmp = tempfile.mkdtemp()
    v_ref = clone_video(video)
    opt = torch.optim.AdamW([{'params': nets[1].get_training_parameters(), 'lr': 0.001},
                             {'params': nets[1].get_volume_parameters(), 'lr': 0.01}],
                            betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    sched = mo.MapperSchedule(cfg, mo.stub_slam(v_ref, nets[1], _renderer(H, W, intr), intr, tmp), lietorch.SE3,
                              lambda s, *a: mo.reference_optimize_map(s, *a), optimizer=opt)
    mapper = mapping.Mapper(cfg, types.SimpleNamespace(), mo.stub_slam(video, nets[0], _renderer(H, W, intr), intr,
                                                                       tmp))
    for s, (runner, v) in enumerate(((sched, v_ref), (mapper, video))):
        side[0] = s
        np.random.seed(4)
        torch.manual_seed(4)
        for cur in (6, 10, 12):
            v.filtered_id[0] = cur
            runner()
    a, b = np.array(losses[0]), np.array(losses[1])
    assert len(a) == len(b) > 10
    assert np.all(np.abs(a - b) <= 1e-4 * np.abs(b)), np.abs(a - b).max()
    moved = [not torch.equal(p0, p) for p0, p in zip(start, trained)]
    assert all(moved)


def test_render_img_matches_chunked_reference():
    import bench
    from goslam_b200 import mapping
    H, W = 60, 80
    intr = (70.0, 71.5, 39.5, 29.5)
    net = bench.make_renderer(DEV, 43)[0]
    rend = _renderer(H, W, intr, ray_batch_size=1500)              # 4 chunks, the last one short
    g = torch.Generator().manual_seed(3)
    pose = mo.random_pose(g, 0.3)
    from goslam_b200 import lietorch
    c2w = lietorch.SE3(pose).inv().matrix().to(DEV)
    gt_depth = (0.5 + 2.0 * torch.rand(H, W, generator=g)).to(DEV)
    # the rays: the kernel against the reference's build_all_rays
    ro, rd = mapping.all_rays(H, W, intr, c2w)
    wo, wd = mo.build_all_rays(H, W, *intr, c2w, DEV)
    assert torch.equal(ro, wo.reshape(-1, 3))
    ulp_check(rd, wd.reshape(-1, 3))
    # the chunking: bit for bit against the restated render_img fed the same rays
    real = mo.build_all_rays
    torch.manual_seed(8)
    got = rend.render_img(net, c2w, DEV, gt_depth=gt_depth)
    try:
        mo.build_all_rays = lambda *a: (ro.reshape(H, W, 3), rd.reshape(H, W, 3))
        torch.manual_seed(8)
        want = mo.render_img(rend, net, c2w, DEV, gt_depth)
    finally:
        mo.build_all_rays = real
    assert set(got) == set(want) and got["gradient_error"].shape == want["gradient_error"].shape == (4,)
    for k in got:
        if torch.is_tensor(got[k]):
            assert torch.equal(got[k], want[k]), k
    # end to end against the reference's own rays, with a pose and intrinsics that make every direction exact (so
    # cuBLAS's order cannot show): every output bit-identical, z_vals included
    intr = (32.0, 32.0, 40.0, 30.0)
    rend = _renderer(H, W, intr, ray_batch_size=1500)
    c2w = lietorch.SE3(mo.exact_pose(torch.Generator().manual_seed(4), 0.3)).inv().matrix().to(DEV)
    torch.manual_seed(9)
    got = rend.render_img(net, c2w, DEV, gt_depth=gt_depth)
    torch.manual_seed(9)
    ref = mo.render_img(rend, net, c2w.cpu().numpy(), DEV, gt_depth)
    for k in got:
        if torch.is_tensor(got[k]):
            assert torch.equal(got[k], ref[k]), k
