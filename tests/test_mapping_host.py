"""CPU checks of the mapping process: the restatement (oracle/mapping_oracle.py) reproduces the reference's own
Mapper.__call__, build_rays, build_all_rays and random_select (tests/golden/mapping.npz) bit for bit; the host planner
of goslam_b200.mapping gives the reference's frame lists, branches and offsets; the C entries reject bad arguments
without touching a device."""
import ctypes
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import mapping_oracle as mo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mapping.npz")
EINVAL, EWORKSPACE = -1, -3


def load_golden():
    g = dict(np.load(GOLDEN))
    S = mo.GOLDEN_SIZE
    n = S["buffer"] * S["ht"] * S["wd"]
    g["in_mask_filtered"] = np.unpackbits(g["in_mask_filtered"])[:n].reshape(S["buffer"], S["ht"], S["wd"]).astype(
        np.float32)
    return g


def run_oracle(g, device="cpu"):
    """the restated schedule over the golden calls with a recording optimize_map"""
    from goslam_b200 import lietorch
    S = mo.GOLDEN_SIZE
    video = mo.video_from_golden(g, device)
    batches, calls = [], []

    def record(sched, rays_o, rays_d, rays_color, rays_depth, optimizer, n):
        batches.append((len(calls), rays_o, rays_d, rays_depth, rays_color))

    slam = mo.stub_slam(video, mo.StubNet(device), None, mo.GOLDEN_INTR, None)
    sched = mo.MapperSchedule(mo.mapping_cfg(device, S["pixels"], S["window"], S["iters"]), slam, lietorch.SE3, record)
    np.random.seed(S["seed"])
    torch.manual_seed(S["seed"])
    trained = []
    for cur, the_end in mo.GOLDEN_CALLS:
        video.filtered_id[0] = cur
        trained.append(sched(the_end=the_end))
        calls.append((video.update_priority.cpu().numpy().copy(), sched.last_visit, sched.init))
    return sched, batches, calls, trained


def test_oracle_reproduces_reference_golden():
    g = load_golden()
    sched, batches, calls, _ = run_oracle(g)
    assert [b[0] for b in batches] == g["batch_call"].tolist()
    assert [len(b[1]) for b in batches] == g["batch_rows"].tolist()
    for i, k in enumerate(("rays_o", "rays_d", "depth", "color")):
        got = torch.cat([b[i + 1] for b in batches]).numpy()
        assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), g["batch_" + k].view(np.int32)), k
    assert [len(d) for d in sched.draws] == g["draw_sizes"].tolist()
    assert np.array_equal(torch.cat(sched.draws).numpy(), g["draws"])
    for c, (prio, last_visit, init) in enumerate(calls):
        assert np.array_equal(prio.view(np.int32), g["call_priority"][c].view(np.int32)), c
        assert last_visit == g["call_last_visit"][c] and init == g["call_init"][c], c


def test_golden_covers_the_scenario():
    g = load_golden()
    S = mo.GOLDEN_SIZE
    counts = g["in_mask_filtered"].reshape(S["buffer"], -1).sum(1)
    n_unvisit = S["pixels"] // S["window"]
    assert (counts == 0).any() and (counts == 2 * n_unvisit).any() and ((counts > 0) & (counts < 2 * n_unvisit)).any()
    assert not np.array_equal(g["in_pose_compensate"][0], [0, 0, 0, 0, 0, 0, 1])
    assert g["call_init"].tolist() == [True, False, False, False, False]
    assert g["call_the_end"].any() and (g["call_last_visit"] > 0).any()
    sched, _, _, trained = run_oracle(g)
    assert not all(t for call in trained for t in call)                  # some batches are under 100 rays
    assert any(len(set(f)) < len(f) for f, _ in sched.frame_lists)        # repeated frames in a list


def test_build_all_rays_and_random_select_match_reference():
    g = load_golden()
    S = mo.GOLDEN_SIZE
    ro, rd = mo.build_all_rays(S["ht"], S["wd"], *mo.GOLDEN_INTR, torch.from_numpy(g["img_c2w"]), "cpu")
    assert np.array_equal(ro.numpy(), g["img_rays_o"]) and np.array_equal(rd.numpy(), g["img_rays_d"])
    from goslam_b200 import mapping
    for fn in (mo.random_select, mapping.random_select):
        np.random.seed(3)
        sel = [fn(l, k) for l, k in ((6, 2), (10, 10), (37, 10), (100, 10))]
        assert [len(s) for s in sel] == g["select_sizes"].tolist()
        assert np.concatenate([np.array(s, np.int64) for s in sel]).tolist() == g["select"].tolist()


def test_host_planner_gives_reference_lists_branches_and_offsets():
    """replays Mapper.__call__'s list building with goslam_b200.mapping's planner and checks every iteration's frame
    list, n_rays, batch size and draw sizes against the restated schedule on the golden"""
    from goslam_b200 import mapping
    g = load_golden()
    S = mo.GOLDEN_SIZE
    sched, batches, _, trained = run_oracle(g)
    counts = g["in_mask_filtered"].reshape(S["buffer"], -1).sum(1).astype(int).tolist()
    np.random.seed(S["seed"])
    lists, last_visit, init, prio = [], 0, True, g["in_update_priority"]
    for c, (cur, the_end) in enumerate(mo.GOLDEN_CALLS):
        if cur <= 1:
            continue
        iters = S["iters"] * (10 if the_end else 1)
        unvisit = list(range(last_visit, cur))
        order = torch.sort(torch.from_numpy(prio[:last_visit]), descending=True)[1].numpy() if last_visit > 0 else None
        visit = mapping.visit_frames(cur, last_visit, order, S["window"])
        if len(unvisit) > 2:
            last_visit = cur
            for _ in range(iters * 10 if init else iters):
                sub = list(np.random.choice(unvisit, S["window"]))
                lists.append((sub, S["pixels"] // len(sub)))
        lists += [(visit, S["pixels"] // len(visit))] * iters
        init = False
        prio = g["call_priority"][c]
    assert [([int(f) for f in fl], n) for fl, n in lists] == sched.frame_lists
    rows = iter(g["batch_rows"].tolist())
    draw_sizes = iter(g["draw_sizes"].tolist())
    flat = [t for call in trained for t in call]
    for (frames, n_rays), was_trained in zip(lists, flat):
        plan = mapping.plan_batch([counts[f] for f in frames], n_rays)
        assert plan.R == sum(plan.rows) and plan.offsets == list(np.cumsum([0] + plan.rows[:-1]))
        assert was_trained == (plan.R >= 100)
        if was_trained:
            assert plan.R == next(rows)
        assert [d for d in plan.draw if d > 0] == [next(draw_sizes) for d in plan.draw if d > 0]
    assert next(rows, None) is None and next(draw_sizes, None) is None


def test_plan_batch_rule():
    from goslam_b200 import mapping
    p = mapping.plan_batch([0, 19, 20, 21, 22, 500], 10)
    assert p.draw == [0, 0, 0, 0, 10, 10] and p.rows == [0, 19, 20, 21, 10, 10]
    assert p.offsets == [0, 0, 19, 39, 60, 70] and p.R == 80 and p.n_draws == 20
    assert mapping.plan_batch([50], 0).draw == [0]
    assert mapping.distinct_frames([5, 4, 5, 1, 4, 5]) == ([5, 4, 1], [3, 2, 1])


def test_entry_points_reject_bad_arguments(lib):
    ws = lib.goslam_mapping_snapshot_workspace_bytes
    assert ws(0, 8, 8) == 0 and ws(-1, 8, 8) == 0 and ws(2, 0, 8) == 0 and ws(2, 8, -1) == 0
    assert ws(65536, 8, 8) == 0 and ws(1, 1 << 14, 1 << 13) == 0
    t = (1024 * 3 + 1023) // 1024
    want = 2 * (-(-4 * 2 * t // 256) * 256) + (-(-4 * 2 * 3072 // 256) * 256) + 16 * 2 * 3072
    assert ws(2, 32, 96) == want
    assert 0 < ws(2, 8, 8) < ws(3, 8, 8) < ws(3, 16, 8)

    def snap(F, H, W, nbytes=1 << 20, buffer=4):
        return lib.goslam_mapping_snapshot(*([None] * 4), buffer, H, W, None, None, F, 0.8, None,
                                           ctypes.c_size_t(nbytes), None, None)

    for args in ((-1, 8, 8), (2, 0, 8), (2, 8, -1), (70000, 8, 8)):
        assert snap(*args) == EINVAL, args
    assert snap(2, 8, 8, buffer=0) == EINVAL
    assert snap(0, 8, 8) == 0                                              # nothing to do
    p = ctypes.c_void_p(16)
    assert lib.goslam_mapping_snapshot(p, p, p, p, 4, 8, 8, p, p, 2, 0.8, None, ctypes.c_size_t(1 << 20), p,
                                       None) == EWORKSPACE
    assert lib.goslam_mapping_snapshot(p, p, p, p, 4, 8, 8, p, p, 2, 0.8, p, ctypes.c_size_t(ws(2, 8, 8) - 1), p,
                                       None) == EWORKSPACE

    arr = ctypes.c_int * 3

    def rays(slots, counts, draw, n_draws=100, max_rays=1000, workspace=p, nbytes=1 << 20, F=2):
        return lib.goslam_mapping_rays(workspace, ctypes.c_size_t(nbytes), F, 8, 8, p, p, n_draws, 3, arr(*slots),
                                       arr(*counts), arr(*draw), 1.0, 1.0, 0.0, 0.0, p, p, p, p, max_rays, None)

    assert rays([0, 1, 2], [4, 4, 4], [0, 0, 0]) == EINVAL                 # slot outside the snapshot
    assert rays([0, 1, -1], [4, 4, 4], [0, 0, 0]) == EINVAL
    assert rays([0, 1, 1], [4, 65, 4], [0, 0, 0]) == EINVAL                # N_f beyond H*W
    assert rays([0, 1, 1], [4, 0, 4], [0, 2, 0]) == EINVAL                 # draws from an empty frame
    assert rays([0, 1, 1], [4, 4, 4], [0, -1, 0]) == EINVAL
    assert rays([0, 1, 1], [40, 40, 40], [0, 0, 0], max_rays=119) == EINVAL   # outputs too short
    assert rays([0, 1, 1], [40, 40, 40], [5, 5, 0], n_draws=9) == EINVAL      # draw buffer too short
    assert rays([0, 1, 1], [40, 40, 40], [5, 5, 0], workspace=None) == EWORKSPACE
    assert rays([0, 1, 1], [40, 40, 40], [5, 5, 0], nbytes=ws(2, 8, 8) - 1) == EWORKSPACE
    assert rays([0, 1, 1], [0, 0, 0], [0, 0, 0]) == 0                       # empty batch: no launch
    assert lib.goslam_mapping_all_rays(p, 0, 8, 1.0, 1.0, 0.0, 0.0, p, p, None) == EINVAL
    assert lib.goslam_mapping_all_rays(None, 8, 8, 1.0, 1.0, 0.0, 0.0, p, p, None) == EINVAL


def test_mapper_needs_cuda_and_rejects_camera_refinement():
    from goslam_b200 import mapping
    S = mo.GOLDEN_SIZE
    video = mo.stub_video(4, 8, 8)
    with tempfile.TemporaryDirectory() as tmp:
        slam = mo.stub_slam(video, mo.StubNet(), None, mo.GOLDEN_INTR, tmp)
        with pytest.raises(RuntimeError, match="CUDA"):
            mapping.Mapper(mo.mapping_cfg("cpu", S["pixels"], S["window"], 1), None, slam)
        cfg = mo.mapping_cfg("cuda:0", S["pixels"], S["window"], 1)
        cfg["mapping"]["BA"] = True
        with pytest.raises(NotImplementedError):
            mapping.Mapper(cfg, None, slam)
        with pytest.raises(RuntimeError, match="CUDA"):
            mapping.snapshot_frames(video, [1, 0], 0.8)
