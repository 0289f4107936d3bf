"""goslam_b200.MultiviewFilter on the GPU against the twin of the reference's forward (oracle/mvfilter_oracle.py)
running on this library's droid_backends.iproj / depth_filter, and against the reference-generated golden."""
import contextlib
import io
import types

import numpy as np
import pytest
import torch

from oracle import mvfilter_oracle as mv
from test_multiview_filter_host import _kernel_size, load_golden, load_pass_inputs

pytestmark = pytest.mark.gpu

STATE = ("poses_filtered", "disps_filtered", "mask_filtered", "update_priority", "filtered_id", "bound")


def dev():
    return torch.device("cuda:0")


def make_video(n, ht, wd, intrinsics):
    import goslam_b200
    cfg = {"cam": {"H_out": ht, "W_out": wd}, "mode": "mono", "tracking": {"buffer": n}}
    video = goslam_b200.DepthVideo(cfg, types.SimpleNamespace(device="cuda:0"))
    video.intrinsics[:] = torch.as_tensor(intrinsics, dtype=torch.float32, device=dev())
    return video


def make_pair(n, ht, wd, intrinsics, kernel_size, warmup):
    """(mirror on one DepthVideo, twin on another) with the same configuration"""
    import goslam_b200
    from goslam_b200 import droid_backends, lietorch
    vm, vt = make_video(n, ht, wd, intrinsics), make_video(n, ht, wd, intrinsics)
    args, slam_m = mv.stub_slam(vm, "cuda:0")
    _, slam_t = mv.stub_slam(vt, "cuda:0")
    cfg = mv.filter_cfg(kernel_size, warmup)
    return (vm, goslam_b200.MultiviewFilter(cfg, args, slam_m),
            vt, mv.MultiviewFilterTwin(cfg, args, slam_t, droid_backends.iproj, droid_backends.depth_filter, lietorch.SE3))


def state(video):
    torch.cuda.synchronize()
    return {k: getattr(video, k).detach().cpu().clone() for k in STATE}


def run(fn):
    """(raised exception type or None, console output)"""
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        try:
            fn()
        except Exception as e:  # noqa: BLE001
            return type(e), buf.getvalue()
    return None, buf.getvalue()


def ulp_diff(a, b):
    ia = a.numpy().view(np.int32).astype(np.int64)
    ib = b.numpy().view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return int(np.abs(ia - ib).max()) if ia.size else 0


def assert_same_state(sm, st, what):
    for k in STATE:
        if k == "update_priority":
            d = ulp_diff(sm[k], st[k])
            assert d <= 2, (what, k, d)
            if d:
                print("%s: update_priority differs by %d ulp" % (what, d))
        else:
            assert torch.equal(sm[k].view(torch.uint8), st[k].view(torch.uint8)), (what, k)


def set_ks(flt, twin, ks):
    flt.kernel_size = twin.kernel_size = ks


def test_golden_scenario_mirror_equals_twin():
    g = load_golden()
    n, ht, wd, warmup = [int(x) for x in g["size"]]
    vm, flt, vt, twin = make_pair(n, ht, wd, g["intrinsics"], 1, warmup)
    exact = True
    for p in range(len(g["counter"])):
        for v in (vm, vt):
            load_pass_inputs(v, g, p)
        set_ks(flt, twin, _kernel_size(g["kernel_size"][p]))
        before = state(vm)
        em, log_m = run(flt.forward)
        et, log_t = run(twin.forward)
        sm, st = state(vm), state(vt)
        assert_same_state(sm, st, "pass %d" % p)
        exact &= torch.equal(sm["update_priority"], st["update_priority"])
        assert log_m == log_t, (p, log_m, log_t)
        if g["raised"][p]:
            assert em is RuntimeError and et is IndexError, (p, em, et)
        else:
            assert em is None and et is None, (p, em, et)
        prev_id = int(g["out_filtered_id"][p - 1][0]) if p else -1
        if int(g["out_filtered_id"][p][0]) == prev_id:       # no-op, early return or empty point set
            assert_same_state(sm, before, "pass %d leaves the state untouched" % p)
            assert log_m == ""
    print("update_priority bit-identical on every pass: %s" % exact)


def test_golden_scenario_against_reference_golden():
    g = load_golden()
    n, ht, wd, warmup = [int(x) for x in g["size"]]
    vm, flt, _, _ = make_pair(n, ht, wd, g["intrinsics"], 1, warmup)
    for p in range(len(g["counter"])):
        load_pass_inputs(vm, g, p)
        flt.kernel_size = _kernel_size(g["kernel_size"][p])
        em, _ = run(flt.forward)
        assert (em is not None) == bool(g["raised"][p]), p
        sm = state(vm)
        assert np.array_equal(sm["filtered_id"].numpy(), g["out_filtered_id"][p]), p
        agree = (sm["mask_filtered"].numpy() == g["out_mask_filtered"][p]).mean()
        assert agree >= 0.995, (p, agree)
        assert np.array_equal(sm["disps_filtered"].numpy(), g["out_disps_filtered"][p]), p
        assert np.array_equal(sm["poses_filtered"].numpy(), g["out_poses_filtered"][p]), p


def seeded_scene(video, T, seed, compensate=True):
    ht, wd = video.disps_up.shape[1:]
    intr_full = tuple((video.intrinsics[0] * 8).tolist())
    tc, qc, w2c = mv.trajectory(T, seed)
    video.poses[:T] = w2c.to(dev())
    video.disps_up[:T] = mv.make_disps(tc, qc, intr_full, ht, wd, seed + 1, device=dev())
    video.pose_compensate[:] = mv.compensate_pose().to(dev()) if compensate else video.pose_compensate
    video.counter.value = T


@pytest.mark.parametrize("ht,wd,T,kernels", [
    (320, 640, 100, (1, 3)),          # Replica
    (320, 640, 200, ("inf", 5)),
    (240, 320, 400, (1, "inf")),      # ScanNet
])
def test_large_mirror_equals_twin(ht, wd, T, kernels):
    f = round(0.8 * wd * 8) / 8.0
    intr = [f / 8, f / 8, (wd - 1) / 16.0, (ht - 1) / 16.0]
    vm, flt, vt, twin = make_pair(T, ht, wd, intr, kernels[0], 8)
    for i, ks in enumerate(kernels):
        Tp = T - 2 + 2 * i                # second pass: more frames, new poses -> priority accumulates
        for v in (vm, vt):
            seeded_scene(v, Tp, 1000 + 17 * i + T)
        set_ks(flt, twin, ks)
        em, log_m = run(flt.forward)
        et, log_t = run(twin.forward)
        assert em is None and et is None
        sm, st = state(vm), state(vt)
        assert int(sm["filtered_id"][0]) == Tp, "pass did not commit"
        assert_same_state(sm, st, "T=%d kernel %s" % (Tp, ks))
        assert log_m == log_t
        m = sm["mask_filtered"][:Tp]
        assert 0 < float(m.mean()) < 1


def test_pass_is_deterministic():
    ht, wd, T = 320, 640, 100
    f = round(0.8 * wd * 8) / 8.0
    intr = [f / 8, f / 8, (wd - 1) / 16.0, (ht - 1) / 16.0]
    vm, flt, _, _ = make_pair(T, ht, wd, intr, 3, 8)
    seeded_scene(vm, T, 77)
    s0 = state(vm)
    outs = []
    for _ in range(2):
        for k, v in s0.items():
            getattr(vm, k).copy_(v.to(dev()))
        em, _ = run(flt.forward)
        assert em is None
        outs.append(state(vm))
    for k in STATE:
        assert torch.equal(outs[0][k].view(torch.uint8), outs[1][k].view(torch.uint8)), k


def test_radius_out_of_range_raises():
    vm, flt, _, _ = make_pair(16, 48, 64, [6.4, 6.4, 3.9375, 2.9375], 32, 8)
    seeded_scene(vm, 12, 5)
    before = state(vm)
    with pytest.raises(RuntimeError, match="mvfilter_compute"):
        flt.forward()
    assert_same_state(state(vm), before, "radius 16")
