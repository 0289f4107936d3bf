"""CPU checks of the multiview filter: the twin (oracle/mvfilter_oracle.py) reproduces the reference's own
MultiviewFilter.forward (tests/golden/multiview_filter.npz) bit for bit on every pass, and the three C entry points
reject bad arguments without touching a device."""
import contextlib
import ctypes
import io
import os

import numpy as np
import pytest
import torch

from oracle import geom_oracle
from oracle import mvfilter_oracle as mv

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multiview_filter.npz")
EINVAL, EWORKSPACE = -1, -3


def load_golden():
    return mv.golden_unpack(np.load(GOLDEN))


def _kernel_size(code):
    return "inf" if int(code) == 0 else int(code)


def load_pass_inputs(video, g, p):
    video.poses[:] = torch.from_numpy(g["in_poses"][p]).to(video.poses.device)
    video.disps_up[:] = torch.from_numpy(g["in_disps"][p]).to(video.disps_up.device)
    video.pose_compensate[:] = torch.from_numpy(g["in_compensate"][p]).to(video.pose_compensate.device)
    video.counter.value = int(g["counter"][p])


def test_twin_reproduces_reference_golden():
    from goslam_b200 import lietorch
    g = load_golden()
    n, ht, wd, warmup = [int(x) for x in g["size"]]
    video = mv.stub_video(n, ht, wd)
    video.intrinsics[:] = torch.from_numpy(g["intrinsics"])
    args, slam = mv.stub_slam(video, "cpu")
    for k, v in mv.numpy_state(video).items():
        assert np.array_equal(v, g["init_" + k]), k

    def iproj(poses, disps, intr):
        return torch.from_numpy(geom_oracle.iproj(poses.numpy(), disps.numpy(), intr.numpy()))

    def depth_filter(poses, disps, intr, ix, thresh):
        return torch.from_numpy(geom_oracle.depth_filter(poses.numpy(), disps.numpy(), intr.numpy(), ix.numpy(),
                                                         thresh.numpy()))

    for p in range(len(g["counter"])):
        load_pass_inputs(video, g, p)
        twin = mv.MultiviewFilterTwin(mv.filter_cfg(_kernel_size(g["kernel_size"][p]), warmup), args, slam,
                                      iproj, depth_filter, lietorch.SE3)
        buf = io.StringIO()
        raised = False
        with contextlib.redirect_stdout(buf):
            try:
                twin.forward()
            except IndexError:
                raised = True
        assert raised == bool(g["raised"][p]), p
        assert buf.getvalue() == str(g["log"][p]), p
        for k, v in mv.numpy_state(video).items():
            assert v.dtype == g["out_" + k].dtype
            assert np.array_equal(v.view(np.uint8), g["out_" + k][p].view(np.uint8)), (p, k)


def test_golden_covers_every_branch():
    g = load_golden()
    fid = g["out_filtered_id"][:, 0]
    committed = [p for p in range(len(fid)) if fid[p] == g["counter"][p] and (p == 0 or fid[p - 1] != fid[p])]
    assert sorted(set(int(k) for k in g["kernel_size"][committed])) == [0, 1, 2]
    assert bool(g["raised"].any())
    assert (g["out_update_priority"][-1] > 0).any()
    assert not np.array_equal(g["in_compensate"][-1][0], [0, 0, 0, 0, 0, 0, 1])
    assert (g["in_disps"] == 0).any()
    # no pixel near its frame's 0.01 * mean threshold, so the mean's rounding cannot flip a mask
    for p in range(len(g["counter"])):
        assert mv.threshold_margin_ok(torch.from_numpy(g["in_disps"][p][:int(g["counter"][p])]))


def test_entry_points_reject_bad_arguments(lib):
    ws = ctypes.c_size_t(1 << 20)
    assert lib.goslam_mvfilter_workspace_bytes(-1, 8, 8) == 0
    assert lib.goslam_mvfilter_workspace_bytes(4, 0, 8) == 0
    assert lib.goslam_mvfilter_workspace_bytes(4, 8, -2) == 0
    small = lib.goslam_mvfilter_workspace_bytes(4, 8, 8)
    assert 0 < small < lib.goslam_mvfilter_workspace_bytes(8, 8, 8) < lib.goslam_mvfilter_workspace_bytes(8, 16, 8)

    def compute(T, ht, wd, ks, nbytes=ws):
        return lib.goslam_mvfilter_compute(None, None, None, None, 0.01, 2, ks, T, ht, wd, None, nbytes, None)

    def commit(T, ht, wd, nbytes=ws):
        return lib.goslam_mvfilter_commit(None, None, None, nbytes, T, ht, wd, *([None] * 8))

    for args in ((-1, 8, 8, 1), (4, 0, 8, 1), (4, 8, 0, 1), (4, -3, 8, 1), (4, 8, 8, -1),
                 (4, 8, 8, 32), (4, 8, 8, 33), (70000, 8, 8, 1)):
        assert compute(*args) == EINVAL, args
    for args in ((-1, 8, 8), (4, 0, 8), (4, 8, -1)):
        assert commit(*args) == EINVAL, args
    # radius 15 (kernel 30 or 31) is the largest box; a missing workspace is reported, not dereferenced
    assert compute(4, 8, 8, 31, ctypes.c_size_t(0)) == EWORKSPACE
    assert compute(4, 8, 8, 30, ctypes.c_size_t(0)) == EWORKSPACE
    assert commit(4, 8, 8, ctypes.c_size_t(small - 1)) == EWORKSPACE


def test_mirror_needs_cuda():
    import goslam_b200
    video = mv.stub_video(4, 8, 8)
    args, slam = mv.stub_slam(video, "cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        goslam_b200.MultiviewFilter(mv.filter_cfg(1, 2), args, slam)
