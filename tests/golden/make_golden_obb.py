"""Generate tests/golden/obb.npz by running THE REFERENCE'S OWN Mesher.update_param_from_mapping(the_end=True)
(src/mesher.py:242-281) on the CPU and recording what it hands to OrientedBoundingBox.compute_from_pointcloud.

Stand-ins for what the reference imports: droid_backends.iproj / depth_filter -> oracle.geom_oracle, lietorch ->
go-slam_b200/lietorch.py (both installed by make_golden.install_stubs); open3d, matplotlib and pyrender are empty
modules (the method only imports open3d); src.oriented_bounding_box.OrientedBoundingBox is a recording class.  The
scene is oracle.mvfilter_oracle's analytic surface with holes, far pixels and a non-identity pose_compensate.

Run:  python tests/golden/make_golden_obb.py      (needs the reference source tree, see make_golden.REF)
"""
import os
import sys
import types

import numpy as np
import torch

import make_golden as mg
from oracle import geom_oracle  # noqa: E402  (make_golden puts the repository on sys.path)
from oracle import mvfilter_oracle as mv  # noqa: E402

T, HT, WD, SEED = 10, 24, 32, 21


def main():
    mg.install_stubs()
    db = sys.modules["droid_backends"]
    db.iproj = lambda poses, disps, intr: torch.from_numpy(
        geom_oracle.iproj(poses.numpy(), disps.numpy(), intr.numpy()))
    db.depth_filter = lambda poses, disps, intr, ix, thresh: torch.from_numpy(
        geom_oracle.depth_filter(poses.numpy(), disps.numpy(), intr.numpy(), ix.numpy(), thresh.numpy()))
    for name in ("open3d", "matplotlib", "matplotlib.pyplot", "pyrender"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    obb = types.ModuleType("src.oriented_bounding_box")
    seen = {}

    class RecordingBox:
        def compute_from_pointcloud(self, pointcloud, extend=0.0):
            seen["sel_points"], seen["extend"] = np.array(pointcloud), extend

    obb.OrientedBoundingBox = RecordingBox
    sys.modules["src.oriented_bounding_box"] = obb
    ref = mg.ref_import("src.mesher")

    intr_full = mv.full_intrinsics(HT, WD)
    video = mv.stub_video(T + 2, HT, WD)
    video.intrinsics[:] = torch.tensor(intr_full, dtype=torch.float32) / 8
    video.pose_compensate[:] = mv.compensate_pose()
    tc, qc, w2c = mv.trajectory(T, SEED)
    video.poses[:T] = w2c
    video.disps_up[:T] = mv.make_disps(tc, qc, intr_full, HT, WD, SEED + 1)
    video.counter.value = T
    video.timestamp = torch.arange(T + 2, dtype=torch.float32)
    self_ = types.SimpleNamespace(shared_mapping_net=torch.nn.Linear(1, 1), video=video, device="cpu")
    out = ref.Mesher.update_param_from_mapping(self_, the_end=True)
    assert isinstance(out[3], RecordingBox) and out[1] == T - 1
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "obb.npz")
    np.savez_compressed(path, cur_idx=T, poses=video.poses.numpy(), disps_up=video.disps_up.numpy(),
                        intrinsics=video.intrinsics.numpy(), pose_compensate=video.pose_compensate.numpy(),
                        sel_points=seen["sel_points"], extend=np.float64(seen["extend"]),
                        kf_c2w=out[4].numpy())
    print("wrote", path, seen["sel_points"].shape)


if __name__ == "__main__":
    main()
