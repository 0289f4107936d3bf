"""Generate tests/golden/multiview_filter.npz by running THE REFERENCE'S OWN MultiviewFilter.forward
(src/multiview_filter.py:98-170) on the CPU over the pass schedule of oracle.mvfilter_oracle.GOLDEN_PASSES:
warmup and filtered_t >= cur_t no-ops, the < 100 early return, the empty in-bound set (the reference raises),
kernel_size 1 / 2 / 'inf', holes and a non-identity pose_compensate.

Stand-ins for what the reference imports: droid_backends.iproj / depth_filter -> oracle.geom_oracle, lietorch ->
go-slam_b200/lietorch.py (both installed by make_golden.install_stubs), colorama -> its two escape codes.
The file records the inputs of every pass and the committed state after it (layout: mvfilter_oracle.golden_pack).

Run:  python tests/golden/make_golden_mvfilter.py      (needs the reference source tree, see make_golden.REF)
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

import make_golden as mg
from oracle import geom_oracle  # noqa: E402  (make_golden puts the repository on sys.path)
from oracle import mvfilter_oracle as mv  # noqa: E402


def main():
    mg.install_stubs()
    db = sys.modules["droid_backends"]
    db.iproj = lambda poses, disps, intr: torch.from_numpy(
        geom_oracle.iproj(poses.numpy(), disps.numpy(), intr.numpy()))
    db.depth_filter = lambda poses, disps, intr, ix, thresh: torch.from_numpy(
        geom_oracle.depth_filter(poses.numpy(), disps.numpy(), intr.numpy(), ix.numpy(), thresh.numpy()))
    cm = types.ModuleType("colorama")
    cm.Fore = types.SimpleNamespace(CYAN="\x1b[36m")
    cm.Style = types.SimpleNamespace(RESET_ALL="\x1b[0m")
    sys.modules["colorama"] = cm
    ref = mg.ref_import("src.multiview_filter")

    S = mv.GOLDEN_SIZE
    n, ht, wd = S["buffer"], S["ht"], S["wd"]
    intr_full = mv.full_intrinsics(ht, wd)
    video = mv.stub_video(n, ht, wd)
    video.intrinsics[:] = torch.tensor(intr_full, dtype=torch.float32) / 8
    video.pose_compensate[:] = mv.compensate_pose()
    args, slam = mv.stub_slam(video, "cpu")

    def scene(seed):
        tc, qc, w2c = mv.trajectory(n, seed)
        return w2c, mv.make_disps(tc, qc, intr_full, ht, wd, seed + 1, fp16_exact=True)

    init = mv.numpy_state(video)
    passes = []
    g = torch.Generator().manual_seed(5)
    for p, (counter, ks, change) in enumerate(mv.GOLDEN_PASSES):
        if change == "base":
            video.poses[:], video.disps_up[:] = scene(100)
        elif change == "perturb":
            video.poses[:], video.disps_up[:] = scene(100 + 10 * p)
            video.pose_compensate[:] = mv.compensate_pose()
        elif change == "scramble":
            q = torch.randn(n, 4, generator=g)
            video.poses[:, 3:] = q / q.norm(dim=-1, keepdim=True)
        elif change == "flat":
            video.poses[:] = torch.tensor([0, 0, 0, 0, 0, 0, 1.0])
            video.disps_up[:] = 0.5
            video.pose_compensate[:] = torch.tensor([0, 0, 0, 0, 0, 0, 1.0])
        video.counter.value = counter
        flt = ref.MultiviewFilter(mv.filter_cfg(ks, S["warmup"]), args, slam)
        buf = io.StringIO()
        raised = False
        with contextlib.redirect_stdout(buf):
            try:
                flt.forward()
            except (IndexError, RuntimeError):
                raised = True
        assert raised == (change == "flat"), (p, raised)
        passes.append(dict(counter=counter, kernel_size=0 if ks == "inf" else ks, raised=raised, log=buf.getvalue(),
                           poses=video.poses.numpy().copy(), disps=video.disps_up.numpy().copy(),
                           compensate=video.pose_compensate.numpy().copy(), state=mv.numpy_state(video)))
        print("pass %d: counter %d kernel %s -> filtered_id %d raised %s mask %d" % (
            p, counter, ks, int(video.filtered_id[0]), raised, int(video.mask_filtered.sum())))
    out = mv.golden_pack(passes, init, video.intrinsics[0].numpy().copy(), [n, ht, wd, S["warmup"]])
    path = os.path.join(mg.HERE, "multiview_filter.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        raise SystemExit("needs the reference source tree at %s" % mg.REF)
    main()
