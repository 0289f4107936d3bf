"""Generate tests/golden/mapping_refine.npz by running THE REFERENCE'S OWN Mapper.__call__ with mapping.BA: True
(src/mapping.py:151-300, camera refinement at :173-194, 266-273) on the CPU over oracle.mapping_oracle's golden scene,
with oracle.refine_oracle's schedule: calls before last_visit reaches 10 (no leaves), the first call that adds the
camera group, later calls that replace it (one with an unvisit pass while leaves exist), a the_end call, repeated
frames in the visit list and batches under 100 rays.

Stand-ins: lietorch and colorama as make_golden_mapping.py; mathutils -> a Matrix whose to_quaternion is
refine_oracle.matrix_to_quaternion; the renderer and net -> refine_oracle.StubRenderer / StubNet (smooth functions of
rays_o, rays_d and five parameters); torch.randint wrapped to record the draws (a device run replays them);
Tensor.get_device answers "cpu" for CPU tensors (quad2rotation allocates with .to(quad.get_device())).

Stored: per call the optimizer's group count, learning rates and last_visit; per training iteration the
loss, the batch size, the call, and every leaf after the step; the recorded draws.

Run:  python tests/golden/make_golden_refine.py      (needs the reference source tree, see make_golden.REF)
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

import make_golden as mg
from oracle import mapping_oracle as mo  # noqa: E402  (make_golden puts the repository on sys.path)
from oracle import refine_oracle as ro  # noqa: E402


class _Matrix:
    def __init__(self, R):
        self.R = np.asarray(R, np.float64)

    def to_quaternion(self):
        return ro.matrix_to_quaternion(self.R)


def main():
    mg.install_stubs()
    cm = types.ModuleType("colorama")
    cm.Fore = types.SimpleNamespace(MAGENTA="\x1b[35m")
    cm.Style = types.SimpleNamespace(RESET_ALL="\x1b[0m")
    sys.modules["colorama"] = cm
    mu = types.ModuleType("mathutils")
    mu.Matrix = _Matrix
    sys.modules["mathutils"] = mu
    ref_map = mg.ref_import("src.mapping")
    ref_dv = mg.ref_import("src.depth_video")
    torch.autograd.set_detect_anomaly(False)           # src/mapping.py turns it on at import; it changes no value

    S = mo.GOLDEN_SIZE
    video = mo.golden_video()
    video.get_mapping_item = types.MethodType(ref_dv.DepthVideo.get_mapping_item, video)
    cfg = ro.refine_cfg("cpu")

    draws, losses = [], []
    real_randint, real_backward, real_get_device = torch.randint, torch.Tensor.backward, torch.Tensor.get_device

    def randint(*a, **k):
        r = real_randint(*a, **k)
        draws.append(r.clone())
        return r

    def backward(self, *a, **k):
        losses.append(float(self.detach()))
        return real_backward(self, *a, **k)

    iters, calls = [], []
    with tempfile.TemporaryDirectory() as tmp:
        slam = mo.stub_slam(video, ro.StubNet(), ro.StubRenderer(), mo.GOLDEN_INTR, tmp)
        mapper = ref_map.Mapper(cfg, types.SimpleNamespace(), slam)
        real_optimize = mapper.optimize_map

        def optimize_map(rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters):
            real_optimize(rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters)
            groups = optimizer.param_groups
            leaves = torch.stack([q.detach().clone() for q in groups[2]['params']]) if len(groups) > 2 else None
            iters.append((len(calls), len(rays_o), losses[-1], leaves))

        mapper.optimize_map = optimize_map
        np.random.seed(S["seed"])
        torch.manual_seed(S["seed"])
        torch.randint, torch.Tensor.backward = randint, backward
        torch.Tensor.get_device = lambda t: "cpu" if t.device.type == "cpu" else real_get_device(t)
        try:
            for cur, the_end in ro.REFINE_CALLS:
                video.filtered_id[0] = cur
                mapper(the_end=the_end)
                groups = mapper.optimizer.param_groups
                calls.append((len(groups), [g['lr'] for g in groups], mapper.last_visit))
        finally:
            torch.randint, torch.Tensor.backward, torch.Tensor.get_device = real_randint, real_backward, real_get_device

    out = {
        "call_filtered_id": np.array([c[0] for c in ro.REFINE_CALLS], np.int64),
        "call_the_end": np.array([c[1] for c in ro.REFINE_CALLS], bool),
        "call_groups": np.array([c[0] for c in calls], np.int64),
        "call_lr": np.array([c[1] + [np.nan] * (3 - len(c[1])) for c in calls], np.float64),
        "call_last_visit": np.array([c[2] for c in calls], np.int64),
        "iter_call": np.array([i[0] for i in iters], np.int64),
        "iter_rows": np.array([i[1] for i in iters], np.int64),
        "iter_loss": np.array([i[2] for i in iters], np.float64),
        "iter_n_leaves": np.array([0 if i[3] is None else len(i[3]) for i in iters], np.int64),
        "iter_leaves": np.concatenate([i[3].numpy() for i in iters if i[3] is not None] or [np.zeros((0, 7), np.float32)]),
        "draw_sizes": np.array([len(d) for d in draws], np.int64),
        "draws": torch.cat(draws).numpy(),
    }
    path = os.path.join(mg.HERE, "mapping_refine.npz")
    np.savez_compressed(path, **out)
    print("iterations %d (leaves %s), groups per call %s, last_visit %s, draws %d -> %s (%d bytes)" % (
        len(iters), out["iter_n_leaves"].tolist(), out["call_groups"].tolist(), out["call_last_visit"].tolist(),
        len(draws), path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
