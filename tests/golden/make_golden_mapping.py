"""Generate tests/golden/mapping.npz by running THE REFERENCE'S OWN Mapper.__call__ (src/mapping.py:151-300),
build_rays / build_all_rays / random_select (src/nerf_func.py) and DepthVideo.get_mapping_item
(src/depth_video.py:153-173) on the CPU over oracle.mapping_oracle's golden scenario: a no-op call, an init call
(unvisit_factor x10), a call with last_visit > 0, a one-frame unvisit list and a the_end call, with an empty mask,
N_f < 2 n_rays, N_f == 2 n_rays, repeated frames, a non-identity pose_compensate and batches under 100 rays.

Stand-ins: lietorch -> go-slam_b200/lietorch.py (make_golden.install_stubs), colorama -> its escape codes, the
video -> oracle.mapping_oracle.stub_video with the reference's get_mapping_item bound to it, the net -> StubNet,
optimize_map -> a recorder of its batches.  torch.randint is wrapped to record the draws.  Masks are stored as bits.

Run:  python tests/golden/make_golden_mapping.py      (needs the reference source tree, see make_golden.REF)
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

import make_golden as mg
from oracle import mapping_oracle as mo  # noqa: E402  (make_golden puts the repository on sys.path)


def main():
    mg.install_stubs()
    cm = types.ModuleType("colorama")
    cm.Fore = types.SimpleNamespace(MAGENTA="\x1b[35m")
    cm.Style = types.SimpleNamespace(RESET_ALL="\x1b[0m")
    sys.modules["colorama"] = cm
    ref_map = mg.ref_import("src.mapping")
    ref_nerf = mg.ref_import("src.nerf_func")
    ref_dv = mg.ref_import("src.depth_video")

    S = mo.GOLDEN_SIZE
    video = mo.golden_video()
    inputs = mo.golden_inputs(video)
    video.get_mapping_item = types.MethodType(ref_dv.DepthVideo.get_mapping_item, video)
    cfg = mo.mapping_cfg("cpu", S["pixels"], S["window"], S["iters"])
    out = {"in_" + k: v for k, v in inputs.items()}
    out["in_mask_filtered"] = np.packbits(inputs["mask_filtered"].astype(bool))

    draws = []
    real_randint = torch.randint

    def randint(*a, **k):
        r = real_randint(*a, **k)
        draws.append(r.clone())
        return r

    batches, calls = [], []
    with tempfile.TemporaryDirectory() as tmp:
        slam = mo.stub_slam(video, mo.StubNet(), None, mo.GOLDEN_INTR, tmp)
        mapper = ref_map.Mapper(cfg, types.SimpleNamespace(), slam)

        def record(rays_o, rays_d, rays_color, rays_depth, optimizer, num_joint_iters):
            batches.append((len(calls), rays_o.clone(), rays_d.clone(), rays_depth.clone(), rays_color.clone()))

        mapper.optimize_map = record
        np.random.seed(S["seed"])
        torch.manual_seed(S["seed"])
        torch.randint = randint
        try:
            for cur, the_end in mo.GOLDEN_CALLS:
                video.filtered_id[0] = cur
                mapper(the_end=the_end)
                calls.append((video.update_priority.numpy().copy(), mapper.last_visit, mapper.init))
        finally:
            torch.randint = real_randint

    out["call_filtered_id"] = np.array([c[0] for c in mo.GOLDEN_CALLS], np.int64)
    out["call_the_end"] = np.array([c[1] for c in mo.GOLDEN_CALLS], bool)
    out["call_priority"] = np.stack([c[0] for c in calls])
    out["call_last_visit"] = np.array([c[1] for c in calls], np.int64)
    out["call_init"] = np.array([c[2] for c in calls], bool)
    out["batch_call"] = np.array([b[0] for b in batches], np.int64)
    out["batch_rows"] = np.array([len(b[1]) for b in batches], np.int64)
    for i, k in enumerate(("rays_o", "rays_d", "depth", "color")):
        out["batch_" + k] = torch.cat([b[i + 1] for b in batches]).numpy()
    out["draw_sizes"] = np.array([len(d) for d in draws], np.int64)
    out["draws"] = torch.cat(draws).numpy()

    # build_all_rays on one frame's c2w, and random_select on a few sizes
    c2w = video.get_mapping_item(7, "cpu", decay=1.0)[2]
    ro, rd = ref_nerf.build_all_rays(S["ht"], S["wd"], *mo.GOLDEN_INTR, c2w, "cpu", nerf_coordinate=False)
    out["img_c2w"], out["img_rays_o"], out["img_rays_d"] = c2w.numpy(), ro.numpy(), rd.numpy()
    np.random.seed(3)
    sel = [ref_nerf.random_select(l, k) for l, k in ((6, 2), (10, 10), (37, 10), (100, 10))]
    out["select_sizes"] = np.array([len(s) for s in sel], np.int64)
    out["select"] = np.concatenate([np.array(s, np.int64) for s in sel])

    path = os.path.join(mg.HERE, "mapping.npz")
    np.savez_compressed(path, **out)
    print("batches %d (rows %s), draws %d, calls %s -> %s (%d bytes)" % (
        len(batches), out["batch_rows"].tolist(), len(draws), out["call_last_visit"].tolist(), path,
        os.path.getsize(path)))


if __name__ == "__main__":
    main()
