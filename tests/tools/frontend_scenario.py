"""The tracking scenario of the Frontend / Backend drop-in test: keyframes appended one at a time to a DepthVideo and a
Frontend called after each, then one global dense_ba.  Run
  * by tests/golden/make_golden_frontend.py on the REFERENCE classes (src/frontend.py, src/backend.py,
    src/factor_graph.py, src/depth_video.py; CPU, natives from the oracle) -> tests/golden/frontend.npz, and
  * by tests/test_gpu_backend.py on goslam_b200.Frontend / Backend / FactorGraph / DepthVideo on the GPU.

The camera moves out along x and comes back to where it started, so loop closure finds edges between the last and the
first keyframes; two frames nearly repeat their predecessor, and the keyframe test removes one keyframe.  After every
Frontend call the graph and video state is snapshotted (the fields of fg_scenario.snapshot over the whole buffer),
with t1, the keyframe counter, last_loop_t, whether the call removed a keyframe, and the return value of every
loop_ba; the final dense_ba's return value and the video state after it close the record."""
import types

import numpy as np
import torch

from stub_update_op import update_op

HT8, WD8, BUFFER, WARMUP = 16, 24, 24, 6
# camera centre along x per appended frame: out to 0.42 and back; frames 7 and 11 nearly repeat their predecessor
CENTRES = [0.0, 0.07, 0.14, 0.21, 0.28, 0.35,          # warm-up
           0.42, 0.4215, 0.35, 0.28, 0.21, 0.2085, 0.14, 0.07, 0.0]
CFG_TRACKING = {
    "buffer": BUFFER, "warmup": WARMUP, "upsample": True, "beta": 0.75,
    "frontend": {"max_factors": 48, "nms": 1, "keyframe_thresh": 0.45, "window": 6, "thresh": 3.0, "radius": 1,
                 "enable_loop": True},
    "backend": {"thresh": 3.0, "radius": 1, "nms": 2, "loop_window": 6, "loop_thresh": 2.0, "loop_radius": 1,
                "loop_nms": 1},
}
DENSE_STEPS = 2


def cfg_and_args(device):
    cfg = {"cam": {"H_out": 8 * HT8, "W_out": 8 * WD8}, "mode": "rgbd", "verbose": False, "tracking": CFG_TRACKING}
    return cfg, types.SimpleNamespace(device=device)


def make_frames(seed=5):
    """the appended items (CPU tensors): (timestamp, image, pose, disp, depth, intrinsics, fmap, net, inp)"""
    g = torch.Generator().manual_seed(seed)
    n = len(CENTRES)
    low = torch.rand(n, 1, 4, 6, generator=g)
    disps = 0.45 + 0.4 * torch.nn.functional.interpolate(low, size=(HT8, WD8), mode="bilinear", align_corners=True)[:, 0]
    intr = torch.tensor([0.9 * WD8, 0.9 * WD8, WD8 / 2.0 - 0.3, HT8 / 2.0 + 0.2])
    frames = []
    for k, cx in enumerate(CENTRES):
        pose = torch.tensor([-cx, 0.01 * np.sin(k), 0.0, 0.0, 0.0, 0.0, 1.0], dtype=torch.float32)
        th = 0.004 * k * (1 if k < 7 else -1)                       # a slight yaw, world -> camera
        pose[4], pose[6] = np.sin(th / 2), np.cos(th / 2)
        depth = (1.0 / disps[k]).repeat_interleave(8, 0).repeat_interleave(8, 1)
        depth[torch.rand(8 * HT8, 8 * WD8, generator=g) < 0.05] = 0.0           # missing sensor readings
        frames.append((float(k), torch.zeros(3, 8 * HT8, 8 * WD8), pose, None, depth, intr.clone(),
                       torch.randn(1, 128, HT8, WD8, generator=g).half(),
                       (0.5 * torch.randn(128, HT8, WD8, generator=g)).half(),
                       (0.5 * torch.randn(128, HT8, WD8, generator=g)).half()))
    return frames


def snapshot(graph, video, tag, out):
    def put(name, t):
        out["%s_%s" % (tag, name)] = t.detach().cpu().numpy().copy()
    for k in ("ii", "jj", "age", "ii_inac", "jj_inac", "ii_bad", "jj_bad"):
        put(k, getattr(graph, k))
    put("poses", video.poses)
    put("disps", video.disps)
    put("target", graph.target[0, :, ::3, ::3])
    put("weight", graph.weight[0, :, ::3, ::3])
    put("target_inac", graph.target_inac[0, :, ::3, ::3])
    put("damping", graph.damping[:, ::2, ::2])
    put("disps_up", video.disps_up[:, ::16, ::16])


def run(Frontend, video, device, frames=None):
    """returns {name: array}; per Frontend call c: f<cc>_<field> snapshots and f<cc>_{t1, counter, last_loop_t, removed}"""
    frames = make_frames() if frames is None else frames
    cfg, args = cfg_and_args(device)
    net = types.SimpleNamespace(update=update_op)
    fe = Frontend(net, video, args, cfg)
    loops = []
    real_loop_ba = fe.loop_closing.loop_ba

    def loop_ba(*a, **k):
        r = real_loop_ba(*a, **k)
        loops.append(r)
        return r
    fe.loop_closing.loop_ba = loop_ba
    out = {}
    for c, item in enumerate(frames):
        video.append(*[x.to(device) if isinstance(x, torch.Tensor) else x for x in item])
        before = video.counter.value
        n_loops = len(loops)
        fe()
        tag = "f%02d" % c
        snapshot(fe.graph, video, tag, out)
        out[tag + "_t1"] = np.int64(fe.t1)
        out[tag + "_counter"] = np.int64(video.counter.value)
        out[tag + "_last_loop_t"] = np.int64(fe.last_loop_t)
        out[tag + "_removed"] = np.int64(before - video.counter.value)
        out[tag + "_loops"] = np.array(loops[n_loops:], np.int64).reshape(-1, 2)
    out["n_calls"] = np.int64(len(frames))
    n = video.counter.value
    out["dense_ba"] = np.array(fe.loop_closing.dense_ba(0, n, steps=DENSE_STEPS), np.int64)
    out["final_poses"] = video.poses.detach().cpu().numpy().copy()
    out["final_disps"] = video.disps.detach().cpu().numpy().copy()
    out["final_dirty"] = video.dirty.detach().cpu().numpy().copy()
    return out
