"""The trajectory-filler scenario: 7 keyframes with uneven timestamp gaps in a small video (h/8 x w/8 = 16 x 24) and
three image streams, run
  * by tests/golden/make_golden_filler.py through the REFERENCE PoseTrajectoryFiller (src/trajectory_filler.py; CPU,
    natives stubbed by the oracle) -> tests/golden/trajectory_filler.npz, and
  * by tests/test_gpu_trajectory_filler.py through goslam_b200.PoseTrajectoryFiller on the GPU.
Everything is generated from seeds on the CPU, so both sides start from the same video and stream."""
import types

import torch

from stub_fnet import features

HT8, WD8 = 16, 24
H, W = 8 * HT8, 8 * WD8
BUFFER = 24
KF_T = (0, 3, 4, 9, 15, 22, 34)               # keyframe timestamps (frame indices), uneven gaps
NUM_FRAMES = 37                               # RGB-D stream: chunks of 16, 16 and 5; frames 35, 36 after the last keyframe
INTR = (100.0, 104.0, 95.5, 63.5)
MEAN = torch.tensor([0.485, 0.456, 0.406])[:, None, None]
STDV = torch.tensor([0.229, 0.224, 0.225])[:, None, None]
STREAMS = ("rgbd", "mono", "stereo")


def cfg_and_args(device, stereo=False):
    cfg = {"cam": {"H_out": H, "W_out": W}, "mode": "stereo" if stereo else "rgbd", "tracking": {"buffer": BUFFER}}
    return cfg, types.SimpleNamespace(device=device)


def images():
    """[NUM_FRAMES, 3, H, W] in [0, 1]: a smooth seeded field seen with a drift of one pixel per frame"""
    from oracle import encoder_oracle as eo
    return eo.sequence(H=H, W=W, seed=17, shifts=tuple(range(NUM_FRAMES)))


def depths():
    g = torch.Generator().manual_seed(18)
    d = 0.8 + 2.0 * torch.rand(NUM_FRAMES, H, W, generator=g)
    d[:, 3::16, 3::24] = 0.0                   # holes at sampled pixels: disps_sens keeps the 0
    return d


def _quat(axis, angle):
    axis = torch.tensor(axis, dtype=torch.float64)
    axis = axis / axis.norm()
    return torch.cat([torch.sin(torch.tensor(0.5 * angle)) * axis, torch.cos(torch.tensor([0.5 * angle]))])


def keyframe_poses():
    """w2c poses [7, 7] along a smooth path; keyframe 3's quaternion is stored negated (same rotation, qw < 0)"""
    out = []
    for k, t in enumerate(KF_T):
        q = _quat((0.3, 1.0, 0.2), 0.02 * t)
        if k == 3:
            q = -q
        out.append(torch.cat([torch.tensor([0.015 * t, -0.004 * t, 0.01 * t], dtype=torch.float64), q]))
    return torch.stack(out).float()


def fill_keyframes(video, stereo=False):
    """the keyframe rows 0..6 of a fresh video (reference or drop-in) and counter = 7"""
    dev = video.poses.device
    n = len(KF_T)
    g = torch.Generator().manual_seed(19)
    img = images()[list(KF_T)]
    rig = torch.stack([img, torch.flip(img, dims=[-1])], 1) if stereo else img[:, None]
    fm = features(((rig.reshape(-1, 3, H, W) - MEAN) / STDV)).view(n, rig.shape[1], 128, HT8, WD8)
    disps = 0.4 + 0.5 * torch.rand(n, HT8, WD8, generator=g)
    video.timestamp[:n] = torch.tensor(KF_T, dtype=torch.float32).to(dev)
    video.images[:n] = img.to(dev)
    video.poses[:n] = keyframe_poses().to(dev)
    video.disps[:n] = disps.to(dev)
    video.disps_sens[:n] = disps.to(dev)
    video.intrinsics[:n] = (torch.tensor(INTR) / 8.0).to(dev)
    video.fmaps[:n] = fm.to(dev)
    video.nets[:n] = (0.5 * torch.randn(n, 128, HT8, WD8, generator=g)).half().to(dev)
    video.inps[:n] = (0.5 * torch.randn(n, 128, HT8, WD8, generator=g)).half().to(dev)
    video.counter.value = n


def stream(kind, device="cpu"):
    """list of (timestamp, image [rig, 3, H, W], depth [H, W] or None, intrinsic [4], gt_pose) on `device`
      rgbd    frames 0..36, integer timestamps (on, between and after the keyframes), with depth: 16 + 16 + 5
      mono    25 float timestamps 0, 1.5, ..., 36, no depth: 16 + 9
      stereo  9 frames 3, 7, ..., 35, the right image the mirrored left, no depth: one chunk"""
    img, dep = images(), depths()
    intr = torch.tensor(INTR)
    if kind == "rgbd":
        items = [(f, img[f][None], dep[f], intr, None) for f in range(NUM_FRAMES)]
    elif kind == "mono":
        items = [(1.5 * f, img[int(1.5 * f)][None], None, intr, None) for f in range(25)]
    elif kind == "stereo":
        items = [(f, torch.stack([img[f], torch.flip(img[f], dims=[-1])]), None, intr, None) for f in range(3, 37, 4)]
    else:
        raise ValueError(kind)
    return [(t, i.to(device).clone(), None if d is None else d.to(device).clone(), k.to(device).clone(), g)
            for t, i, d, k, g in items]
