"""Drop-in for src/trajectory_filler.py's PoseTrajectoryFiller: the poses of every (non-keyframe) frame, filled in
chunks of 16 against the keyframes in the video.

    from goslam_b200.trajectory_filler import PoseTrajectoryFiller   # instead of: from .trajectory_filler import ...

Same constructor, attributes and `__call__`.  Per chunk:
  - the chunk's images, depths and intrinsics are stacked and uploaded once;
  - fnet on every image (mono or stereo), with the reference's normalisation fused into the stem, written into
    video.fmaps[N:N+M];
  - one launch (goslam_fill_interpolate) brackets every frame between keyframes, interpolates its pose in SE3 and
    writes the frame's timestamp, pose, intrinsics / 8, disps and (with depth) disps_sens; t0 / t1 stay on the device
    and are the edge sources of `add_factors`;
  - the reference's two add_factors calls and 6 motion-only updates on goslam_b200.FactorGraph.
Chunks are not merged: the update operator averages hidden state over edges that share a source keyframe, so the
frames of one chunk are coupled and the chunking is part of the result.

Differences from the reference:
  - the caller's images are never written, and video.images receives them as given (the reference normalises the
    stacked chunk in place, so with a CUDA stream its video.images rows hold normalised images);
  - a timestamp before the first keyframe raises ValueError (the reference indexes ts[-1] and builds edges from frame
    -1), and so does a chunk that does not fit behind the keyframes (N + M > buffer; the reference fails on a shape
    mismatch part way through its writes).  Both are checked before the chunk writes anything.
"""
import torch

from . import _lib
from . import lietorch
from .factor_graph import FactorGraph
from .modules.extractor import EncoderPack, encode

CHUNK = 16


def fill_interpolate(video, N, tt, intrinsics, depths=None):
    """one launch: frames tt [M] (f32, device) bracketed between the video's keyframes 0..N-1, their poses interpolated
    and written with timestamp, intrinsics [M, 4] / 8, disps (and, with depths [M, H, W], disps_sens) into rows
    N..N+M of `video`.  Returns t0, t1 [M] (int64, device).  No host synchronisation."""
    dev = video.poses.device
    M = int(tt.shape[0])
    H, W = 8 * video.disps.shape[1], 8 * video.disps.shape[2]
    if tuple(intrinsics.shape) != (M, 4) or (depths is not None and tuple(depths.shape) != (M, H, W)):
        raise ValueError("fill_interpolate: intrinsics must be [%d, 4] and depths [%d, %d, %d], got %s and %s"
                         % (M, M, H, W, tuple(intrinsics.shape), None if depths is None else tuple(depths.shape)))
    tt = tt.to(dev, torch.float32).contiguous()
    intrinsics = intrinsics.to(dev, torch.float32).contiguous()
    depths = depths.to(dev, torch.float32).contiguous() if depths is not None else None
    t0 = torch.empty(M, dtype=torch.long, device=dev)
    t1 = torch.empty(M, dtype=torch.long, device=dev)
    _lib.call("fill_interpolate", video.timestamp, video.poses, video.intrinsics, video.disps, video.disps_sens, N, M, tt,
              intrinsics, depths, H, W, t0, t1)
    return t0, t1


class PoseTrajectoryFiller:
    """ This class is used to fill in non-keyframe poses """

    def __init__(self, net, video, device="cuda:0"):
        self.cnet = net.cnet
        self.fnet = net.fnet
        self.update = net.update

        self.count = 0
        self.video = video
        self.device = device

        self.MEAN = torch.tensor([0.485, 0.456, 0.406], device=device)[:, None, None]
        self.STDV = torch.tensor([0.229, 0.224, 0.225], device=device)[:, None, None]
        self._fpack = EncoderPack()

    def _feature_encoder(self, inputs):
        """inputs [b, 3, H, W] raw -> fmap f16 [b, 128, H/8, W/8]"""
        return encode(self._fpack.get(self.fnet), self.fnet.norm_fn, 128, inputs, self.MEAN, self.STDV)

    def _fill(self, timestamps, images, depths, intrinsics, ts_first):
        """one chunk (src/trajectory_filler.py:29-76)"""
        v = self.video
        N, M = v.counter.value, len(timestamps)
        buffer = v.poses.shape[0]
        tt = torch.tensor([float(t) for t in timestamps], dtype=torch.float32)   # the video's timestamp type
        if float(tt.min()) < ts_first:
            raise ValueError("PoseTrajectoryFiller: timestamp %r lies before the first keyframe (%r)"
                             % (float(tt.min()), ts_first))
        if N + M > buffer:
            raise ValueError("PoseTrajectoryFiller: %d keyframes + a chunk of %d frames exceed the video's buffer of %d"
                             % (N, M, buffer))
        dev = v.poses.device
        images = torch.stack(images, dim=0).to(dev)                               # [M, rig, 3, H, W]
        depths = torch.stack(depths, dim=0).to(dev) if depths is not None else None
        intrinsics = torch.stack(intrinsics, dim=0).to(dev)
        _, rig, _, H, W = images.shape

        fmap = self._feature_encoder(images.reshape(M * rig, 3, H, W))
        v.fmaps[N:N + M] = fmap.view(M, rig, 128, H // 8, W // 8)

        v.counter.value += M
        t0, t1 = fill_interpolate(v, N, tt.to(dev), intrinsics, depths)
        v.images[N:N + M] = images[:, 0]
        if depths is not None:
            v.depths_gt[N:N + M] = depths

        graph = FactorGraph(v, self.update, device=self.device)
        jj = torch.arange(N, N + M, device=dev)
        graph.add_factors(t0, jj)
        graph.add_factors(t1, jj)
        for _ in range(6):
            graph.update(N, N + M, motion_only=True)

        Gs = lietorch.SE3(v.poses[N:N + M].clone())
        v.counter.value -= M
        return [Gs]

    @torch.no_grad()
    def __call__(self, image_stream):
        """ fill in poses of non-keyframe images. """
        ts_first = None
        pose_list = []
        timestamps, images, depths, intrinsics = [], [], [], []

        def flush():
            nonlocal ts_first
            if ts_first is None:
                ts_first = float(self.video.timestamp[0])
            return self._fill(timestamps, images, depths if len(depths) > 0 else None, intrinsics, ts_first)

        for (timestamp, image, depth, intrinsic, gt_pose) in image_stream:
            timestamps.append(timestamp)
            images.append(image)
            if depth is not None:
                depths.append(depth)
            intrinsics.append(intrinsic)

            if len(timestamps) == CHUNK:
                pose_list += flush()
                timestamps, images, depths, intrinsics = [], [], [], []

        if len(timestamps) > 0:
            pose_list += flush()

        return lietorch.cat(pose_list, dim=0)
