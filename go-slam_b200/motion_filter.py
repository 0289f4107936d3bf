"""Drop-in for src/motion_filter.py's MotionFilter: the per-frame keyframe gate of tracking on the encoder kernels.

    from goslam_b200.motion_filter import MotionFilter     # instead of: from .motion_filter import MotionFilter

Same constructor, attributes and `track` signature.  Per frame:
  - fnet on every image of the frame (mono or stereo), with the reference's normalisation fused into the stem;
  - the motion probe: the library's CorrBlock at coords0 plus `net.update`, one `.item()` for the threshold test
    (the only host synchronisation of the call).  Like the reference, `track` runs under CUDA autocast, so a
    reference `UpdateModule` with f32 weights takes the f16 context features;
  - cnet on the left image of an accepted frame, the tanh / relu context split fused into its last layer.
The encoders' weights are taken from `net.fnet` / `net.cnet` by parameter name, so the result is the same whether
those are the reference's modules or `goslam_b200.modules.extractor.BasicEncoder`.

Differences from the reference: the caller's image is never written (the reference's `sub_` / `div_` rewrite a CUDA
input in place), and H or W not a multiple of 8 raises.
"""
import torch

from . import lietorch
from .modules.corr import CorrBlock
from .modules.extractor import EncoderPack, encode


def coords_grid(ht, wd, device):
    y, x = torch.meshgrid(torch.arange(ht, device=device).float(), torch.arange(wd, device=device).float(),
                          indexing="ij")
    return torch.stack([x, y], dim=-1)


class MotionFilter:
    """ This class is used to filter incoming frames and extract features """

    def __init__(self, net, video, thresh=2.5, device="cuda:0"):
        self.cnet = net.cnet
        self.fnet = net.fnet
        self.update = net.update

        self.video = video
        self.thresh = thresh
        self.device = device

        self.count = 0

        self.MEAN = torch.tensor([0.485, 0.456, 0.406], device=device)[:, None, None]
        self.STDV = torch.tensor([0.229, 0.224, 0.225], device=device)[:, None, None]
        self._fpack, self._cpack = EncoderPack(), EncoderPack()

    def _feature_encoder(self, inputs):
        """inputs [b, 3, H, W] raw -> fmap f16 [b, 128, H/8, W/8]"""
        return encode(self._fpack.get(self.fnet), self.fnet.norm_fn, 128, inputs, self.MEAN, self.STDV)

    def _context_encoder(self, inputs):
        """inputs [1, 3, H, W] raw -> net = tanh, inp = relu, each f16 [1, 128, H/8, W/8]"""
        return encode(self._cpack.get(self.cnet), self.cnet.norm_fn, 256, inputs, self.MEAN, self.STDV, split=True)

    @torch.autocast("cuda")
    @torch.no_grad()
    def track(self, timestamp, image, depth=None, intrinsic=None, gt_pose=None):
        """ main update operation - run on every frame in video """
        scale_factor = 8.0
        IdentityMat = lietorch.SE3.Identity(1, ).data.squeeze()

        batch, _, imh, imw = image.shape
        ht, wd = imh // 8, imw // 8

        inputs = image.to(self.device)
        gmap = self._feature_encoder(inputs)  # [b, 128, ht, wd]

        left_idx = 0
        if self.video.counter.value == 0:
            net, inp = self._context_encoder(inputs[[left_idx]])
            self.net, self.inp, self.fmap = net, inp, gmap
            self.video.append(timestamp, image[left_idx], IdentityMat, 1.0, depth,
                              intrinsic / scale_factor, gmap, net[left_idx], inp[left_idx], gt_pose)

        else:
            coords0 = coords_grid(ht, wd, device=self.device)[None, None]
            corr = CorrBlock(self.fmap[None, [left_idx]], gmap[None, [left_idx]])(coords0)

            _, delta, weight = self.update(self.net[None], self.inp[None], corr)

            if delta.norm(dim=-1).mean().item() > self.thresh:
                self.count = 0
                net, inp = self._context_encoder(inputs[[left_idx]])
                self.net, self.inp, self.fmap = net, inp, gmap
                self.video.append(timestamp, image[left_idx], None, None, depth,
                                  intrinsic / scale_factor, gmap, net[left_idx], inp[left_idx], gt_pose)

            else:
                self.count += 1
