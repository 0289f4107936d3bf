"""DroidNet's BasicEncoder (src/modules/extractor.py) on the sm_90a encoder kernels (csrc/encoder.cu).

`BasicEncoder` and `ResidualBlock` keep the reference's submodules, so `state_dict` keys are the reference's and the
`fnet.*` / `cnet.*` entries of pretrained/droid.pth load with strict=True.  The whole forward is one library call
(goslam_basic_encoder).  Only the two configurations DroidNet uses run: norm_fn 'instance' (fnet) and 'none' (cnet).
"""
import ctypes

import torch
import torch.nn as nn

from .. import _lib

_NORMS = {"none": 0, "instance": 1}
DIM = 32


def _check_norm(norm_fn):
    if norm_fn in ("batch", "group"):
        raise NotImplementedError("BasicEncoder: norm_fn %r is not supported (DroidNet uses 'instance' and 'none')"
                                  % norm_fn)
    if norm_fn not in _NORMS:
        raise TypeError(norm_fn)


def _pack_conv(conv, kpad=None):
    """nn.Conv2d [cout, cin, ky, kx] -> f16 [cout, Kpad] with k = (ky * ks + kx) * cin + ci, bias f32 [cout]"""
    w = conv.weight.detach()
    cout = w.shape[0]
    w = w.permute(0, 2, 3, 1).reshape(cout, -1)
    if kpad is not None and kpad > w.shape[1]:
        w = torch.nn.functional.pad(w, (0, kpad - w.shape[1]))
    return w.half().contiguous(), conv.bias.detach().float().contiguous()


class EncoderPack:
    """Kernel-side weights of a BasicEncoder-shaped module (ours or the reference's), taken by submodule name and
    cached per parameter version (include/goslam_b200.h: goslam_encoder_weights)."""

    def __init__(self):
        self._key = None
        self._tensors = None
        self.weights = None

    def get(self, enc):
        params = list(enc.parameters())
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._key == key:
            return self.weights
        st = _lib.EncoderWeights()
        keep = []

        def put(slot, conv, kpad=None):
            w, b = _pack_conv(conv, kpad)
            keep.extend((w, b))
            slot.w, slot.b = w.data_ptr(), b.data_ptr()

        put(st.stem, enc.conv1, 160)
        blocks = [blk for layer in (enc.layer1, enc.layer2, enc.layer3) for blk in layer]
        for i, blk in enumerate(blocks):
            put(st.block[i][0], blk.conv1)
            put(st.block[i][1], blk.conv2)
            if blk.downsample is not None:
                put(st.block[i][2], blk.downsample[0])
        put(st.out, enc.conv2)
        self._key, self._tensors, self.weights = key, keep, st
        return st


def encode(weights, norm_fn, out_dim, image, mean=None, std=None, split=False):
    """image [B, 3, H, W] (CUDA, f32 or f16) -> f16 [B, out_dim, H/8, W/8], or with split (out_dim 256) the pair
    (tanh of channels 0-127, relu of channels 128-255).  mean / std [3] apply (x - mean) / std before the stem."""
    _lib.need_cuda("BasicEncoder", image)
    B, C, H, W = image.shape
    if C != 3 or H % 8 or W % 8:
        raise ValueError("BasicEncoder: image must be [B, 3, H, W] with H and W multiples of 8, got %s"
                         % (tuple(image.shape),))
    if image.dtype not in (torch.float16, torch.float32):
        image = image.float()
    image = image.contiguous()
    dev = image.device
    norm = _NORMS[norm_fn]
    if split:
        out = torch.empty((B, 128, H // 8, W // 8), dtype=torch.float16, device=dev)
        out2 = torch.empty_like(out)
    else:
        out, out2 = torch.empty((B, out_dim, H // 8, W // 8), dtype=torch.float16, device=dev), None
    if mean is not None:
        mean = mean.reshape(3).to(dev, torch.float32).contiguous()
        std = std.reshape(3).to(dev, torch.float32).contiguous()
    ws = _lib.workspace(_lib.load().goslam_encoder_workspace_bytes(B, H, W, norm), dev)
    _lib.call("basic_encoder", ctypes.byref(weights), norm, out_dim, image, 1 if image.dtype == torch.float16 else 0,
              mean, std, B, H, W, out, out2, 1 if split else 0, ws, ws.numel())
    return (out, out2) if split else out


class ResidualBlock(nn.Module):
    def __init__(self, in_planes, planes, norm_fn="group", stride=1):
        super().__init__()
        _check_norm(norm_fn)
        self.conv1 = nn.Conv2d(in_planes, planes, kernel_size=3, padding=1, stride=stride)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, padding=1)
        self.relu = nn.ReLU(inplace=True)
        norm = nn.InstanceNorm2d if norm_fn == "instance" else (lambda _: nn.Sequential())
        self.norm1 = norm(planes)
        self.norm2 = norm(planes)
        if stride > 1:
            self.norm3 = norm(planes)
        if stride == 1:
            self.downsample = None
        else:
            self.downsample = nn.Sequential(nn.Conv2d(in_planes, planes, kernel_size=1, stride=stride, padding=0),
                                            self.norm3)


class BasicEncoder(nn.Module):
    """forward(x [b, n, 3, H, W]) -> [b, n, out_dim, H/8, W/8]: f16 under autocast (how DroidNet runs it), otherwise
    the input's dtype; no gradients."""

    def __init__(self, out_dim, norm_fn="batch"):
        super().__init__()
        _check_norm(norm_fn)
        self.out_dim = out_dim
        self.norm_fn = norm_fn
        self.norm1 = nn.InstanceNorm2d(DIM) if norm_fn == "instance" else nn.Sequential()
        self.conv1 = nn.Conv2d(3, DIM, 7, 2, 3)
        self.relu1 = nn.ReLU(inplace=True)
        self.in_planes = DIM
        self.layer1 = self._make_layer(DIM, stride=1)
        self.layer2 = self._make_layer(2 * DIM, stride=2)
        self.layer3 = self._make_layer(4 * DIM, stride=2)
        self.conv2 = nn.Conv2d(4 * DIM, out_dim, kernel_size=(1, 1))
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
        self._pack = EncoderPack()

    def _make_layer(self, dim, stride=1):
        layers = [ResidualBlock(self.in_planes, dim, self.norm_fn, stride=stride),
                  ResidualBlock(dim, dim, self.norm_fn, stride=1)]
        self.in_planes = dim
        return nn.Sequential(*layers)

    @torch.no_grad()
    def forward(self, x):
        b, n, c1, h1, w1 = x.shape
        out = encode(self._pack.get(self), self.norm_fn, self.out_dim, x.reshape(b * n, c1, h1, w1))
        dtype = torch.float16 if torch.is_autocast_enabled("cuda") else x.dtype
        return out.to(dtype).view(b, n, self.out_dim, h1 // 8, w1 // 8)
