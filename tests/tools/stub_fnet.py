"""A deterministic stand-in for DroidNet's `fnet` (src/modules/extractor.py BasicEncoder, out_dim 128): an 8 x 8
average pool followed by a fixed seeded 3 -> 128 projection, cast to f16.  Used by tests/golden/make_golden_filler.py
(driving the REFERENCE PoseTrajectoryFiller on the CPU) and by the GPU drop-in test (in place of
PoseTrajectoryFiller._feature_encoder).  Every sum is spelled out as a chain of elementwise adds in a fixed order and
there is no transcendental, so the CPU and the GPU round the same way and the golden needs no stored feature maps."""
import torch

SEED = 29
_W = None


def _weights():
    global _W
    if _W is None:
        g = torch.Generator().manual_seed(SEED)
        _W = (0.7 * torch.randn(128, 3, generator=g), 0.1 * torch.randn(128, generator=g))
    return _W


def features(x):
    """x [B, 3, H, W] f32, already normalised -> f16 [B, 128, H/8, W/8]"""
    B, _, H, W = x.shape
    t = x.float().reshape(B, 3, H // 8, 8, W // 8, 8)
    s = t[:, :, :, 0, :, 0]
    for a in range(8):
        for b in range(8):
            if a or b:
                s = s + t[:, :, :, a, :, b]
    p = s * (1.0 / 64.0)
    w, bias = (u.to(x.device) for u in _weights())
    out = p[:, 0:1] * w[:, 0].view(1, 128, 1, 1)
    out = out + p[:, 1:2] * w[:, 1].view(1, 128, 1, 1)
    out = out + p[:, 2:3] * w[:, 2].view(1, 128, 1, 1)
    out = out + bias.view(1, 128, 1, 1)
    return out.half()


class StubFnet:
    """the reference's call form: fnet(x [M, rig, 3, H, W]) -> [M, rig, 128, H/8, W/8]"""

    def __call__(self, x):
        M, rig, _, H, W = x.shape
        return features(x.reshape(M * rig, 3, H, W)).view(M, rig, 128, H // 8, W // 8)
