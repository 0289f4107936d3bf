"""The drop-in MotionFilter on the device: a replay of the reference's own MotionFilter.track on the golden 12-frame
sequence (tests/golden/encoder.npz), feature / context maps against the encoder restatement, a plain torch update
module with f32 weights (how a reference DroidNet's `update` runs), stereo input, and the caller's image left as it
was."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import encoder_oracle as eo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DEV = torch.device("cuda:0")
G = np.load(os.path.join(HERE, "golden", "encoder.npz"))


class _Recorder(nn.Module):
    """net.update with each call's mean flow magnitude (the quantity track compares with thresh) recorded"""

    def __init__(self, update):
        super().__init__()
        self.inner = update
        self.deltas = []
        self.autocast = []

    def forward(self, net, inp, corr):
        self.autocast.append(torch.is_autocast_enabled("cuda"))
        out = self.inner(net, inp, corr)
        self.deltas.append(out[1].float().norm(dim=-1).mean())
        return out


class _TorchUpdate(nn.Module):
    """a plain torch stand-in for the reference's UpdateModule: f32 convolutions over net, inp and corr -> delta"""

    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.conv = nn.Conv2d(128 + 128 + 196, 2, 3, padding=1)

    def forward(self, net, inp, corr):
        b, n, _, h, w = net.shape
        x = torch.cat([net, inp, corr], dim=2).reshape(b * n, -1, h, w)
        d = self.conv(x).permute(0, 2, 3, 1).reshape(b, n, h, w, 2)
        return net, d, d


class _Net:
    def __init__(self, update=None):
        from goslam_b200.droid_net import UpdateModule
        from goslam_b200.modules.extractor import BasicEncoder
        torch.manual_seed(int(G["enc_seed_instance"]))
        self.fnet = BasicEncoder(out_dim=128, norm_fn="instance").to(DEV)
        torch.manual_seed(int(G["enc_seed_none"]))
        self.cnet = BasicEncoder(out_dim=256, norm_fn="none").to(DEV)
        self.update = _Recorder(update if update is not None else eo.motion_update_params(UpdateModule(), 21)).to(DEV)


def _sequence():
    images = eo.sequence(seed=5)
    g = torch.Generator().manual_seed(8)
    depth = (1.0 + 2.0 * torch.rand(images.shape[0], 128, 128, generator=g)).float()
    return images.to(DEV), depth.to(DEV), torch.from_numpy(G["mf_intrinsic"]).to(DEV)


@pytest.fixture(scope="module")
def replay():
    from goslam_b200.motion_filter import MotionFilter
    net = _Net()
    video = eo.RecordingVideo()
    mf = MotionFilter(net, video, thresh=float(G["mf_thresh"]), device=DEV)
    images, depth, intr = _sequence()
    decisions = []
    for t in range(images.shape[0]):
        before = video.counter.value
        mf.track(float(t), images[t:t + 1].clone(), depth=depth[t].clone(), intrinsic=intr.clone())
        decisions.append(int(video.counter.value > before))
    return net, mf, video, decisions, images, depth, intr


def test_golden_decisions(replay):
    net, mf, video, decisions, images, depth, intr = replay
    assert decisions == G["mf_decisions"].tolist()
    assert mf.count == int(G["mf_count"])
    # every frame's mean flow against the reference's (f32 on the CPU); the threshold is >= 5 % away from each
    got = np.array([d.item() for d in net.update.deltas])
    want = G["mf_delta_mean"][1:]
    assert np.all(np.abs(got - want) <= 0.03 * want + 0.02 * float(G["mf_thresh"])), (got, want)
    slots = [t for t, d in enumerate(decisions) if d]
    assert [it[0] for it in video.items] == G["mf_timestamps"].tolist()
    for k, t in enumerate(slots):
        item = video.items[k]
        assert torch.equal(item[1], images[t])
        assert torch.equal(item[4], depth[t])
        assert np.array_equal(item[5].cpu().numpy(), G["mf_video_intrinsics"][k])
    assert video.items[0][2].tolist() == [0, 0, 0, 0, 0, 0, 1] and video.items[0][3] == 1.0
    assert all(it[2] is None and it[3] is None for it in video.items[1:])


def test_maps_within_contract(replay):
    net, _, video, decisions, images, _, _ = replay
    fsd, csd = net.fnet.state_dict(), net.cnet.state_dict()
    slots = [t for t, d in enumerate(decisions) if d]
    for k, t in enumerate(slots):
        x = images[t:t + 1]
        _, _, _, _, _, _, gmap, n_, i_, _ = video.items[k]
        ref = eo.basic_encoder(fsd, "instance", x, eo.MEAN, eo.STDV)
        auto = eo.basic_encoder(fsd, "instance", x, eo.MEAN, eo.STDV, autocast=True)
        ok, ek, ea = eo.contract_ok(gmap, auto, ref)
        assert ok and gmap.dtype == torch.float16, (t, ek, ea)
        c64 = eo.basic_encoder(csd, "none", x, eo.MEAN, eo.STDV)
        cau = eo.basic_encoder(csd, "none", x, eo.MEAN, eo.STDV, autocast=True)
        for got, r, a in zip((n_, i_), eo.context_split(c64), eo.context_split(cau)):
            ok, ek, ea = eo.contract_ok(got[None], a, r)
            assert ok and got.shape == (128, 16, 16), (t, ek, ea)


def test_torch_update_module_with_f32_weights():
    """a reference DroidNet keeps `update` as an nn module with f32 weights; track runs it under autocast, as the
    reference's decorated track does, so the f16 context features are accepted without the caller enabling autocast"""
    from goslam_b200.motion_filter import MotionFilter
    net = _Net(_TorchUpdate())
    assert not torch.is_autocast_enabled("cuda")
    images, depth, intr = _sequence()
    mf = MotionFilter(net, eo.RecordingVideo(), thresh=0.0, device=DEV)
    mf.track(0.0, images[0:1], depth=depth[0], intrinsic=intr)
    mf.track(1.0, images[4:5], depth=depth[4], intrinsic=intr)
    mf.thresh = 1e9
    mf.track(2.0, images[5:6], depth=depth[5], intrinsic=intr)
    assert net.update.autocast == [True, True]
    assert mf.video.counter.value == 2 and mf.count == 1
    assert all(torch.isfinite(d).item() and d.item() > 0 for d in net.update.deltas)


def test_stereo_and_input_untouched():
    """fnet runs on both images, cnet and the motion probe on the left one: the stereo run's maps, context and
    per-frame mean flow equal a mono run on the left images, bit for bit"""
    from goslam_b200.motion_filter import MotionFilter
    images, depth, intr = _sequence()
    thresh = float(G["mf_thresh"])
    stereo = MotionFilter(_Net(), eo.RecordingVideo(), thresh=thresh, device=DEV)
    mono = MotionFilter(_Net(), eo.RecordingVideo(), thresh=thresh, device=DEV)
    right = torch.flip(images, dims=[-1])
    for t in range(images.shape[0]):
        pair = torch.cat([images[t:t + 1], right[t:t + 1]]).clone()
        keep = pair.clone()
        stereo.track(float(t), pair, depth=depth[t], intrinsic=intr)
        assert torch.equal(pair, keep)
        mono.track(float(t), images[t:t + 1].clone(), depth=depth[t], intrinsic=intr)
        assert torch.equal(stereo.fmap[0], mono.fmap[0])
    assert len(stereo.video.items) == len(mono.video.items) == int(G["mf_decisions"].sum())
    assert stereo.count == mono.count
    assert [d.item() for d in stereo.update.deltas] == [d.item() for d in mono.update.deltas]
    for s, m in zip(stereo.video.items, mono.video.items):
        assert s[6].shape == (2, 128, 16, 16) and torch.equal(s[6][0], m[6][0])
        assert torch.equal(s[7], m[7]) and torch.equal(s[8], m[8])
    flip = mono._feature_encoder(right[0:1])
    assert torch.equal(stereo.video.items[0][6][1], flip[0])
