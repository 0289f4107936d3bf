"""CPU checks of the feature / context encoder: the float64 restatement against the reference's own BasicEncoder
(tests/golden/encoder.npz), its round16 mirror, the drop-in module's parameter names against pretrained/droid.pth, and
argument validation of the C entries without a GPU."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import encoder_oracle as eo

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "encoder.npz"))


def _ours(norm):
    from goslam_b200.modules.extractor import BasicEncoder
    torch.manual_seed(int(G["enc_seed_" + norm]))
    return BasicEncoder(out_dim=128 if norm == "instance" else 256, norm_fn=norm)


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_oracle_matches_reference_float64(norm):
    enc = _ours(norm)
    sd = enc.state_dict()
    x = torch.from_numpy(G["enc_image_u8"]).double() / 255.0
    got = eo.basic_encoder(sd, norm, x)
    want = torch.from_numpy(G["enc_%s_out" % norm]).double()
    assert got.dtype == torch.float64 and got.shape == want.shape
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()


def _functional64(sd, norm_fn, x):
    """the reference's BasicEncoder.forward as plain nn.functional calls in float64"""
    n = (lambda t: F.instance_norm(t, eps=1e-5)) if norm_fn == "instance" else (lambda t: t)   # noqa: E731
    w = {k: v.double() for k, v in sd.items()}
    conv = lambda t, p, s, pad: F.conv2d(t, w[p + ".weight"], w[p + ".bias"], s, pad)         # noqa: E731
    x = F.relu(n(conv(x.double(), "conv1", 2, 3)))
    for layer, stride in ((1, 1), (2, 2), (3, 2)):
        for i, s in ((0, stride), (1, 1)):
            p = "layer%d.%d." % (layer, i)
            y = F.relu(n(conv(x, p + "conv1", s, 1)))
            y = F.relu(n(conv(y, p + "conv2", 1, 1)))
            if s > 1:
                x = n(conv(x, p + "downsample.0", s, 0))
            x = F.relu(x + y)
    return conv(x, "conv2", 1, 0)


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_round16_off_is_the_float64_graph(norm):
    """round16=False runs the reference's op sequence unchanged: bit-identical to it"""
    sd = _ours(norm).state_dict()
    x = torch.from_numpy(G["enc_image_u8"][:2]).float() / 255.0
    want = _functional64(sd, norm, x)
    assert torch.equal(eo.basic_encoder(sd, norm, x), want)
    assert torch.equal(eo.basic_encoder(sd, norm, x, round16=False), want)


# the round16 mirror's distance from the reference's float64 output, relative to its RMS, in units of 2^-11 (half an f16
# ulp at the RMS's binade or less): each of the 16 stored layers adds a rounding error of at most half an ulp of its
# values, which instance norm and the following convolutions carry at about their own scale, so the RMS error is a few
# units and the largest of the 6 x 128 x 48 (or x 256) outputs a few times that
ROUND16_RMS_UNITS, ROUND16_MAX_UNITS = 8, 32


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_round16_golden(norm):
    sd = _ours(norm).state_dict()
    x = torch.from_numpy(G["enc_image_u8"]).float() / 255.0
    got = eo.basic_encoder(sd, norm, x, round16=True)
    want = torch.from_numpy(G["enc_%s_out" % norm]).double()
    assert got.dtype == torch.float64 and got.shape == want.shape
    assert torch.equal(got, got.half().double())                        # the output is stored as f16
    e_max, e_rms = eo.errors(got, want)
    assert 0 < e_rms <= ROUND16_RMS_UNITS * 2.0 ** -11 and e_max <= ROUND16_MAX_UNITS * 2.0 ** -11, (e_max, e_rms)


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_round16_stem_input(norm):
    """the stem operand is what torch's own sub / div produce, in f32 or (rounding after each op) in f16"""
    sd = _ours(norm).state_dict()
    x = torch.from_numpy(G["enc_image_u8"][:1, :, :16, :24]).float() / 255.0
    mean, std = torch.tensor(eo.MEAN)[:, None, None], torch.tensor(eo.STDV)[:, None, None]
    for xi in (x, x.half()):
        fused = eo.basic_encoder(sd, norm, xi, eo.MEAN, eo.STDV, round16=True)
        assert torch.equal(fused, eo.basic_encoder(sd, norm, xi.clone().sub_(mean).div_(std), round16=True))
    assert not torch.equal(eo.basic_encoder(sd, norm, x.half(), eo.MEAN, eo.STDV, round16=True),
                           eo.basic_encoder(sd, norm, x, eo.MEAN, eo.STDV, round16=True))


def test_round16_statistics():
    """one (mean, rstd, min, max) per instance norm: stem, 6 x (conv1, conv2), 2 downsamples; a constant channel has
    rstd = 1 / sqrt(1e-5) and normalises to exactly 0"""
    sd = _ours("instance").state_dict()
    sd["conv1.weight"][3].zero_()
    x = torch.from_numpy(G["enc_image_u8"][:2, :, :16, :24]).float() / 255.0
    trace = {}
    eo.basic_encoder(sd, "instance", x, round16=True, trace=trace)
    stats = trace["norm"]
    assert trace["head"].shape == (2, 128, 2, 3)
    assert [s[0].shape for s in stats] == [(2, c) for c in (32, 32, 32, 32, 32, 64, 64, 64, 64, 64, 128, 128, 128, 128,
                                                             128)]
    mean, rstd, lo, hi = stats[0]
    assert torch.equal(lo[:, 3], hi[:, 3]) and (rstd[:, 3] == 1.0 / np.sqrt(1e-5)).all()
    assert (lo[:, 3] == sd["conv1.bias"][3].half().double()).all()


def test_instance_norm_needs_two_pixels_at_eighth():
    sd = _ours("instance").state_dict()
    x = torch.rand(1, 3, 8, 8)
    for r16 in (False, True):
        with pytest.raises(ValueError, match="spatial element"):
            eo.basic_encoder(sd, "instance", x, round16=r16)
    assert eo.basic_encoder(sd, "instance", torch.rand(1, 3, 8, 16), round16=True).shape == (1, 128, 1, 2)
    assert eo.basic_encoder(_ours("none").state_dict(), "none", x, round16=True).shape == (1, 256, 1, 1)


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_seeded_init_equals_reference(norm):
    """the same seed gives the reference's kaiming-initialised weights (the GPU tests rebuild them this way)"""
    sd = _ours(norm).state_dict()
    sums = np.array([sd[k].double().sum().item() for k in sorted(sd)])
    assert np.allclose(sums, G["enc_%s_wsum" % norm], rtol=0, atol=1e-9)


def test_state_dict_matches_droid_checkpoint():
    from goslam_b200.modules.extractor import BasicEncoder
    want = dict(zip(G["droid_keys"].tolist(), G["droid_shapes"].tolist()))
    got = {}
    for prefix, enc in (("fnet", BasicEncoder(128, "instance")), ("cnet", BasicEncoder(256, "none"))):
        for k, v in enc.state_dict().items():
            got[prefix + "." + k] = ";".join(map(str, v.shape))
    assert got == want


def test_unsupported_norms_raise():
    from goslam_b200.modules.extractor import BasicEncoder
    for norm in ("batch", "group"):
        with pytest.raises(NotImplementedError):
            BasicEncoder(128, norm)
    with pytest.raises(TypeError):
        BasicEncoder(128, "layer")


def test_sequence_is_the_golden_one():
    x = eo.sequence(seed=5)
    assert x.shape == (12, 3, 128, 128) and G["mf_shifts"].tolist() == list(eo.SHIFTS)
    assert int((x.double() * 255).round().sum().item()) == int(G["mf_image_u8_sum"])
    assert G["mf_decisions"][0] == 1 and 0 < G["mf_decisions"][1:].sum() < 11
    d = G["mf_delta_mean"][1:]
    assert (np.abs(d - G["mf_thresh"]) >= 0.05 * G["mf_thresh"]).all()
    # the gate follows the motion: 8-9 pixel jumps from the last keyframe are accepted, repeats and 1-pixel steps not
    key, want = 0, []
    for s in eo.SHIFTS[1:]:
        want.append(int(s - key >= 8))
        key = s if s - key >= 8 else key
    assert G["mf_decisions"][1:].tolist() == want


def test_argument_validation_without_gpu(lib):
    from goslam_b200 import _lib
    null = ctypes.c_void_p(None)
    fake = ctypes.c_void_p(256)
    assert lib.goslam_encoder_workspace_bytes(1, 240, 320, 1) > lib.goslam_encoder_workspace_bytes(1, 240, 320, 0) > 0
    assert lib.goslam_encoder_workspace_bytes(16, 240, 320, 1) > lib.goslam_encoder_workspace_bytes(1, 240, 320, 1)
    for B, H, W, norm in ((1, 60, 80, 1), (1, 64, 84, 0), (0, 64, 64, 1), (1, 64, 64, 2), (1, 8, 8, 1), (3, 8, 8, 1)):
        assert lib.goslam_encoder_workspace_bytes(B, H, W, norm) == 0
    for B, H, W, norm in ((1, 8, 8, 0), (1, 8, 16, 1), (1, 16, 8, 1), (65535, 8, 16, 1), (1, 4096, 4096, 1)):
        assert lib.goslam_encoder_workspace_bytes(B, H, W, norm) > 0
    assert lib.goslam_encoder_workspace_bytes(1, 4096, 4104, 1) == 0           # H * W above 2^24
    assert lib.goslam_encoder_workspace_bytes(65536, 8, 16, 1) == 0           # B above the grid's y limit

    full = _lib.EncoderWeights()
    for conv in [full.stem, full.out] + [full.block[i][j] for i in range(6) for j in range(3)]:
        conv.w, conv.b = 256, 256

    def call(w, B=1, H=64, W=64, out_dim=128, split=0, ws=null, nbytes=0, image=fake, out=fake, out2=null, mean=null,
             std=null, norm=1):
        return lib.goslam_basic_encoder(ctypes.byref(w), norm, out_dim, image, 0, mean, std, B, H, W, out, out2, split,
                                        ws, ctypes.c_size_t(nbytes), null)
    assert call(full, H=60) == -1                          # not a multiple of 8
    assert call(full, W=68) == -1
    assert call(full, B=0) == -1
    assert call(_lib.EncoderWeights()) == -1               # null weights
    part = _lib.EncoderWeights.from_buffer_copy(full)
    part.block[2][2].w = None                              # a stride-2 block without its downsample
    assert call(part) == -1
    assert call(full, out_dim=100) == -1
    assert call(full, out_dim=128, split=1, out2=fake) == -1   # split needs 256 outputs
    assert call(full, mean=fake) == -1                     # mean without std
    assert call(full, image=null) == -1
    assert call(full, H=8, W=8) == -1                      # instance norm of one pixel at 1/8
    assert call(full, H=8, W=8, norm=0) == -3              # valid without the norm: only the workspace is missing
    need = lib.goslam_encoder_workspace_bytes(1, 64, 64, 1)
    assert call(full) == -3                                # no workspace
    assert call(full, ws=fake, nbytes=need - 1) == -3      # short workspace
