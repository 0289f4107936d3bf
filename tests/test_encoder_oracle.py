"""CPU checks of the feature / context encoder: the float64 restatement against the reference's own BasicEncoder
(tests/golden/encoder.npz), the drop-in module's parameter names against pretrained/droid.pth, and argument
validation of the C entries without a GPU."""
import ctypes
import os

import numpy as np
import pytest
import torch

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
    for B, H, W, norm in ((1, 60, 80, 1), (1, 64, 84, 0), (0, 64, 64, 1), (1, 64, 64, 2)):
        assert lib.goslam_encoder_workspace_bytes(B, H, W, norm) == 0

    full = _lib.EncoderWeights()
    for conv in [full.stem, full.out] + [full.block[i][j] for i in range(6) for j in range(3)]:
        conv.w, conv.b = 256, 256

    def call(w, B=1, H=64, W=64, out_dim=128, split=0, ws=null, nbytes=0, image=fake, out=fake, out2=null, mean=null,
             std=null):
        return lib.goslam_basic_encoder(ctypes.byref(w), 1, out_dim, image, 0, mean, std, B, H, W, out, out2, split, ws,
                                        ctypes.c_size_t(nbytes), null)
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
    need = lib.goslam_encoder_workspace_bytes(1, 64, 64, 1)
    assert call(full) == -3                                # no workspace
    assert call(full, ws=fake, nbytes=need - 1) == -3      # short workspace
