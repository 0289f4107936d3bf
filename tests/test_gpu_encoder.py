"""BasicEncoder on the device (csrc/encoder.cu) against the reference's float64 output (golden) and the float64 /
autocast restatement (oracle/encoder_oracle.py).  Contract: the kernel's error against float64, as max-abs and RMS
relative to the output's RMS, is at most twice the autocast path's plus one f16 ulp of the output's scale."""
import os

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "encoder.npz"))


def _encoder(norm, seed):
    from goslam_b200.modules.extractor import BasicEncoder
    torch.manual_seed(seed)
    return BasicEncoder(out_dim=128 if norm == "instance" else 256, norm_fn=norm).to(DEV)


def _run(enc, x):
    with torch.autocast("cuda"):
        return enc(x)


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_golden(golden, norm):
    enc = _encoder(norm, int(golden["enc_seed_" + norm]))
    x = torch.from_numpy(golden["enc_image_u8"]).to(DEV).float() / 255.0
    ref = torch.from_numpy(golden["enc_%s_out" % norm]).to(DEV).double()
    auto = eo.basic_encoder(enc.state_dict(), norm, x, autocast=True)
    for b, n in ((1, 1), (1, 2), (2, 3)):
        got = _run(enc, x[: b * n].reshape(b, n, 3, 48, 64))
        assert got.dtype == torch.float16 and got.shape == (b, n, enc.out_dim, 6, 8)
        ok, ek, ea = eo.contract_ok(got.reshape(b * n, -1, 6, 8), auto[: b * n], ref[: b * n])
        assert ok, (b, n, ek, ea)


@pytest.mark.parametrize("H,W", [(240, 320), (384, 512), (320, 640)])
@pytest.mark.parametrize("B", [1, 2, 16])
@pytest.mark.parametrize("norm", ["instance", "none"])
def test_shipped_sizes(norm, B, H, W):
    enc = _encoder(norm, 5)
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + H)
    x = torch.rand(B, 3, H, W, device=DEV, generator=g)
    got = _run(enc, x[None])[0]
    sd = enc.state_dict()
    ok_all = []
    for i in range(0, B, 4):      # the float64 restatement in chunks of 4 images
        xi = x[i:i + 4]
        ref = eo.basic_encoder(sd, norm, xi)
        auto = eo.basic_encoder(sd, norm, xi, autocast=True)
        ok, ek, ea = eo.contract_ok(got[i:i + 4], auto, ref)
        ok_all.append((ok, ek, ea))
    assert all(o[0] for o in ok_all), ok_all


def test_fused_normalisation_is_bit_exact():
    from goslam_b200.modules.extractor import encode
    enc = _encoder("instance", 6)
    w = enc._pack.get(enc)
    mean = torch.tensor(eo.MEAN, device=DEV)
    std = torch.tensor(eo.STDV, device=DEV)
    x = torch.rand(2, 3, 64, 96, device=DEV)
    fused = encode(w, "instance", 128, x, mean, std)
    plain = encode(w, "instance", 128, x.clone().sub_(mean[:, None, None]).div_(std[:, None, None]).half())
    assert torch.equal(fused, plain)
    x16 = x.half()
    fused = encode(w, "instance", 128, x16, mean, std)
    plain = encode(w, "instance", 128, x16.clone().sub_(mean[:, None, None]).div_(std[:, None, None]))
    assert torch.equal(fused, plain)


def test_context_split():
    from goslam_b200.modules.extractor import encode
    enc = _encoder("none", 7)
    w = enc._pack.get(enc)
    x = torch.rand(1, 3, 240, 320, device=DEV)
    full = encode(w, "none", 256, x)
    net, inp = encode(w, "none", 256, x, split=True)
    assert torch.equal(inp, full[:, 128:].relu())
    want = full[:, :128].float().tanh().half()
    assert (net.float() - want.float()).abs().max().item() <= 2.0 ** -11


def test_deterministic_and_pack_cache():
    enc = _encoder("instance", 8)
    x = torch.rand(1, 2, 3, 240, 320, device=DEV)
    a, b = _run(enc, x), _run(enc, x)
    assert torch.equal(a, b)
    with torch.no_grad():
        enc.conv2.bias.add_(1.0)
    c = _run(enc, x)
    assert torch.allclose(c.float(), a.float() + 1.0, atol=2e-2)
    assert _run(enc, x).dtype == torch.float16 and enc(x).dtype == torch.float32


def test_no_host_sync():
    enc = _encoder("instance", 9)
    x = torch.rand(1, 1, 3, 240, 320, device=DEV)
    _run(enc, x)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _run(enc, x)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_bad_shape_raises():
    enc = _encoder("none", 10)
    with pytest.raises(ValueError):
        _run(enc, torch.rand(1, 1, 3, 60, 80, device=DEV))
