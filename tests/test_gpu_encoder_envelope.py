"""BasicEncoder on the device (goslam_basic_encoder, through modules.extractor.encode and BasicEncoder) across its
envelope: tile remainders at every level, batch sizes up to the grid limit, a 2048 x 2048 image, inputs that load the
instance statistics, both stem dtypes, every output-tile width and the context split, for both norms.

Each output is checked three ways:
  * against oracle/encoder_oracle.py's round16 mirror (float64, rounded to f16 wherever encoder.cu stores f16), per
    element: |got - want| <= ULPS * G * conv(ulp16(|x| + rms(x)), |w|) + ulp16(|want|), where x is the output conv's
    input in the mirror (rms over each image and channel), w its f16 weights;
  * against the plain float64 path under test_gpu_encoder.py's contract (error relative to the output's RMS at most
    twice the autocast path's plus one f16 ulp of the output's scale), per image, wherever instance norm sees at least
    16 pixels per channel at 1/8 (MIN_PIXELS_CONTRACT);
  * in the shape and batch cases, every image of a batch against its own B = 1 encoding, bit for bit: statistics,
    tails and outputs indexed by the wrong image fail this whatever the conditioning.

Why that bound.  The kernels and the mirror store f16 at the same points from the same f16 operands; what is left is
the kernels' fp32 accumulation (mma.sync, in their own order) and their fp32 statistics.
  * A convolution output sums K <= 1152 exact f16 x f16 products plus the bias.  fp32 accumulation in any order, with
    rounded or truncated adds, is off from the exact sum by at most K * 2^-23 * S (S = conv(|x|, |w|)), typically far
    less, and well under the 2^-11 relative half-ulp of an f16 store.  So both round to the same f16, except where the
    exact value lies that close to a rounding boundary: there the stored values differ by one f16 ulp (a flip).
  * A flipped operand moves the next layer's exact value by |w| * ulp, which flips some of that layer's roundings in
    turn: flips spread through the 16 stored layers, and most outputs end up a few ulps off.  They do not grow: every
    layer is rounded again, each flip is one ulp of the value it lands on, relu and the residual add are 1-Lipschitz
    and the weights (kaiming scale) keep each layer's output at its input's scale.  So each element of the output
    conv's input x stays within a few f16 ulps of its channel's scale: ULPS * ulp16(|x| + rms(x)), ULPS = 4.
  * The output conv (1 x 1) carries that as conv(ULPS * ulp16(|x| + rms(x)), |w|), then rounds once more: a flip of
    ulp16(|want|).  Scaling by the input (not by the output's own RMS) matters: the output conv's sums cancel.
  * Instance norm normalises a stored y by rstd.  A flip of y, one ulp16(|y|), becomes ulp16(|y|) * rstd: about one
    ulp of the normalised value for a centred channel, but |mean| / spread times more for a channel with a small spread
    on a large mean (a uniform or offset image).  G is the largest such factor of any normalised layer and channel of
    the image, ulp16(max |y|) * rstd / ulp16(max |(y - mean) * rstd|), from the mirror's statistics; 1 for norm
    'none' and for constant channels, which normalise to exactly 0 on both sides.
  * The fp32 statistics (per-tile two-pass mean and M2, Chan's merge) are within a few fp32 ulps of float64: their
    effect on a normalised value is far below an f16 ulp.
  * split: tanh and relu are 1-Lipschitz; tanh's f16 rounding can flip once more: + ulp16(|want|).

What the bound can see.  The triangle inequality through the output conv's 128 inputs assumes every error has the
same sign; they do not, so the bound sits about sqrt(128) above the typical worst error: some 50-250 output f16 ulps,
at most 0.42 of the image's output RMS here, except instance norm at 16 x 16, where 4 pixels per channel at 1/8 make
G up to about 20 and the bound up to 1.1 RMS.  It catches what moves many outputs (statistics, padding, tails, eps,
the split); an error confined to a few elements is left to the float64 contract.  Two guards keep it from going
vacuous: no element's bound may exceed MAX_BOUND_RMS times its image's output RMS, and in the shape and batch cases
another image's mirror output must fail it.
Instance norm over 2 pixels per channel at 1/8 (8 x 16 and 16 x 8) is ill-conditioned: a flip of either pixel moves
the normalised pair by up to 1, G reaches 10^2-10^3 and the bound exceeds the output itself.  Those cases are not
compared with the mirror or float64; they check the launch, shape, dtype, finiteness and bit-for-bit batch
independence.
Measured on an H100 SXM (80 GB HBM3, 700 W limit) over every case here: worst error / bound 0.11; from 7 % (instance
norm) to all of a case's outputs bit-equal to the mirror.
"""
import time

import pytest
import torch
import torch.nn.functional as F

from oracle import encoder_oracle as eo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ULPS = 4
MIN_PIXELS_CONTRACT = 16
MIN_PIXELS_MIRROR = 4       # instance norm over fewer pixels per channel at 1/8 is ill-conditioned (see above)
MAX_BOUND_RMS = 2.0
NORMS = ["instance", "none"]
ZEROED = ("conv1", "layer1.0.conv1", "layer1.1.conv2", "layer2.0.conv1", "layer2.0.downsample.0", "layer3.0.conv2",
          "layer3.0.downsample.0", "layer3.1.conv1", "layer3.1.conv2")


def _ulp16(x):
    """spacing of f16 at |x| (2^-24 below the normal range)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def _encoder(norm, out_dim=None, seed=5, zeroed=False):
    """a seeded BasicEncoder; zeroed: every fifth output channel of the ZEROED convolutions has zero weights, so it
    is exactly its bias at every pixel (m2 = 0)"""
    from goslam_b200.modules.extractor import BasicEncoder
    torch.manual_seed(seed)
    enc = BasicEncoder(out_dim or (128 if norm == "instance" else 256), norm)
    if zeroed:
        mods = dict(enc.named_modules())
        with torch.no_grad():
            for name in ZEROED:
                mods[name].weight[::5].zero_()
    return enc.to(DEV)


def _gain(stats, B):
    g = torch.ones(B, dtype=torch.float64, device=DEV)
    for mean, rstd, lo, hi in stats:
        spread = torch.maximum(hi - mean, mean - lo) * rstd
        flip = _ulp16(torch.maximum(hi.abs(), lo.abs())) * rstd
        ratio = torch.where(hi == lo, torch.ones_like(flip), flip / _ulp16(spread))
        g = torch.maximum(g, ratio.amax(dim=1))
    return g


def _slack(enc, trace, B):
    """ULPS * G * conv(ulp16(|x| + rms(x)), |w|): the bound before the output's own rounding"""
    x = trace["head"]
    u = _ulp16(x.abs() + x.pow(2).mean(dim=(2, 3), keepdim=True).sqrt())
    w = enc.conv2.weight.detach().half().double().abs()
    return ULPS * _gain(trace.get("norm", []), B).view(-1, 1, 1, 1) * F.conv2d(u, w)


def _check(got, want, bound, what, distinct=False):
    """per-element bound against the round16 mirror; returns the worst error / bound.  distinct: the batch's images
    differ, and each image's bound must reject the next image's mirror output"""
    assert got.shape == want.shape and got.dtype == torch.float16, (what, got.shape, want.shape, got.dtype)
    got = got.double()
    assert torch.isfinite(got).all(), what
    loose = (bound.amax(dim=(1, 2, 3)) / want.pow(2).mean(dim=(1, 2, 3)).sqrt()).max().item()
    assert loose <= MAX_BOUND_RMS, (what, "bound / output RMS", loose)
    if distinct and want.shape[0] > 1:
        passes = ((want.roll(1, 0) - want).abs() <= bound).flatten(1).all(dim=1)
        assert not passes.any(), (what, "another image's output passes the bound", passes.tolist())
    err = (got - want).abs()
    ratio = (err / bound).amax().item()
    print("[envelope] %s: worst error / bound %.3f (max err %.3g), bit-equal %.4f, bound / RMS %.3f"
          % (what, ratio, err.max().item(), (got == want).double().mean().item(), loose))
    assert ratio <= 1.0, (what, ratio)
    return ratio


def _contract(got, auto, ref, what):
    for i in range(got.shape[0]):
        ok, ek, ea = eo.contract_ok(got[i:i + 1], auto[i:i + 1], ref[i:i + 1])
        assert ok, (what, i, ek, ea)


def _stat_args(mean_std):
    if not mean_std:
        return None, None, None, None
    return eo.MEAN, eo.STDV, torch.tensor(eo.MEAN, device=DEV), torch.tensor(eo.STDV, device=DEV)


def _encode_and_check(enc, x, what, mean_std=False):
    """run encode on x and check it against the mirror (and the float64 contract); returns the output"""
    from goslam_b200.modules.extractor import encode
    mean, std, mean_t, std_t = _stat_args(mean_std)
    got = encode(enc._pack.get(enc), enc.norm_fn, enc.out_dim, x, mean_t, std_t)
    _mirror_check(enc, x, got, what, mean, std)
    return got


def _mirror_check(enc, x, got, what, mean=None, std=None, distinct=False):
    sd, norm = enc.state_dict(), enc.norm_fn
    pixels = (x.shape[2] // 8) * (x.shape[3] // 8)
    assert got.dtype == torch.float16 and torch.isfinite(got).all(), what
    if norm == "instance" and pixels < MIN_PIXELS_MIRROR:
        return
    trace = {}
    want = eo.basic_encoder(sd, norm, x, mean, std, round16=True, trace=trace)
    _check(got, want, _slack(enc, trace, x.shape[0]) + _ulp16(want), what, distinct)
    if norm == "none" or pixels >= MIN_PIXELS_CONTRACT:
        # below that, instance norm of a few pixels turns a flipped rounding into an O(1) change of the output: the
        # statistics of the float64 comparison say nothing more there than the mirror's bound
        ref = eo.basic_encoder(sd, norm, x, mean, std)
        auto = eo.basic_encoder(sd, norm, x, mean, std, autocast=True)
        _contract(got, auto, ref, what)


# ---- shapes and batch sizes --------------------------------------------------------------------------------------
# H x W chosen so that HW mod 64 at 1/2, 1/4 and 1/8 takes 0, small (1, 4, 16), large (48, 52, 53, 60) and less than one
# tile (2, 8, 15, 32), with thin images in both orientations for the row / column split of the tile's pixels
SHAPES = [(8, 16), (16, 8), (16, 16), (24, 40), (8, 520), (520, 8), (136, 136), (376, 1240), (240, 320), (384, 512)]


@pytest.mark.parametrize("B", [1, 3, 17])
@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("norm", NORMS)
def test_shapes_and_batches(norm, H, W, B):
    enc = _encoder(norm, seed=H + W)
    g = torch.Generator(device=DEV).manual_seed(B * 7919 + H * 31 + W)
    x = torch.rand(B, 3, H, W, device=DEV, generator=g)
    from goslam_b200.modules.extractor import encode
    with torch.autocast("cuda"):
        got = enc(x[None])[0]
    assert got.shape == (B, enc.out_dim, H // 8, W // 8)
    w = enc._pack.get(enc)
    for i in range(B):
        assert torch.equal(got[i:i + 1], encode(w, norm, enc.out_dim, x[i:i + 1])), (norm, H, W, B, i)
    _mirror_check(enc, x, got, "%s %dx%d B=%d" % (norm, H, W, B), distinct=True)


@pytest.mark.parametrize("norm,H,W", [("instance", 8, 16), ("instance", 32, 32), ("none", 8, 16)])
def test_batch_at_grid_limit(norm, H, W):
    """B = 65535 (gridDim.y): copies of one image, distinct images at the first, middle and last positions.  Every
    image equals its own B = 1 result bit for bit; the distinct images are checked against the mirror (instance norm
    at 32 x 32, 16 pixels per channel at 1/8, since 8 x 16 is ill-conditioned there)."""
    from goslam_b200.modules.extractor import encode
    B = 65535
    enc = _encoder(norm, seed=21)
    g = torch.Generator(device=DEV).manual_seed(22)
    imgs = torch.rand(4, 3, H, W, device=DEV, generator=g)
    pos = [0, B // 2, B - 1]
    x = imgs[3:4].expand(B, 3, H, W).contiguous()
    x[pos] = imgs[:3]
    w = enc._pack.get(enc)
    got = encode(w, norm, enc.out_dim, x)
    single = encode(w, norm, enc.out_dim, imgs[3:4].contiguous())
    copies = torch.ones(B, dtype=torch.bool, device=DEV)
    copies[pos] = False
    assert torch.equal(got[copies], single.expand(B - 3, -1, -1, -1)), norm
    for i, p in enumerate(pos):
        assert torch.equal(got[p:p + 1], encode(w, norm, enc.out_dim, imgs[i:i + 1].contiguous())), (norm, p)
    _mirror_check(enc, imgs, torch.cat([got[pos], single]), "%s %dx%d B=65535 distinct + copy" % (norm, H, W),
                  distinct=True)


@pytest.mark.parametrize("norm", NORMS)
def test_large_image(norm):
    """one 2048 x 2048 image (about 10^6 stem pixels, 2^16 pixels at 1/8), compared in full"""
    enc = _encoder(norm, seed=23)
    x = torch.rand(1, 3, 2048, 2048, device=DEV, generator=torch.Generator(device=DEV).manual_seed(24))
    t = time.perf_counter()
    _encode_and_check(enc, x, "%s 2048x2048" % norm, mean_std=True)
    print("[envelope] %s 2048x2048: %.1f s with the float64 mirrors" % (norm, time.perf_counter() - t))


# ---- inputs that target the instance statistics -----------------------------------------------------------------
def _image(kind, B, H, W):
    g = torch.Generator(device=DEV).manual_seed(len(kind) * 101 + B)
    if kind == "uniform":
        return torch.tensor([0.5, 0.25, 0.75][:B], device=DEV).view(B, 1, 1, 1).expand(B, 3, H, W).contiguous()
    if kind == "black":
        return torch.zeros(B, 3, H, W, device=DEV)
    if kind == "saturated":
        return torch.ones(B, 3, H, W, device=DEV)
    if kind == "offset":       # a large common offset: every stem channel has a small spread on a large mean
        return 0.9 + 0.01 * torch.rand(B, 3, H, W, device=DEV, generator=g)
    return torch.rand(B, 3, H, W, device=DEV, generator=g)


@pytest.mark.parametrize("mean_std", [False, True])
@pytest.mark.parametrize("kind", ["uniform", "black", "saturated", "offset", "zeroed"])
@pytest.mark.parametrize("norm", NORMS)
def test_statistics_inputs(norm, kind, mean_std):
    """40 x 72: 720, 180 and 45 pixels at 1/2, 1/4 and 1/8 (partial tiles of 16, 52 and 45).  'zeroed' makes some
    channels of seven layers exactly constant: m2 = 0 must normalise to exactly 0, never NaN."""
    enc = _encoder(norm, seed=25, zeroed=kind == "zeroed")
    x = _image(kind, 3, 40, 72)
    got = _encode_and_check(enc, x, "%s %s mean_std=%d" % (norm, kind, mean_std), mean_std=mean_std)
    if kind == "black" and not mean_std and norm == "instance":
        # zero image, zero padding: every layer is constant, every normalised activation 0 and the output the bias
        assert torch.equal(got, enc.conv2.bias.detach().half().view(1, -1, 1, 1).expand_as(got))


@pytest.mark.parametrize("mean_std", [False, True])
def test_constant_channels_normalise_to_exactly_zero(mean_std):
    """every fifth channel of layer3's conv2s and downsample has zero weights: constant at its bias on a random image,
    m2 = 0, normalised to exactly 0, so layer3's tails leave those channels exactly 0.  With the output conv reading
    only them, the output is exactly its bias; a normalised residue of any size would show."""
    from goslam_b200.modules.extractor import encode
    enc = _encoder("instance", seed=35, zeroed=True)
    with torch.no_grad():
        keep = torch.ones(128, dtype=torch.bool)
        keep[::5] = False
        enc.conv2.weight[:, keep] = 0.0
    x = torch.rand(3, 3, 40, 72, device=DEV, generator=torch.Generator(device=DEV).manual_seed(36))
    mean, std, mean_t, std_t = _stat_args(mean_std)
    got = encode(enc._pack.get(enc), "instance", 128, x, mean_t, std_t)
    bias = enc.conv2.bias.detach().half().view(1, -1, 1, 1).expand_as(got)
    trace = {}
    want = eo.basic_encoder(enc.state_dict(), "instance", x, mean, std, round16=True, trace=trace)
    assert (trace["head"][:, ::5] == 0).all() and (trace["head"][:, 1::5] != 0).any()
    assert torch.equal(want, bias.double()) and torch.equal(got, bias)


# ---- stem input dtypes, output widths, split ---------------------------------------------------------------------
@pytest.mark.parametrize("mean_std", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("norm", NORMS)
def test_stem_dtypes(norm, dtype, mean_std):
    enc = _encoder(norm, seed=26)
    x = torch.rand(2, 3, 240, 320, device=DEV, generator=torch.Generator(device=DEV).manual_seed(27)).to(dtype)
    _encode_and_check(enc, x, "%s %s mean_std=%d" % (norm, dtype, mean_std), mean_std=mean_std)


@pytest.mark.parametrize("out_dim", [32, 64, 96, 128, 256])
@pytest.mark.parametrize("norm", NORMS)
def test_out_dims(norm, out_dim):
    """the output conv at 32-, 64- and 128-wide channel tiles (96 takes three 32-wide ones); 56 x 88 has 77 pixels
    at 1/8"""
    enc = _encoder(norm, out_dim=out_dim, seed=28 + out_dim)
    x = torch.rand(3, 3, 56, 88, device=DEV, generator=torch.Generator(device=DEV).manual_seed(29))
    _encode_and_check(enc, x, "%s out_dim=%d" % (norm, out_dim), mean_std=True)


@pytest.mark.parametrize("norm", NORMS)
def test_split(norm):
    from goslam_b200.modules.extractor import encode
    enc = _encoder(norm, out_dim=256, seed=30)
    x = torch.rand(3, 3, 56, 88, device=DEV, generator=torch.Generator(device=DEV).manual_seed(31))
    mean, std, mean_t, std_t = _stat_args(True)
    net, inp = encode(enc._pack.get(enc), norm, 256, x, mean_t, std_t, split=True)
    trace = {}
    pre = eo.basic_encoder(enc.state_dict(), norm, x, mean, std, round16=True, trace=trace)
    bound = _slack(enc, trace, 3) + _ulp16(pre)      # the f16 conv output's bound, carried through tanh / relu
    want_net, want_inp = eo.context_split(pre)
    want_net = want_net.half().double()
    _check(net, want_net, bound[:, :128] + _ulp16(want_net), "%s split tanh" % norm)
    _check(inp, want_inp, bound[:, 128:], "%s split relu" % norm)
    ref_net, ref_inp = eo.context_split(eo.basic_encoder(enc.state_dict(), norm, x, mean, std))
    auto_net, auto_inp = eo.context_split(eo.basic_encoder(enc.state_dict(), norm, x, mean, std, autocast=True))
    _contract(net, auto_net, ref_net, "%s split tanh" % norm)
    _contract(inp, auto_inp, ref_inp, "%s split relu" % norm)


# ---- the 8 x 8 contract ------------------------------------------------------------------------------------------
def test_instance_norm_8x8_raises():
    """1 x 1 at 1/8: F.instance_norm raises ValueError, so do encode and BasicEncoder (the library returns EINVAL)"""
    from goslam_b200.modules.extractor import encode
    enc = _encoder("instance", seed=32)
    x = torch.rand(2, 3, 8, 8, device=DEV)
    with pytest.raises(ValueError, match="spatial element"):
        encode(enc._pack.get(enc), "instance", 128, x)
    with pytest.raises(ValueError, match="spatial element"):
        enc(x[None])
    with pytest.raises(ValueError, match="spatial element"):
        eo.basic_encoder(enc.state_dict(), "instance", x)


def test_none_8x8():
    enc = _encoder("none", seed=33)
    x = torch.rand(3, 3, 8, 8, device=DEV, generator=torch.Generator(device=DEV).manual_seed(34))
    _encode_and_check(enc, x, "none 8x8")
    _encode_and_check(enc, x, "none 8x8 mean_std", mean_std=True)
