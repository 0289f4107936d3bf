"""The update operator's kernels (csrc/conv_tc.cu) layer by layer and end to end against float64 references.

Per layer, goslam_conv2d_nhwc against conv2d in float64 on the fp16 operands the kernel multiplies, plus bias,
activation and scale.  Bounds, with K = taps * cin products per output, S = conv(|x|, |w|) and pre = conv(x, w) + b:
  * fp32 accumulation of K exact fp16 x fp16 products (any order, rounded or truncated adds) is off by at most
    K * 2^-23 * S, adding the bias by 2^-24 * |pre| more; the activations are 1-Lipschitz and `out_scale` multiplies:
    acc = (2K * 2^-24 * S + 2^-23 * |pre|) * |scale|.
  * For sigmoid and softplus, the error of __expf(x) = ex2.approx(x * log2 e) on top: relative 2^-21 for ex2 and
    |x| * 2^-24 for the rounded product, which both activations pass on at most doubled: (2^-20 + |pre| * 2^-23) * |ref|.
    Plus 2^-23 * |ref| for the final fp32 roundings.  Together: delta >= |kernel's fp32 result - ref|.
  * fp32 outputs: |got - ref| <= delta.
  * fp16 outputs: the kernel's fp32 result and ref both lie within |ref| + delta, so rounding each to fp16 moves it by at
    most half an fp16 ulp of that magnitude (whichever binade either falls in):
    |got - fl16(ref)| <= ulp16(|ref| + delta) + delta; nearly all elements are bit-equal to fl16(ref).

End to end, goslam_update_op against oracle/update_oracle.py with round16=True, which rounds to fp16 exactly where the
kernels store fp16.  The only differences left are fp32 summation order flipping an fp16 rounding of an intermediate,
which the following layers carry forward as an error of the order of one fp16 ulp of that intermediate.  So most elements
are bit-equal and the rest are within a few fp16 ulps of the output's own scale: |got - ref| <= n * ulp16(|ref| + rms(ref)).
The layer bounds are derived (only the bit-equal fraction is calibrated); the operator's n and bit-equal fractions are
calibrated (see OP_ULPS).
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ACTS = ("none", "relu", "sigmoid", "softplus")


def dev():
    return torch.device("cuda:0")


def _ulp16(x):
    """spacing of fp16 at |x| (2^-24 below the normal range)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def _act64(v, act):
    if act == "relu":
        return torch.relu(v)
    if act == "sigmoid":
        return torch.sigmoid(v)
    if act == "softplus":
        return F.softplus(v)          # threshold 20: x itself above it, as the kernel
    return v


# ------------------------------------------------------------------------------------------------------
# B. one layer of goslam_conv2d_nhwc
# ------------------------------------------------------------------------------------------------------
FP16_BITEQ_MIN = 0.98


def _make_layer(B, h, w, taps, srcs, cout, cout_pad, seed):
    """srcs: list of (cin, cin_off, cin_stride).  Inputs in [-1, 1], weights and biases sized so that the pre-activations
    spread over about [-30, 30] (softplus's linear branch above 20 is taken)."""
    from goslam_b200.modules.gru import pack_conv
    g = torch.Generator().manual_seed(seed)
    xs = [(torch.rand(B, h, w, stride, generator=g) * 2 - 1).half().to(dev()) for (_, _, stride) in srcs]
    cin = sum(c for c, _, _ in srcs)
    k = 3 if taps == 9 else 1
    wt = torch.randn(cout, cin, k, k, generator=g) * (10.0 / (taps * cin / 3) ** 0.5)
    bias = (torch.rand(cout, generator=g) * 2 - 1) * 8
    w16, b32 = pack_conv([wt.to(dev())], [bias.to(dev())], cout_pad=cout_pad)
    return xs, w16, b32


def _reference(xs, srcs, w16, b32, cout, taps):
    """float64 pre-activation and S = conv(|x|, |w|), NHWC [B, h, w, cout]"""
    x = torch.cat([t[..., off:off + c] for t, (c, off, _) in zip(xs, srcs)], dim=-1).permute(0, 3, 1, 2).double()
    k = 3 if taps == 9 else 1
    wt = w16[:, :cout].double().reshape(k, k, cout, -1).permute(2, 3, 0, 1)
    b = b32[:cout].double()
    pre = F.conv2d(x, wt, b, padding=k // 2).permute(0, 2, 3, 1)
    S = F.conv2d(x.abs(), wt.abs(), padding=k // 2).permute(0, 2, 3, 1)
    return pre, S


def _check_layer(got, pre, S, act, scale, K, out_f32, stats):
    ref = _act64(pre, act) * scale
    acc = (2 * K * 2.0 ** -24 * S + 2.0 ** -23 * pre.abs()) * abs(scale)
    expf = (2.0 ** -20 + 2.0 ** -23 * pre.abs()) if act in ("sigmoid", "softplus") else 0.0
    delta = acc + (expf + 2.0 ** -23) * ref.abs() + 1e-30     # bound on |kernel's fp32 result - ref|
    if out_f32:
        bound = delta
        err = (got.double() - ref).abs()
    else:
        r16 = ref.half().double()
        bound = _ulp16(ref.abs() + delta) + delta
        err = (got.double() - r16).abs()
        frac = (got.double() == r16).double().mean().item()
        stats["biteq_min"] = min(stats.get("biteq_min", 1.0), frac)
        assert frac >= FP16_BITEQ_MIN, ("bit-equal fraction", frac)
    ratio = (err / bound).max().item()
    stats["ratio_max"] = max(stats.get("ratio_max", 0.0), ratio)
    assert torch.isfinite(got).all()
    assert ratio <= 1.0, ("worst error / bound", ratio, err.max().item())


def _run_layer(B, h, w, taps, srcs, cout, cout_pad, act, scale, out_f32=False, out_offset=0, seed=0, stats=None):
    from goslam_b200.modules.gru import conv2d_nhwc
    stats = {} if stats is None else stats
    xs, w16, b32 = _make_layer(B, h, w, taps, srcs, cout, cout_pad, seed)
    width = out_offset + (cout + 7) // 8 * 8 + 8
    sentinel = -12345.0 if out_f32 else -1234.0
    out = torch.full((B, h, w, width), sentinel, dtype=torch.float32 if out_f32 else torch.float16, device=dev())
    conv2d_nhwc([(t, c, off) for t, (c, off, _) in zip(xs, srcs)], w16, b32, cout, act=act, out=out,
                out_offset=out_offset, out_scale=scale)
    torch.cuda.synchronize()
    # channels outside [out_offset, out_offset + cout) are never written
    outside = torch.cat([out[..., :out_offset], out[..., out_offset + cout:]], dim=-1)
    assert bool((outside == sentinel).all()), "layer wrote outside its output channels"
    pre, S = _reference(xs, srcs, w16, b32, cout, taps)
    _check_layer(out[..., out_offset:out_offset + cout], pre, S, act, scale, taps * sum(c for c, _, _ in srcs), out_f32,
                 stats)
    return stats


_STATS = {}


def _record(group, st):
    agg = _STATS.setdefault(group, {})
    agg["ratio_max"] = max(agg.get("ratio_max", 0.0), st.get("ratio_max", 0.0))
    if "biteq_min" in st:
        agg["biteq_min"] = min(agg.get("biteq_min", 1.0), st["biteq_min"])
    print("[%s] worst error / bound %.3f, min bit-equal fraction %s" % (
        group, agg["ratio_max"], "%.4f" % agg["biteq_min"] if "biteq_min" in agg else "-"))


@pytest.mark.parametrize("cout_pad", list(range(16, 257, 16)))
def test_conv_tile_widths(cout_pad):
    """every conv_tc_kernel<N> instance (N = cout_pad <= 256), full and with an odd cout (single-half tail store);
    64 images of 16x32 = 256 tiles, about twice the SM count (the persistent loop runs)."""
    i = cout_pad // 16
    for cout in (cout_pad, cout_pad - 1 - 2 * (i % 7)):
        act = ACTS[(i + cout) % 4]
        st = _run_layer(64, 16, 32, 9 if i % 2 else 1, [(64 * (1 + i % 2), 0, 64 * (1 + i % 2))], cout, cout_pad, act,
                        0.75, out_offset=8 * (i % 3), seed=cout)
        _record("tile widths", st)


@pytest.mark.parametrize("cout_pad,cout", [(384, 384), (512, 509), (576, 576), (640, 637), (1024, 1024)])
def test_conv_multi_channel_tiles(cout_pad, cout):
    """cout_pad > 256: N = 192 (384, 576), 256 (512, 1024) or 128 (640), several channel tiles per pixel tile"""
    for taps in (1, 9):
        st = _run_layer(24, 16, 32, taps, [(128, 0, 128)], cout, cout_pad, "relu", 1.0, seed=cout_pad + taps)
        _record("multi-tile channels", st)


@pytest.mark.parametrize("taps", [1, 9])
@pytest.mark.parametrize("n_in", [1, 2, 3, 4])
def test_conv_inputs_and_channel_slices(taps, n_in):
    """up to four inputs read as one concatenation, each a channel slice (cin_off != 0, cin_stride > cin)"""
    srcs = [(64, 128, 192), (128, 0, 256), (64, 64, 128), (192, 64, 256)][:n_in]
    st = _run_layer(12, 24, 40, taps, srcs, 96, 96, "sigmoid", 1.0, out_offset=16, seed=10 * taps + n_in)
    _record("inputs / slices", st)


@pytest.mark.parametrize("out_f32", [False, True])
@pytest.mark.parametrize("act", ACTS)
def test_conv_activations_and_outputs(act, out_f32):
    """every activation with out_scale != 1, fp16 and fp32 outputs into a wider sentinel-filled tensor"""
    for scale in (0.01, 1.7):
        st = _run_layer(32, 16, 32, 9, [(128, 0, 128)], 37, 48, act, scale, out_f32=out_f32, out_offset=8,
                        seed=ACTS.index(act) + 5 * out_f32)
        _record("activations fp32" if out_f32 else "activations fp16", st)


@pytest.mark.parametrize("act", ACTS)
def test_conv_activation_curves(act):
    """pre-activations swept over [-30, 30] in steps of about 1/64, exactly: a 1x1 layer whose only nonzero weight
    copies input channel 0 (fp16 grid values) to every output, so the accumulation is exact and what is left is the
    activation's own arithmetic (softplus's switch to x above 20 included)"""
    from goslam_b200.modules.gru import conv2d_nhwc
    B, h, w, cout = 8, 16, 32, 16
    grid = torch.linspace(-30, 30, B * h * w).half().view(B, h, w, 1)
    x = torch.zeros(B, h, w, 64, dtype=torch.float16)
    x[..., :1] = grid
    x = x.to(dev())
    w16 = torch.zeros(1, cout, 64, dtype=torch.float16, device=dev())
    w16[0, :, 0] = 1.0
    b32 = torch.zeros(cout, device=dev())
    for scale in (0.01, 1.0):
        out = conv2d_nhwc([(x, 64, 0)], w16, b32, cout, act=act, out_f32=True, out_scale=scale)
        pre, S = _reference([x], [(64, 0, 64)], w16, b32, cout, 1)
        st = {}
        _check_layer(out, pre, S, act, scale, 1, True, st)      # one nonzero product per output: K = 1
        _record("activation curves", st)


@pytest.mark.parametrize("shape", [(512, 1, 1), (256, 9, 13), (512, 8, 16), (48, 30, 40), (24, 40, 80), (16, 60, 80)])
def test_conv_image_shapes(shape):
    """image borders (TMA zero fill) and partial patches; n_tiles several times the SM count"""
    B, h, w = shape
    st = _run_layer(B, h, w, 9, [(64, 0, 64)], 64, 64, "relu", 1.0, seed=h * w)
    _record("image shapes", st)
    st = _run_layer(B, h, w, 1, [(64, 0, 64)], 16, 16, "none", 1.0, out_f32=True, seed=h * w + 1)
    _record("image shapes", st)


@pytest.mark.parametrize("act2", ACTS)
@pytest.mark.parametrize("act", ACTS)
def test_conv_split_heads(act, act2):
    """two small heads in one pass: channels < split take act and go to out, channels >= split take act2 and go to
    out2 (as channel - split), both fp32 with the same stride"""
    from goslam_b200 import _lib
    from goslam_b200.modules.gru import ACT
    B, h, w, cout, split = 20, 24, 40, 6, 2
    srcs = [(128, 0, 128)]
    xs, w16, b32 = _make_layer(B, h, w, 9, srcs, cout, 16, seed=ACTS.index(act) * 4 + ACTS.index(act2))
    stride = cout - split
    out = torch.full((B, h, w, stride), -12345.0, device=dev())
    out2 = torch.full((B, h, w, stride), -12345.0, device=dev())
    d = _lib.ConvDesc()
    d.inp[0], d.cin[0], d.cin_off[0], d.cin_stride[0], d.n_in = xs[0].data_ptr(), 128, 0, 128, 1
    d.weight, d.bias, d.taps, d.cout, d.cout_pad = w16.data_ptr(), b32.data_ptr(), 9, cout, 16
    d.act, d.act2, d.split, d.out_scale = ACT[act], ACT[act2], split, 1.0
    d.out, d.out2, d.out_f32, d.out_stride, d.out_offset = out.data_ptr(), out2.data_ptr(), 1, stride, 0
    with torch.cuda.device(dev()):
        _lib.check(_lib.load().goslam_conv2d_nhwc(ctypes.byref(d), B, h, w, _lib.stream_ptr()), "conv2d_nhwc")
    torch.cuda.synchronize()
    assert bool((out[..., split:] == -12345.0).all())
    pre, S = _reference(xs, srcs, w16, b32, cout, 9)
    st = {}
    _check_layer(out[..., :split], pre[..., :split], S[..., :split], act, 1.0, 9 * 128, True, st)
    _check_layer(out2, pre[..., split:], S[..., split:], act2, 1.0, 9 * 128, True, st)
    _record("split heads", st)


# ------------------------------------------------------------------------------------------------------
# C. the whole operator (goslam_update_op through UpdateModule) against the round16 restatement
# ------------------------------------------------------------------------------------------------------
# |got - ref| <= OP_ULPS * ulp16(|ref| + rms(ref)) per output, and at least OP_BITEQ_MIN of the fp16 outputs bit-equal.
# Measured on H100s (80 GB HBM3; 400 W and 700 W limits, identical results) over the cases below: worst error / bound
# 0.71 (net), 0.35 (delta), 0.18 (weight), 0.11 (eta), 0.42 (upmask); bit-equal at least 0.958 (net) and 0.68 (upmask:
# its 1x1 over 128 channels of a2 picks up most of a2's flipped roundings).  delta, weight and eta are fp32 results of fp16 inputs: a fraction of an
# fp16 ulp.  On top, every output stays within a tenth of the tolerance test_update_module_vs_reference_golden allows.
OP_ULPS = {"net": 5, "delta": 4, "weight": 0.25, "eta": 0.25, "upmask": 4}
OP_BITEQ_MIN = {"net": 0.93, "upmask": 0.6}
OP_GOLDEN_TOL = {"net": 1.5e-2, "delta": 1.5e-2, "weight": 1e-2, "eta": 1e-3, "upmask": 2e-2}


def _module():
    from goslam_b200.droid_net import UpdateModule
    torch.manual_seed(78)
    return UpdateModule().to(dev())


def _neighborhood(t0, t1, r):
    """FactorGraph.add_neighborhood_factors(t0, t1, r) edges on a mono video"""
    ii, jj = torch.meshgrid(torch.arange(t0, t1), torch.arange(t0, t1), indexing="ij")
    ii, jj = ii.reshape(-1), jj.reshape(-1)
    keep = ((ii - jj).abs() > 0) & ((ii - jj).abs() <= r)
    return ii[keep], jj[keep]


def _lowmem_chunk():
    """update_lowmem's chunk: the edges of a 20-frame, r = 4 window whose source lies in 13 consecutive frames (94)"""
    ii = _neighborhood(0, 20, 4)[0]
    return ii[ii < 13]


def _inputs(num, h, w, seed):
    """the golden's input distributions (tests/golden/make_golden.py gen_update_module)"""
    g = torch.Generator().manual_seed(seed)
    net = torch.tanh(torch.randn(1, num, 128, h, w, generator=g)).half()
    inp = torch.relu(torch.randn(1, num, 128, h, w, generator=g)).half()
    corr = (0.7 * torch.randn(1, num, 196, h, w, generator=g)).half()
    flow = (4.0 * torch.randn(1, num, 4, h, w, generator=g)).clamp(-64, 64)
    return [t.to(dev()) for t in (net, inp, corr, flow)]


def _golden_inputs():
    g = np.load(os.path.join(HERE, "golden", "update_module.npz"))
    t = lambda k: torch.from_numpy(g[k]).to(dev())                                  # noqa: E731
    return t("net"), t("inp"), t("corr"), t("flow").float(), t("ii")


def _case(name):
    if name == "golden":
        return _golden_inputs()
    h, w, ii = {
        "frontend_40x80": (40, 80, _neighborhood(0, 8, 3)[0]),
        "18_edges_30x40": (30, 40, _neighborhood(0, 6, 2)[0][:18]),
        "60x80": (60, 80, _neighborhood(0, 4, 2)[0]),
        "lowmem_chunk_30x40": (30, 40, _lowmem_chunk()),
        "5_edges_9x13": (9, 13, torch.tensor([2, 0, 2, 1, 0])),
        "one_frame": (16, 32, torch.tensor([4, 4, 4, 4])),
        "all_distinct": (16, 32, torch.tensor([5, 1, 7, 0, 3])),
        "unsorted_repeats": (24, 40, torch.tensor([6, 2, 6, 9, 2, 2, 6, 0])),
    }[name]
    net, inp, corr, flow = _inputs(int(ii.numel()), h, w, seed=h * w + int(ii.numel()))
    return net, inp, corr, flow, ii.to(dev())


def _compare_op(got, want, stats, case):
    names = ("net", "delta", "weight", "eta", "upmask")
    assert len(got) == len(want)
    fails = []
    for name, a, b in zip(names, got, want):
        assert a.shape == b.shape, (name, a.shape, b.shape)
        a = a.double()
        err = (a - b).abs()
        bound = OP_ULPS[name] * _ulp16(b.abs() + b.pow(2).mean().sqrt())
        ratio = (err / bound).max().item()
        st = stats.setdefault(name, {})
        st["ratio_max"] = max(st.get("ratio_max", 0.0), ratio)
        frac = (a == b).double().mean().item()
        if name in OP_BITEQ_MIN:
            st["biteq_min"] = min(st.get("biteq_min", 1.0), frac)
        print("[operator %s] %s worst error / bound %.3f (max err %.3g), bit-equal %.4f" % (name, case, ratio, err.max().item(), frac))
        fails += [(name, "worst error / bound", ratio)] if ratio > 1.0 else []
        fails += [(name, "max error", err.max().item())] if err.max().item() > OP_GOLDEN_TOL[name] / 10 else []
        fails += [(name, "bit-equal fraction", frac)] if frac < OP_BITEQ_MIN.get(name, 0.0) else []
    assert not fails, fails


OP_CASES = ["golden", "frontend_40x80", "18_edges_30x40", "60x80", "lowmem_chunk_30x40", "5_edges_9x13", "one_frame",
            "all_distinct", "unsorted_repeats"]


@pytest.mark.parametrize("case", OP_CASES)
def test_update_op_vs_round16_oracle(case):
    from oracle import update_oracle
    m = _module()
    net, inp, corr, flow, ii = _case(case)
    got = m(net, inp, corr, flow, ii, ii)
    want = update_oracle.update_forward(m.state_dict(), net, inp, corr, flow, ii, round16=True)
    stats = {}
    _compare_op(got, want, stats, case)
    for k, v in stats.items():
        _record("operator " + k, v)
    # fixed summation order (GLO partials, scatter-mean): a second call is bit for bit the same
    again = m(net, inp, corr, flow, ii, ii)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    # FactorGraph's source-frame hint gives what torch.unique gives
    frames, slot = torch.unique(ii, sorted=True, return_inverse=True)
    m.set_source_frames(frames, slot)
    hinted = m(net, inp, corr, flow, ii, ii)
    assert all(torch.equal(a, b) for a, b in zip(got, hinted))


def test_update_op_no_flow_and_fp32_net():
    from oracle import update_oracle
    m = _module()
    net, inp, corr, flow, ii = _case("18_edges_30x40")
    stats = {}
    got = m(net, inp, corr, None, ii, ii)
    want = update_oracle.update_forward(m.state_dict(), net, inp, corr, None, ii, round16=True)
    _compare_op(got, want, stats, "no_flow")
    # an fp32 net (not fp16-representable) is rounded to fp16 on the way in; the new state comes back as fp32
    net32 = net.float() + torch.rand(net.shape, device=dev()) * 1e-4
    got32 = m(net32, inp, corr, flow, ii, ii)
    assert got32[0].dtype == torch.float32
    want = update_oracle.update_forward(m.state_dict(), net32, inp, corr, flow, ii, round16=True)
    _compare_op(got32, want, stats, "fp32_net")
    got16 = m(net32.half(), inp, corr, flow, ii, ii)
    assert torch.equal(got32[0], got16[0].float()) and all(torch.equal(a, b) for a, b in zip(got32[1:], got16[1:]))
    # ii = None: no GraphAgg, the first three outputs unchanged
    three = m(net32.half(), inp, corr, flow)
    assert len(three) == 3 and all(torch.equal(a, b) for a, b in zip(three, got16[:3]))
    for k, v in stats.items():
        _record("operator " + k, v)
