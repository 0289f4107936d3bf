"""GPU parity of the wgmma ConvGRU (SURVEY §8f-4, csrc/conv_tc.cu) behind the reference's module interface
(src/modules/gru.py): against the reference module's own output (tests/golden/conv_gru.npz, fp32 on the CPU) and
against the same arithmetic in plain torch on the GPU (fp32 math on the fp16-rounded operands the kernel sees)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def dev():
    return torch.device("cuda:0")


def _torch_gru(m, net, inp, corr, flow):
    """ConvGRU.forward in fp32 torch ops on fp16-rounded weights / inputs (what the kernel multiplies)"""
    def r(t):
        return t.half().float()
    w = lambda conv: r(conv.weight)                                              # noqa: E731
    x = torch.cat([r(inp), r(corr), r(flow)], dim=1)
    net = r(net)
    glo = (torch.sigmoid(F.conv2d(net, w(m.w), m.w.bias)) * net).mean(dim=(2, 3), keepdim=True)
    zin = torch.cat([net, x], dim=1)
    z = torch.sigmoid(F.conv2d(zin, w(m.convz), m.convz.bias, padding=1) + F.conv2d(glo, m.convz_glo.weight, m.convz_glo.bias))
    rr = torch.sigmoid(F.conv2d(zin, w(m.convr), m.convr.bias, padding=1) + F.conv2d(glo, m.convr_glo.weight, m.convr_glo.bias))
    q = torch.tanh(F.conv2d(torch.cat([r(rr * net), x], dim=1), w(m.convq), m.convq.bias, padding=1) +
                   F.conv2d(glo, m.convq_glo.weight, m.convq_glo.bias))
    return (1 - r(z)) * net + r(z) * q


def _module():
    from goslam_b200.modules.gru import ConvGRU
    torch.manual_seed(77)
    return ConvGRU(128, 128 + 128 + 64)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_conv_gru_vs_reference_module_golden(tag):
    g = np.load(os.path.join(HERE, "golden", "conv_gru.npz"))
    m = _module()
    assert abs(sum(float(p.double().sum()) for p in m.parameters()) - float(g[tag + "_wsum"])) < 1e-6   # same weights as the golden
    m = m.to(dev())
    args = [torch.from_numpy(g[tag + "_" + k]).to(dev()).float() for k in ("net", "inp", "corr", "flow")]
    out = m(*args)
    want = torch.from_numpy(g[tag + "_out"]).to(dev())
    assert out.shape == want.shape and out.dtype == args[0].dtype
    # fp16 operands (2^-11 relative each, 4032-term dot products) and fp16 state vs the fp32 reference
    assert (out - want).abs().max().item() < 1e-2
    assert (out - want).abs().mean().item() < 1e-3
    # the kernel's own arithmetic contract: fp32 accumulation over fp16 operands, fp16 z / r*net / state
    tight = _torch_gru(m, *args)
    assert (out - tight).abs().max().item() < 3e-3, (out - tight).abs().max().item()


@pytest.mark.parametrize("shape", [(36, 40, 80), (5, 30, 40), (2, 60, 80), (1, 9, 13)])
def test_conv_gru_shapes_vs_torch(shape):
    B, h, w = shape
    m = _module().to(dev())
    g = torch.Generator().manual_seed(h * w + B)
    net = torch.tanh(torch.randn(B, 128, h, w, generator=g)).to(dev())
    inp, corr = [torch.relu(torch.randn(B, 128, h, w, generator=g)).to(dev()) for _ in range(2)]
    flow = torch.relu(torch.randn(B, 64, h, w, generator=g)).to(dev())
    out = m(net, inp, corr, flow)
    tight = _torch_gru(m, net, inp, corr, flow)
    assert torch.isfinite(out).all()
    assert (out - tight).abs().max().item() < 3e-3, (out - tight).abs().max().item()
    # half-precision state in, half-precision state out (the graph keeps `net` in half)
    out16 = m(net.half(), inp.half(), corr.half(), flow.half())
    assert out16.dtype == torch.float16 and (out16.float() - out).abs().max().item() < 2e-3


def test_layout_helpers_round_trip():
    from goslam_b200.modules.gru import to_nchw, to_nhwc, to_nhwc_padded
    # generic + 64x64-tile paths; (2, 128, 9, 13): hw % 16 != 0 with C % 16 == 0; (2, 48, 8, 16): hw % 16 == 0 with
    # C % 64 != 0, which sends NHWC -> NCHW down the generic path
    for shape in [(3, 70, 11, 13), (5, 128, 40, 80), (2, 576, 30, 40), (2, 64, 12, 20), (3, 128, 9, 16), (2, 128, 9, 13),
                  (2, 48, 8, 16)]:
        x = torch.randn(*shape, device=dev()).half()
        y = to_nhwc(x)
        assert y.shape == (shape[0], shape[2], shape[3], shape[1]) and torch.equal(y, x.permute(0, 2, 3, 1).contiguous())
        assert torch.equal(to_nchw(y), x)
    for shape, cpad in [((4, 196, 40, 80), 256), ((2, 196, 30, 40), 256), ((2, 5, 7, 9), 16)]:
        x = torch.randn(*shape, device=dev()).half()
        y = to_nhwc_padded(x, cpad)
        assert torch.equal(y[..., :shape[1]], x.permute(0, 2, 3, 1)) and float(y[..., shape[1]:].abs().max()) == 0.0


def test_update_module_vs_reference_golden():
    """goslam_b200.droid_net.UpdateModule (the whole operator in one goslam_update_op call: wgmma encoders, ConvGRU,
    heads and GraphAgg in fp16 with fp32 accumulation) against the reference UpdateModule's fp32 outputs
    (tests/golden/update_module.npz): same parameter names (the `update.*` keys of pretrained/droid.pth load), same
    five outputs and shapes.  The tight per-layer and whole-operator checks are in test_gpu_update_op.py."""
    from goslam_b200.droid_net import UpdateModule
    g = np.load(os.path.join(HERE, "golden", "update_module.npz"))
    torch.manual_seed(78)
    m = UpdateModule()
    assert abs(sum(float(p.detach().double().sum()) for p in m.parameters()) - float(g["wsum"])) < 1e-5
    m = m.to(dev())
    t = lambda k: torch.from_numpy(g[k]).to(dev())                              # noqa: E731
    net, delta, weight, eta, upmask = m(t("net"), t("inp"), t("corr"), t("flow"), t("ii"), t("jj"))
    assert net.shape == (1, 6, 128, 16, 24) and delta.shape == weight.shape == (1, 6, 16, 24, 2)
    assert eta.shape == (1, 3, 16, 24) and upmask.shape == (1, 3, 576, 16, 24)
    # fp16 autocast arithmetic (the reference's own precision on a GPU) against the fp32 CPU run
    for name, got, want, tol in (("net", net, g["out_net"], 1.5e-2), ("delta", delta, g["out_delta"], 1.5e-2),
                                 ("weight", weight, g["out_weight"], 1e-2), ("eta", eta, g["out_eta"], 1e-3),
                                 ("upmask", upmask[:, :, ::9], g["out_upmask"], 2e-2)):
        err = (got.float().cpu() - torch.from_numpy(want).float()).abs()
        assert err.max().item() < tol, (name, err.max().item())
        assert err.mean().item() < tol / 8, (name, err.mean().item())
    # and as FactorGraph's update_op: one update of a small graph runs end to end
    import sys
    sys.path.insert(0, os.path.join(HERE, "tools"))
    import fg_scenario
    from goslam_b200.depth_video import DepthVideo
    from goslam_b200.factor_graph import FactorGraph
    cfg, args = fg_scenario.cfg_and_args("cuda:0")
    video = DepthVideo(cfg, args)
    fg_scenario.fill_video(video, fg_scenario.make_inputs())
    graph = FactorGraph(video, m, device="cuda:0", max_factors=40, upsample=True)
    graph.add_neighborhood_factors(0, 6, r=2)
    p0 = video.poses.clone()
    graph.update(1, use_inactive=True)
    graph.update(None, None, use_inactive=True)
    assert torch.isfinite(video.poses).all() and torch.isfinite(video.disps).all() and not torch.equal(video.poses, p0)
    assert graph.net.shape == (1, graph.ii.numel(), 128, 16, 24) and graph.weight.min().item() >= 0.0
