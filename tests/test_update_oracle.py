"""Pin the float64 restatement of the update operator (oracle/update_oracle.py) on the CPU against the reference's own
UpdateModule / ConvGRU outputs (tests/golden/update_module.npz, conv_gru.npz: fp32 on the CPU, default-initialised
weights under the seeds the goldens were written with).  test_gpu_update_op.py then compares the kernels with it."""
import os

import numpy as np
import pytest
import torch

from oracle import update_oracle

HERE = os.path.dirname(os.path.abspath(__file__))


def _golden(name):
    return np.load(os.path.join(HERE, "golden", name + ".npz"))


def _update_module(wsum):
    from goslam_b200.droid_net import UpdateModule
    torch.manual_seed(78)
    m = UpdateModule()
    assert abs(sum(float(p.detach().double().sum()) for p in m.parameters()) - wsum) < 1e-5   # the golden's weights
    return m.state_dict()


def _ulp16(x):
    """spacing of fp16 at |x| (2^-24 below the normal range)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def _run(g, round16, **kw):
    t = lambda k: torch.from_numpy(g[k])                                            # noqa: E731
    args = dict(net=t("net"), inp=t("inp"), corr=t("corr"), flow=t("flow"), ii=t("ii"))
    args.update(kw)
    return update_oracle.update_forward(_update_module(float(g["wsum"])), round16=round16, **args)


def test_update_oracle_exact_matches_reference_golden():
    """round16=False is the reference's arithmetic: agrees with its fp32 CPU run to fp32 accuracy (the golden `net` is
    stored as fp16, so it agrees to that rounding)."""
    g = _golden("update_module")
    net, delta, weight, eta, upmask = _run(g, round16=False)
    assert net.dtype == torch.float64
    want_net = torch.from_numpy(g["out_net"]).double()
    assert ((net - want_net).abs() <= 0.5 * _ulp16(want_net) + 2e-6).all()
    for name, got, key in (("delta", delta, "out_delta"), ("weight", weight, "out_weight"), ("eta", eta, "out_eta"),
                           ("upmask", upmask[:, :, ::9], "out_upmask")):
        want = torch.from_numpy(g[key]).double()
        err = (got - want).abs().max().item()
        assert err < 1e-5 * max(1.0, want.abs().max().item()), (name, err)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_conv_gru_oracle_matches_reference_golden(tag):
    from goslam_b200.modules.gru import ConvGRU
    g = _golden("conv_gru")
    torch.manual_seed(77)
    m = ConvGRU(128, 128 + 128 + 64)
    assert abs(sum(float(p.detach().double().sum()) for p in m.parameters()) - float(g[tag + "_wsum"])) < 1e-6
    args = [torch.from_numpy(g[tag + "_" + k]) for k in ("net", "inp", "corr", "flow")]
    want = torch.from_numpy(g[tag + "_out"]).double()
    exact = update_oracle.conv_gru(m.state_dict(), *args, round16=False)
    assert (exact - want).abs().max().item() < 1e-5
    # the kernels' rounding points: within what test_gpu_gru.py allows the kernel against this golden
    rounded = update_oracle.conv_gru(m.state_dict(), *args, round16=True)
    assert torch.equal(rounded, rounded.half().double())                            # net' is an fp16 value
    assert (rounded - want).abs().max().item() < 1e-2 and (rounded - want).abs().mean().item() < 1e-3


def test_update_oracle_round16_within_golden_tolerances():
    """round16=True agrees with the fp32 reference within the tolerances test_update_module_vs_reference_golden allows
    the kernels, and its fp16 outputs are fp16 values."""
    g = _golden("update_module")
    net, delta, weight, eta, upmask = _run(g, round16=True)
    for name, got, want, tol in (("net", net, g["out_net"], 1.5e-2), ("delta", delta, g["out_delta"], 1.5e-2),
                                 ("weight", weight, g["out_weight"], 1e-2), ("eta", eta, g["out_eta"], 1e-3),
                                 ("upmask", upmask[:, :, ::9], g["out_upmask"], 2e-2)):
        err = (got - torch.from_numpy(want).double()).abs()
        assert err.max().item() < tol, (name, err.max().item())
        assert err.mean().item() < tol / 8, (name, err.mean().item())
    assert torch.equal(net, net.half().double()) and torch.equal(upmask, upmask.half().double())
    # delta / weight / eta are fp32 results in the kernels: not rounded to fp16 here
    assert not torch.equal(delta, delta.half().double()) and not torch.equal(eta, eta.half().double())


def test_update_oracle_shapes_row_order_and_no_flow():
    g = _golden("update_module")
    # unsorted ii with repeats: one row per distinct frame, in sorted frame order, each the mean over its edges
    ii = torch.tensor([3, 0, 3, 5, 0, 3])
    full = _run(g, round16=False, ii=ii)
    net, delta, weight, eta, upmask = full
    assert net.shape == (1, 6, 128, 16, 24) and delta.shape == weight.shape == (1, 6, 16, 24, 2)
    assert eta.shape == (1, 3, 16, 24) and upmask.shape == (1, 3, 576, 16, 24)
    for row, frame in enumerate((0, 3, 5)):
        # GraphAgg for one frame alone: the same row, computed from that frame's edges only
        sel = (ii == frame).nonzero().flatten()
        sub = _run(g, round16=False, net=torch.from_numpy(g["net"])[:, sel], inp=torch.from_numpy(g["inp"])[:, sel],
                   corr=torch.from_numpy(g["corr"])[:, sel], flow=torch.from_numpy(g["flow"])[:, sel], ii=ii[sel])
        assert sub[3].shape[1] == 1
        assert torch.allclose(sub[3][:, 0], eta[:, row], rtol=0, atol=1e-12)
        assert torch.allclose(sub[4][:, 0], upmask[:, row], rtol=0, atol=1e-10)
    # ii = None: the first three outputs only, unchanged
    three = _run(g, round16=False, ii=None)
    assert len(three) == 3 and all(torch.equal(a, b) for a, b in zip(three, full[:3]))
    # flow = None is a zero motion input
    t = torch.from_numpy
    zero = torch.zeros_like(t(g["flow"]))
    a = _run(g, round16=True, flow=None)
    b = _run(g, round16=True, flow=zero)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(a[1], _run(g, round16=True)[1])
