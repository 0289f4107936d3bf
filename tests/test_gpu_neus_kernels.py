"""The NeuS renderer's kernels one by one (csrc/neus.cu) against plain high-precision restatements:
  * goslam_neus_forward at every sample-count layout the warp work split produces, in its persistent loop, and in the
    nothing-in-bound fallback (the reference's `pts_mask[:100] = True`), against oracle/neus_oracle.py;
  * goslam_neus_composite_backward and goslam_neus_grid_backward against the float64 closed forms of
    oracle/neus_grad_oracle.py (themselves pinned to autograd in tests/test_neus_grad_oracle.py);
  * goslam_neus_mlp_backward against a float64 restatement rounded to fp16 where the kernel rounds.
Each tolerance sits next to its assertion with the reason for it."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import neus_grad_oracle as ngo
from oracle import neus_oracle

pytestmark = pytest.mark.gpu

BOUND = [[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]]
RT = [[-1.8, 1.9], [-2.0, 2.0], [-1.5, 2.0]]
FALLBACK_RT = [[1.9, 1.99], [1.9, 1.99], [1.9, 1.99]]      # a corner box no ray of make_rays reaches
EPS32 = 2.0 ** -24


def dev():
    return torch.device("cuda:0")


def _weights(seed=7):
    from goslam_b200 import neus, synthetic
    offs, ress, _, total = neus.hashgrid_layout()
    return synthetic.make_neus_weights(seed=seed, total_grid_params=total, layout=(offs, ress))


def _net(w, bound=BOUND, rt=RT):
    from goslam_b200 import neus, synthetic
    net = neus.InstantNeuS(synthetic.NEUS_CFG, bound)
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to(dev())
    net.update_bound(torch.tensor(rt, dtype=torch.float32))
    return net


def _rays(R, S, seed, shift=None):
    from goslam_b200 import synthetic
    ro, rd, zv, ds = synthetic.make_rays(R, S=S, seed=seed, n_uniform=min(24, max(1, S // 3)))
    if shift is not None:
        ro = (ro + torch.tensor(shift, dtype=torch.float32)).contiguous()
    return ro, rd, zv, ds


def _oracle(w, rays, bound=BOUND, rt=RT):
    return neus_oracle.forward(w["grid"].half().numpy(), w["sdf_w"].numpy(), w["sdf_b"].numpy(), w["color_B"].numpy(),
                               w["mlp"].half().numpy(), np.array(bound, np.float32), np.array(rt, np.float32), 0.2, 10.0,
                               *[t.numpy() for t in rays], debug=True)


def _run(net, rays):
    out = net(*[t.to(dev()) for t in rays], debug=True)
    return {k: v.cpu().numpy() for k, v in out.items()}, {k: v.cpu().numpy() for k, v in net.last_debug.items()}


def _rel(a, b):
    return np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max() / max(np.abs(b).max(), 1e-12)


def _check_forward(got, dbg, ref, gerr=True):
    """the assertions of test_gpu_parity.py::test_neus_forward, for any ray slice"""
    for k in ("z_vals", "sdf", "sdf_variance"):                # per-sample values before the NeuS alpha: 1e-4 relative
        assert got[k].shape == ref[k].shape, k
        assert _rel(got[k], ref[k]) < 1e-4, (k, _rel(got[k], ref[k]))
    inb = ref["sdf"] != 100.0
    assert np.array_equal(inb, got["sdf"] != 100.0)
    if inb.any():
        assert np.abs(got["sdf"][inb] - ref["sdf"][inb]).max() < 1e-4 * np.abs(ref["sdf"][inb]).max()
    assert np.abs(dbg["alpha"] - ref["_alpha"]).max() < 1e-5
    assert np.abs(dbg["grad"].reshape(-1, 3) - ref["_grad"]).max() < 1e-5 * max(1.0, np.abs(ref["_grad"]).max())
    assert np.array_equal(dbg["pos"].reshape(-1, 3)[ref["_mask"]], ref["_xn"])          # bit-identical positions
    for k in ("depth", "weight_sum", "depth_variance"):                                # composited: 1e-4 relative
        assert got[k].shape == ref[k].shape, k
        assert _rel(got[k], ref[k]) < 1e-4, (k, _rel(got[k], ref[k]))
    # the normal is a weighted sum of per-sample normals that may cancel (when few rays render, its largest value can be
    # far below the terms): 1e-4 of the larger of that value and the largest ray's sum of |normal| x weight
    R, S = ref["sdf"].shape
    scale = (np.linalg.norm(ref["_grad"], axis=1).reshape(R, S) * ref["_weights"]).sum(1).max()
    assert got["normal"].shape == ref["normal"].shape
    assert np.abs(got["normal"] - ref["normal"]).max() < 1e-4 * max(np.abs(ref["normal"]).max(), scale, 1e-12)
    # colour: fp16 activations and sigmoid output per sample; one rounding flip of one sample moves the composited colour
    # by at most weight * 2^-11, so half an fp16 ulp of a value in [0.5, 1) absolute for every ray
    cerr = np.abs(got["color"] - ref["color"]).max(1)
    assert cerr.max() < 2.5e-4, float(cerr.max())
    if gerr:
        assert abs(float(got["gradient_error"][0]) - float(ref["gradient_error"][0])) <= 2e-3 * abs(float(ref["gradient_error"][0]))


# ------------------------------------------------------------------------------------------------ forward layouts
def _group(S):
    """rays one warp composites together (goslam_neus_forward): G = 32 / gcd(S, 32), capped so that G * S <= 288"""
    import math
    G = 32 // math.gcd(S, 32)
    return G if G * S <= 288 else 288 // S


# (R, S): the config counts 24 / 48 / 72, then S = 1 (G = 32), 31 (G = 9, G*S = 279: partial last tile), 33 (G = 8, 264:
# partial), 96 (G = 1, 3 tiles per ray), 100 (G = 2, a ray over 4 tiles), 200 (G = 1, 7 tiles, partial), 288 (G = 1, 9
# tiles).  Every R leaves the last group partial.
FORWARD_LAYOUTS = [(37, 24), (37, 48), (37, 72), (70, 1), (40, 31), (37, 33), (37, 96), (37, 100), (23, 200), (19, 288)]


@pytest.mark.parametrize("R,S", FORWARD_LAYOUTS)
def test_neus_forward_sample_counts(R, S):
    G = _group(S)
    assert R % G != 0 or G == 1
    w = _weights()
    net = _net(w)
    rays = _rays(R, S, seed=11 + S)
    got, dbg = _run(net, rays)
    ref = _oracle(w, rays)
    if S >= 24:
        assert (ref["weight_sum"] > 1e-3).mean() > 0.2, "degenerate test scene: nothing is rendered"
    _check_forward(got, dbg, ref)


@pytest.mark.parametrize("S", [0, 289])
def test_neus_forward_rejects_sample_counts_out_of_range(S):
    net = _net(_weights())
    z = torch.zeros((4, S), device=dev())
    o = torch.zeros((4, 3), device=dev())
    with torch.no_grad(), pytest.raises(RuntimeError, match="neus_forward"):
        net(o, o, z, z)


# ------------------------------------------------------------------------------------------------ persistent loop
@pytest.mark.parametrize("R,S", [(5001, 96), (7002, 72)])
def test_neus_forward_persistent_loop(R, S):
    """132 blocks x 12 warps = 1584 warps: here every warp takes several groups.  The grouping depends on the ray index
    only, so the rays give the same bits when run as separate calls split at multiples of G."""
    G = _group(S)
    assert (R + G - 1) // G > 1584
    w = _weights()
    net = _net(w)
    rays = _rays(R, S, seed=5)
    whole, _ = _run(net, rays)
    cuts = [0, 333 * G, 1100 * G, R]
    parts = [_run(net, [t[a:b] for t in rays])[0] for a, b in zip(cuts[:-1], cuts[1:])]
    for k in ("color", "depth", "depth_variance", "normal", "weight_sum", "sdf", "z_vals"):
        assert np.array_equal(whole[k], np.concatenate([p[k] for p in parts])), k
    # gradient_error: per-block partials reduced in float64 then rounded; the split sums in a different order
    ge = sum(float(p["gradient_error"][0]) * (b - a) for p, a, b in zip(parts, cuts[:-1], cuts[1:])) / R
    assert abs(float(whole["gradient_error"][0]) - ge) <= 1e-6 * abs(ge)
    # the last 300+ rays (the last, partial group included) against the oracle
    lo = R - 301
    sl = [t[lo:] for t in rays]
    _, dbg = _run(net, sl)
    _check_forward({k: v[lo:] if v.shape[0] == R else v for k, v in whole.items()}, dbg, _oracle(w, sl), gerr=False)


# ------------------------------------------------------------------------------------------------ nothing in bound
# (name, R, S, bound, rt_bound, ray shift): the forced 100 samples cross ray boundaries (S = 24), at S = 72, within the
# first ray (S = 128), R*S < 100 (every sample forced), and an rt_bound that contains `bound` with every sample outside
# both: the forced samples clamp to x01 = 1 (x) and 0 (y), where the dense levels' +1 corner wraps around
FALLBACK_CASES = [
    ("s24", 13, 24, BOUND, FALLBACK_RT, None),
    ("s72", 9, 72, BOUND, FALLBACK_RT, None),
    ("s128", 5, 128, BOUND, FALLBACK_RT, None),
    ("tiny", 3, 24, BOUND, FALLBACK_RT, None),
    ("clamped", 11, 24, [[-1.0, 1.0]] * 3, [[-1.5, 1.5]] * 3, (4.0, -4.0, 0.0)),
]


def _fallback_inputs(case):
    name, R, S, bound, rt, shift = case
    rays = _rays(R, S, seed=40 + S, shift=shift)
    ro, rd, zv, ds = [t.numpy() for t in rays]
    pts = (ro[:, None] + rd[:, None] * (zv + ds / np.float32(2))[..., None]).reshape(-1, 3)
    rta = np.array(rt, np.float32)
    assert not np.any(np.all((pts > rta[:, 0]) & (pts < rta[:, 1]), axis=1)), "a sample is in bound: not a fallback case"
    return rays, bound, rt


@pytest.mark.parametrize("case", FALLBACK_CASES, ids=[c[0] for c in FALLBACK_CASES])
def test_neus_forward_nothing_in_bound(case):
    rays, bound, rt = _fallback_inputs(case)
    w = _weights()
    net = _net(w, bound, rt)
    got, dbg = _run(net, rays)
    ref = _oracle(w, rays, bound, rt)
    n = rays[2].numel()
    assert np.array_equal(ref["_mask"], np.arange(n) < 100)
    if case[0] != "clamped":                # there the forced samples sit on one clamped point: any alpha will do
        assert ref["weight_sum"].max() > 1e-3, "degenerate case: the forced samples render nothing"
    _check_forward(got, dbg, ref)
    if case[0] == "clamped":
        xn = dbg["pos"].reshape(-1, 3)[:min(n, 100)]
        assert np.all(xn[:, 0] == 1.0) and np.all(xn[:, 1] == -1.0)
    # a normal batch right after: the same bits as on a fresh net (no state carried over from the fallback)
    net.update_bound(torch.tensor(RT))
    after, _ = _run(net, _rays(40, 72, seed=3))
    fresh, _ = _run(_net(w, bound, RT), _rays(40, 72, seed=3))
    for k in fresh:
        assert np.array_equal(after[k], fresh[k]), k


# ------------------------------------------------------------------------------------------------ composite backward
def _train_forward(net, rays):
    out = net._forward_impl(*[t.to(dev()) for t in rays], train=True)
    return out, net.last_debug


def _comp_bwd(net, rays, out, saved, dc, dd, dsd, dge, r0=0, r1=None):
    """goslam_neus_composite_backward on rays [r0, r1) of a forward call"""
    from goslam_b200 import _lib
    R, S = out["sdf"].shape
    r1 = R if r1 is None else r1
    p, keep, _ = net._params_struct()
    ro, rd, zv, ds = [t.to(dev()).contiguous() for t in rays]
    sl = slice(r0, r1)
    n = (r1 - r0) * S
    f32 = dict(dtype=torch.float32, device=dev())
    d_y, d_s, d_g, d_inv = torch.full((n, 3), 7.0, **f32), torch.full((n,), 7.0, **f32), torch.full((n, 3), 7.0, **f32), torch.zeros(1, **f32)
    keepalive = [t[sl].contiguous() for t in (ro, rd, ds, saved["alpha"], saved["rgb"], out["sdf"], saved["grad"], out["z_vals"])]
    ups = [None if t is None else (t[sl].contiguous() if t.shape[0] == R else t) for t in (dc, dd, dsd, dge)]
    rc = _lib.load().goslam_neus_composite_backward(
        ctypes.byref(p), *[_lib.ptr(t) for t in keepalive], *[_lib.ptr(t) for t in ups], _lib.ptr(saved["fallback"]),
        ctypes.c_int64(R * S), ctypes.c_int64(r0 * S), r1 - r0, S, _lib.ptr(d_y), _lib.ptr(d_s), _lib.ptr(d_g), _lib.ptr(d_inv),
        _lib.stream_ptr())
    return rc, d_y.cpu().numpy().reshape(r1 - r0, S, 3), d_s.cpu().numpy().reshape(r1 - r0, S), \
        d_g.cpu().numpy().reshape(r1 - r0, S, 3), float(d_inv[0])


def _comp_reference(net, rays, out, saved, dc, dd, dsd, dge, r0, r1):
    R, S = out["sdf"].shape
    sl = slice(r0, r1)
    c = lambda t: None if t is None else t.detach().cpu().numpy().astype(np.float64)   # noqa: E731
    alpha, rgb, grad = c(saved["alpha"])[sl], c(saved["rgb"])[sl], c(saved["grad"])[sl]
    sdf, zm = c(out["sdf"])[sl], c(out["z_vals"])[sl]
    dists, dirs = rays[3].numpy().astype(np.float64)[sl], rays[1].numpy().astype(np.float64)[sl]
    inb = sdf != 100.0                                              # the forward's own in-bound set (forced samples included)
    inv_s = float(net._params_struct()[2])
    want = ngo.composite_backward_closed_form(alpha, rgb, sdf, grad, zm, dists, dirs, inb, np.float32(inv_s),
                                              None if dc is None else c(dc)[sl], None if dd is None else c(dd)[sl],
                                              None if dsd is None else c(dsd)[sl], None if dge is None else float(dge[0]),
                                              total_samples=R * S)
    # error scales: every term of dL/dalpha_s is bounded by A_r = sum_s |G_s| T_s + |G_s w_s| / (1 - alpha_s); the kernel
    # forms the suffix sums in fp32 across the ray's chunks, so its dL/dalpha is within ~S eps A_r; that error reaches
    # d_sdf / d_normal / d_inv_s through J_s = inv_s |d(p - n ...)/d alpha chain| (computed here in float64)
    dcol = np.zeros((r1 - r0, 3)) if dc is None else c(dc)[sl]
    ddep = np.zeros((r1 - r0, 1)) if dd is None else c(dd)[sl].reshape(-1, 1)
    T = np.cumprod(np.concatenate([np.ones((r1 - r0, 1)), 1.0 - alpha + 1e-7], axis=1), axis=1)[:, :-1]
    G = (rgb * dcol[:, None, :]).sum(-1) + ddep * zm
    A = (np.abs(G) * T + np.abs(G * alpha * T) / (1.0 - alpha + 1e-7)).sum(1, keepdims=True)
    tc = (dirs[:, None, :] * grad).sum(-1)
    hs = -np.maximum(-tc, 0) * dists / 2.0                          # cos_anneal_ratio = 1
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))                       # noqa: E731
    pp, nn = sig((sdf - hs) * inv_s), sig((sdf + hs) * inv_s)
    J = inv_s * (nn / (pp + 1e-5) ** 2 * pp * (1 - pp) + nn * (1 - nn) / (pp + 1e-5)) * inb
    return want, A, J, hs, sdf, inv_s


COMP_S = [1, 24, 31, 32, 33, 48, 72, 96, 127, 128]


@pytest.mark.parametrize("S", COMP_S)
@pytest.mark.parametrize("null", ["none", "d_color", "d_depth", "d_sdf", "d_gradient_error"])
def test_composite_backward_matches_closed_form(S, null):
    w = _weights(5)
    net = _net(w)
    R = 45
    rays = _rays(R, S, seed=60 + S)
    out, saved = _train_forward(net, rays)
    g = torch.Generator().manual_seed(S)
    ups = {"d_color": torch.randn(R, 3, generator=g), "d_depth": torch.randn(R, 1, generator=g),
           "d_sdf": 0.1 * torch.randn(R, S, generator=g), "d_gradient_error": torch.tensor([3.0])}
    if null != "none":
        ups[null] = None
    ups = {k: None if v is None else v.to(dev()) for k, v in ups.items()}
    args = (ups["d_color"], ups["d_depth"], ups["d_sdf"], ups["d_gradient_error"])
    _check_comp(net, rays, out, saved, args, 0, R)


def test_composite_backward_on_a_slice_of_a_larger_call():
    """total_samples != R*S: a ray slice of a forward call; the eikonal term still averages over the whole call"""
    net = _net(_weights(5))
    R, S = 64, 72
    rays = _rays(R, S, seed=77)
    out, saved = _train_forward(net, rays)
    g = torch.Generator().manual_seed(1)
    args = (torch.randn(R, 3, generator=g).to(dev()), torch.randn(R, 1, generator=g).to(dev()),
            (0.1 * torch.randn(R, S, generator=g)).to(dev()), torch.tensor([3.0], device=dev()))
    _check_comp(net, rays, out, saved, args, 20, 51)


def test_composite_backward_with_forced_samples():
    """nothing in bound at S = 24: the 100 forced samples get gradients (the forward's fallback flag and sample0)"""
    net = _net(_weights(5), BOUND, FALLBACK_RT)
    rays = _rays(13, 24, seed=64)
    out, saved = _train_forward(net, rays)
    assert int(saved["fallback"][0]) == 1
    g = torch.Generator().manual_seed(2)
    args = (torch.randn(13, 3, generator=g).to(dev()), torch.randn(13, 1, generator=g).to(dev()),
            (0.1 * torch.randn(13, 24, generator=g)).to(dev()), torch.tensor([3.0], device=dev()))
    for r0, r1 in ((0, 13), (2, 7), (4, 13)):                       # slices whose first sample is 48 / 96 of the call
        d_s = _check_comp(net, rays, out, saved, args, r0, r1)
        forced = (np.arange(r0 * 24, r1 * 24) < 100).reshape(r1 - r0, 24)
        assert np.all(d_s[~forced] == 0.0) and np.count_nonzero(d_s[forced]) > 0.9 * forced.sum()


def _check_comp(net, rays, out, saved, args, r0, r1):
    R, S = out["sdf"].shape
    rc, d_y, d_s, d_g, d_inv = _comp_bwd(net, rays, out, saved, *args, r0=r0, r1=r1)
    assert rc == 0
    (w_y, w_s, w_g, w_inv), A, J, hs, sdf, inv_s = _comp_reference(net, rays, out, saved, *args, r0, r1)
    K = (8 * S + 64) * EPS32
    dc = np.zeros((r1 - r0, 3)) if args[0] is None else args[0].cpu().numpy()[r0:r1]
    wts = np.abs(saved["alpha"].cpu().numpy()[r0:r1])
    # d(pre-sigmoid colour) = d_color w rgb (1 - rgb): w from the kernel's fp32 scan of the saved alpha, ~S eps relative
    assert np.all(np.abs(d_y - w_y) <= K * (np.abs(w_y) + np.abs(dc).max(1)[:, None, None] * wts[..., None]) + 1e-30)
    # d sdf: the closed form's value, plus J_s times the fp32 error of dL/dalpha; the upstream d_sdf adds exactly
    assert np.all(np.abs(d_s - w_s) <= K * (np.abs(w_s) + J * A) + 1e-30), np.abs(d_s - w_s).max()
    # d normal: the alpha path scales dL/d(half step) by dist / 2 along the ray direction; the eikonal term is per sample
    dirn = np.linalg.norm(rays[1].numpy()[r0:r1], axis=1)[:, None]
    dists = rays[3].numpy()[r0:r1]
    gn = np.linalg.norm(saved["grad"].cpu().numpy()[r0:r1], axis=-1)
    eik = 0.0 if args[3] is None else 2.0 * float(args[3][0]) / (R * S) * (1.0 + gn)
    bg = K * (np.linalg.norm(w_g, axis=-1) + J * A * dists / 2 * dirn + eik)
    assert np.all(np.linalg.norm(d_g - w_g, axis=-1) <= bg + 1e-30), np.abs(d_g - w_g).max()
    # d inv_s: a float sum over every sample of terms bounded by A J / inv_s (|sdf| + |h|)
    inb = sdf != 100.0
    binv = K * ((A * J / inv_s * (np.abs(np.where(inb, sdf, 0)) + np.abs(hs))).sum() + abs(w_inv))
    assert abs(d_inv - w_inv) <= binv, (d_inv, w_inv, binv)
    # samples the forward kept out of the network: exact zeros
    assert np.all(d_y[~inb] == 0) and np.all(d_g[~inb] == 0) and np.all(d_s[~inb] == 0)
    return d_s


def test_composite_backward_rejects_more_than_128_samples():
    from goslam_b200 import _lib
    net = _net(_weights(5))
    p, keep, _ = net._params_struct()
    buf = torch.zeros(4 * 129 * 3, device=dev())
    b = _lib.ptr(buf)
    rc = _lib.load().goslam_neus_composite_backward(ctypes.byref(p), b, b, b, b, b, b, b, b, None, None, None, None, None,
                                                    ctypes.c_int64(4 * 129), ctypes.c_int64(0), 4, 129, b, b, b, b,
                                                    _lib.stream_ptr())
    assert rc == -1          # GOSLAM_EINVAL


def test_training_forward_rejects_more_than_128_samples():
    net = _net(_weights(5))
    rays = [t.to(dev()) for t in _rays(4, 160, seed=1)]
    with torch.enable_grad(), pytest.raises(RuntimeError, match="at most 128 samples"):
        net(*rays)
    with torch.no_grad():                                  # the forward alone takes up to 288
        net(*rays)


# ------------------------------------------------------------------------------------------------ grid backward
def _crafted_points(rng):
    """sample positions (S = 1: sample i is ray i, at rays_o[i]) that stress the scatter's same-cell run reduction"""
    pts = []
    base = np.array([0.3, -0.7, 0.45], np.float32)
    pts.append(base + rng.uniform(0, 2e-3, (96, 3)).astype(np.float32))        # 3 warps in one coarse cell
    a, b = np.array([0.3, 0.2, 0.1], np.float32), np.array([-0.9, 1.1, 0.6], np.float32)
    pts.append(np.stack([a if i % 2 == 0 else b for i in range(64)]))            # lanes alternating between two cells
    pts.append(np.stack([a if (i // 3) % 2 == 0 else b for i in range(64)]))     # runs of 3
    face = rng.uniform(-1.5, 1.5, (32, 3)).astype(np.float32)
    face[np.arange(32), rng.integers(0, 3, 32)] = 0.0                           # x01 = 0.5: on level-0 cell faces
    face[::4] = 0.0
    pts.append(face)
    edge = rng.uniform(-1.5, 1.5, (64, 3)).astype(np.float32)                  # outside `bound`, inside rt_bound:
    edge[:, 0] = np.where(np.arange(64) % 2 == 0, 2.5, -2.5)                    # x01 exactly 1 or 0 (clamped)
    edge[::3, 1] = 2.7
    pts.append(edge)
    pts.append(rng.uniform(-1.9, 1.9, (100, 3)).astype(np.float32))
    return np.concatenate(pts).astype(np.float32)


def _grid_case(layout):
    """(rays, rt_bound, d_enc [n,32], d_grad [n,3]) in numpy"""
    rng = np.random.default_rng(3)
    if layout == "crafted":
        pts = _crafted_points(rng)
        n = pts.shape[0]
        rays = (pts, np.zeros((n, 3), np.float32), np.full((n, 1), 0.5, np.float32), np.full((n, 1), 0.1, np.float32))
        rt = [[-3.0, 3.0]] * 3
    else:
        rays = tuple(t.numpy() for t in _rays(40, 72, seed=12))
        rt = RT
        n = rays[2].size
    d_enc = rng.normal(0, 1, (n, 32)).astype(np.float32)
    d_grad = rng.normal(0, 1, (n, 3)).astype(np.float32)
    return rays, rt, d_enc, d_grad


def _grid_positions(rays, rt, bound=BOUND):
    """the kernel's sample positions, in-bound mask, x01 and d xn / d p, op by op in fp32"""
    ro, rd, zv, ds = rays
    S = zv.shape[1]
    zm = (zv + ds / np.float32(2)).astype(np.float32)
    pt = (np.repeat(ro, S, 0) + np.repeat(rd, S, 0) * zm.reshape(-1, 1)).astype(np.float32)
    rta = np.array(rt, np.float32)
    inb = np.all((pt > rta[:, 0]) & (pt < rta[:, 1]), axis=1)
    b = np.array(bound, np.float32)
    raw = (((pt - b[:, 0]) / (b[:, 1] - b[:, 0])) * np.float32(2) - np.float32(1)).astype(np.float32)
    xn = np.clip(raw, -1, 1).astype(np.float32)
    x01 = ((xn + np.float32(1)) / np.float32(2)).astype(np.float32)
    dscale = np.where((raw >= -1) & (raw <= 1), np.float32(2) / (b[:, 1] - b[:, 0]), 0).astype(np.float32)
    return inb, x01, dscale


@pytest.mark.parametrize("layout", ["crafted", "rays"])
@pytest.mark.parametrize("scaled", [False, True])
def test_grid_backward_matches_closed_form_per_entry(layout, scaled):
    from goslam_b200 import _lib
    w = _weights(5)
    rays, rt, d_enc, d_grad = _grid_case(layout)
    net = _net(w, BOUND, rt)
    p, keep, _ = net._params_struct()
    inb, x01, dscale = _grid_positions(rays, rt)
    assert inb.sum() > 100
    R, S = rays[2].shape
    sc = 256.0 if scaled else 1.0
    td = [torch.from_numpy(np.ascontiguousarray(t)).to(dev()) for t in rays]
    t_enc = torch.from_numpy(d_enc * np.float32(sc)).to(dev())
    t_scale = torch.tensor([sc], device=dev())
    t_grad = torch.from_numpy(d_grad).to(dev())
    gg = torch.zeros(w["grid"].numel(), device=dev())
    dw0 = torch.zeros(35, device=dev())
    rc = _lib.load().goslam_neus_grid_backward(ctypes.byref(p), *[_lib.ptr(t) for t in td], None, ctypes.c_int64(0), R, S,
                                               _lib.ptr(t_enc), _lib.ptr(t_scale) if scaled else None, _lib.ptr(t_grad),
                                               _lib.ptr(gg), _lib.ptr(dw0), _lib.stream_ptr())
    assert rc == 0
    got = gg.cpu().numpy().reshape(-1, 2).astype(np.float64)
    table = w["grid"].half().numpy().reshape(-1, 2)
    gy = w["sdf_w"][0, 3:].half().float().numpy()
    q = (np.float32(0.5) * dscale * d_grad).astype(np.float32)
    want, want_gy, a_tab, a_gy = ngo.grid_backward_closed_form(x01[inb], table, d_enc[inb], q[inb], gy, with_abs=True)
    # touched entries: every entry a contribution reaches and no other (a non-zero float64 sum of non-zero terms that
    # comes out as exactly 0.0 in fp32 is measure-zero for these random inputs)
    assert np.array_equal(got != 0, a_tab != 0)
    # fp32 products and reductions (runs of lanes, then atomics in scheduling order): error <= n eps sum|contribution|;
    # 1024 eps covers the coarse entries with ~1000 contributions at worst-case growth
    bound = 1024 * EPS32 * a_tab
    bad = np.abs(got - want) > bound
    assert not bad.any(), (int(bad.sum()), np.abs(got - want)[bad][:5], bound[bad][:5])
    d = dw0.cpu().numpy().astype(np.float64)
    assert np.all(np.abs(d[3:] - want_gy) <= 1024 * EPS32 * a_gy + 1e-30)
    xyz = (dscale[inb].astype(np.float64) * d_grad[inb]).sum(0)
    a_xyz = np.abs(dscale[inb].astype(np.float64) * d_grad[inb]).sum(0)
    assert np.all(np.abs(d[:3] - xyz) <= 1024 * EPS32 * a_xyz)


def test_grid_backward_with_forced_samples():
    """nothing in bound: with the forward's flag set, the call's first 100 samples scatter (sample0 places a slice)"""
    from goslam_b200 import _lib
    w = _weights(5)
    rays = [t.numpy() for t in _rays(13, 24, seed=64)]
    net = _net(w, BOUND, FALLBACK_RT)
    p, keep, _ = net._params_struct()
    rng = np.random.default_rng(8)
    d_enc, d_grad = rng.normal(size=(13 * 24, 32)).astype(np.float32), rng.normal(size=(13 * 24, 3)).astype(np.float32)
    _, x01, dscale = _grid_positions(rays, FALLBACK_RT)
    flag = torch.ones(1, dtype=torch.int32, device=dev())
    table = w["grid"].half().numpy().reshape(-1, 2)
    gy = w["sdf_w"][0, 3:].half().float().numpy()
    q = (np.float32(0.5) * dscale * d_grad).astype(np.float32)
    for r0, r1 in ((0, 13), (2, 5), (4, 13)):
        sl = slice(r0 * 24, r1 * 24)
        td = [torch.from_numpy(np.ascontiguousarray(t[r0:r1])).to(dev()) for t in rays]
        gg, dw0 = torch.zeros(w["grid"].numel(), device=dev()), torch.zeros(35, device=dev())
        t_enc, t_grad = torch.from_numpy(d_enc[sl].copy()).to(dev()), torch.from_numpy(d_grad[sl].copy()).to(dev())
        rc = _lib.load().goslam_neus_grid_backward(ctypes.byref(p), *[_lib.ptr(t) for t in td], _lib.ptr(flag),
                                                   ctypes.c_int64(r0 * 24), r1 - r0, 24, _lib.ptr(t_enc), None,
                                                   _lib.ptr(t_grad), _lib.ptr(gg), _lib.ptr(dw0), _lib.stream_ptr())
        assert rc == 0
        forced = np.arange(r0 * 24, r1 * 24) < 100
        got = gg.cpu().numpy().reshape(-1, 2)
        if not forced.any():
            assert not np.any(got) and not np.any(dw0.cpu().numpy())
            continue
        f = np.flatnonzero(forced) + r0 * 24
        want, _, a_tab, _ = ngo.grid_backward_closed_form(x01[f], table, d_enc[f], q[f], gy, with_abs=True)
        assert np.array_equal(got != 0, a_tab != 0)
        assert np.all(np.abs(got - want) <= 1024 * EPS32 * a_tab)


# ------------------------------------------------------------------------------------------------ MLP backward
def _ulp16(x):
    """spacing of fp16 at |x| (2^-24 below the normal range)"""
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -14)))
    return 2.0 ** (e - 10)


def _f16(x):
    return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def _near16(got, want, acc):
    """got (fp16 out of an fp32 accumulation) within one fp16 ulp of the exact value plus the accumulation error term"""
    got = np.asarray(got, np.float64)
    return np.abs(got - want) <= _ulp16(np.abs(want) + acc) + acc


@pytest.mark.parametrize("scale_log2", [0, 16])
def test_mlp_backward_matches_float64_restatement(scale_log2):
    from goslam_b200 import _lib
    from goslam_b200.neus import MLP_HID, MLP_IN_PAD
    w = _weights(5)
    net = _net(w)
    R, S = 50, 72                                             # 3600 rows: 112.5 warp tiles, the last partial
    rays = _rays(R, S, seed=9)
    out, saved = _train_forward(net, rays)
    n = R * S
    sc = 2.0 ** scale_log2
    rng = np.random.default_rng(scale_log2)
    d_y = (rng.normal(size=(n, 3)) / sc).astype(np.float32)    # d_y * scale is O(1) in both cases
    d_s = (rng.normal(size=n) / sc).astype(np.float32)
    d_g = rng.normal(size=(n, 3)).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev())   # noqa: E731
    f16 = dict(dtype=torch.float16, device=dev())
    H1, H2, dH1, dH2 = (torch.empty(n, MLP_HID, **f16) for _ in range(4))
    dY8, pts_hl, dE, h, d_out = (torch.empty(n, 8, **f16), torch.empty(n, 8, **f16), torch.empty(n, 40, **f16),
                                 torch.empty(n, 40, **f16), torch.empty(n, 32, **f16))
    d_gt = torch.empty(n, 3, device=dev())
    mo = _lib.NeusMlpBwdOut()
    mo.H1, mo.H2, mo.dH1, mo.dH2 = H1.data_ptr(), H2.data_ptr(), dH1.data_ptr(), dH2.data_ptr()
    mo.dY8, mo.dE, mo.d_out, mo.h = dY8.data_ptr(), dE.data_ptr(), d_out.data_ptr(), h.data_ptr()
    mo.pts_hl, mo.d_grad_total = pts_hl.data_ptr(), d_gt.data_ptr()
    p, keep, _ = net._params_struct()
    ro, rd = rays[0].to(dev()), rays[1].to(dev())
    t_y, t_s, t_g, t_sc = T(d_y), T(d_s), T(d_g), torch.tensor([sc], device=dev())
    rc = _lib.load().goslam_neus_mlp_backward(ctypes.byref(p), _lib.ptr(saved["mlp_in"]), _lib.ptr(saved["enc"]),
                                              _lib.ptr(saved["pos"]), _lib.ptr(t_y), _lib.ptr(t_s), _lib.ptr(t_g),
                                              _lib.ptr(ro), _lib.ptr(rd), _lib.ptr(out["z_vals"]), _lib.ptr(t_sc), R, S,
                                              ctypes.byref(mo), _lib.stream_ptr())
    assert rc == 0
    g = lambda t: t.cpu().numpy().astype(np.float64)          # noqa: E731
    X = g(saved["mlp_in"]).reshape(n, MLP_IN_PAD)
    mw = w["mlp"].half().double().numpy()
    W1, W2, W3 = mw[:64 * 80].reshape(64, 80), mw[64 * 80:64 * 80 + 4096].reshape(64, 64), mw[64 * 80 + 4096:].reshape(16, 64)
    kH1, kH2, kdY, kdH2, kdH1 = g(H1), g(H2), g(dY8), g(dH2), g(dH1)
    # layer by layer, each from the kernel's own fp16 input to it: y = fl16(op(a @ b)) accumulated in fp32 over K terms
    acc = lambda a, b, K: K * EPS32 * (np.abs(a) @ np.abs(b))  # noqa: E731
    assert np.all(_near16(kH1, np.maximum(X @ W1.T, 0), acc(X, W1.T, 80)))
    assert np.all(_near16(kH2, np.maximum(kH1 @ W2.T, 0), acc(kH1, W2.T, 64)))
    want_dy = np.zeros((n, 8))
    want_dy[:, :3] = _f16(d_y.astype(np.float32) * np.float32(sc))          # one rounding of an exact product
    assert np.array_equal(kdY, want_dy)
    assert np.all(_near16(kdH2, (kdY[:, :3] @ W3[:3]) * (kH2 > 0), acc(kdY[:, :3], np.abs(W3[:3]), 3)))
    assert np.all(_near16(kdH1, (kdH2 @ W2) * (kH1 > 0), acc(kdH2, W2, 64)))
    dX = kdH1 @ W1                                            # [n, 80], the kernel rounds it to fp16 once
    aX = acc(kdH1, W1, 64)
    kd_out = g(d_out)
    assert np.array_equal(kd_out[:, 0], _f16(d_s * np.float32(sc)))
    assert np.all(_near16(kd_out[:, 1:], dX[:, 36:67], aX[:, 36:67]))
    # embedding: fl16(fl16(dX) cos(arg)), arg = p . B[:, j] in fp32 (|arg| up to ~200: a few 1e-5 absolute through the
    # reduction by 2 pi), so the bound adds |dX| 1e-4 to the fp16 terms
    zm = out["z_vals"].cpu().numpy().reshape(-1).astype(np.float32)
    pt = (np.repeat(rays[0].numpy(), S, 0) + np.repeat(rays[1].numpy(), S, 0) * zm[:, None]).astype(np.float32)
    arg = pt.astype(np.float64) @ w["color_B"].double().numpy()
    want_e = dX[:, :33] * np.cos(arg)
    be = _ulp16(np.abs(want_e)) + _ulp16(np.abs(dX[:, :33]) + aX[:, :33]) + aX[:, :33] + np.abs(dX[:, :33]) * 1e-4
    assert np.all(np.abs(g(dE)[:, :33] - want_e) <= be)
    assert not np.any(g(dE)[:, 33:])
    # normal: d_grad + fl16(dX[33:36]) / scale in fp32
    want_gt = d_g + dX[:, 33:36] / sc
    bgt = (_ulp16(np.abs(dX[:, 33:36]) + aX[:, 33:36]) + aX[:, 33:36]) / sc + 2 * EPS32 * np.abs(want_gt)
    assert np.all(np.abs(g(d_gt) - want_gt) <= bgt)
    # the sdf_layer input row and the position split: exact
    want_h = np.zeros((n, 40))
    want_h[:, :3] = _f16(g(saved["pos"]).reshape(n, 3))
    want_h[:, 3:35] = g(saved["enc"]).reshape(n, 32)
    want_h[:, 35] = 1.0
    assert np.array_equal(g(h), want_h)
    hi = pt.astype(np.float16)
    lo = (pt - hi.astype(np.float32)).astype(np.float16)
    want_pl = np.zeros((n, 8))
    want_pl[:, :3], want_pl[:, 3:6] = hi, lo
    assert np.array_equal(g(pts_hl), want_pl)
