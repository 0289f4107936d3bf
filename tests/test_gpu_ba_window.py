"""Bundle adjustment at local-window sizes, against the fp64 oracle (oracle/ba_oracle.py).

`goslam_ba` picks its solve by pose count P = t1 - t0: P <= 16 runs every iteration inside the cooperative
`ba_persistent_kernel` (solve_small), 17 <= P <= 99 `ba_solve_cluster_kernel`, P >= 100 `ba_solve_kernel`;
the split form (`goslam_ba_phase1/2`) runs `ba_solve_warp_kernel` for P <= 16.  The frontend's local window
(25 keyframes, up to 75 edges) lives in P = 8..20.  This file checks
  A. every solve kernel on crafted reduced systems, at a bound an fp64 Cholesky has to meet;
  B. the device's reduced camera system against the oracle's, block pattern and values;
  C. `goslam_ba` end to end on frontend-like windows, the split form against it, and a failed factorisation
     inside the cooperative kernel;
  D. a second call after the cached workspace was used at another size, and CUDA-graph replay.
The scene generators and their CPU checks are in test_ba_window_cases.py.  Lines starting with [ba-window] report
the measured worst errors next to their bounds (pytest -s)."""
import numpy as np
import pytest
import torch

from oracle import ba_oracle, geom_oracle
from test_ba_window_cases import (EXPECTED_KERNEL, KAPPAS, PATTERNS, SOLVE_P, WINDOW_CASES, block_nonzero,
                                  crafted_rhs, crafted_system, expected_blocks, solve_kernel, window_case)

pytestmark = pytest.mark.gpu

LM_EP = [(1e-4, 0.1), (1e-5, 1e-2)]
WIN_LM, WIN_EP = 1e-4, 0.1                 # the frontend's local BA (src/factor_graph.py update)
MAX_ITERS = 5

# Reduced camera system, device against the fp64 oracle.  Every entry is a sum of per-pixel products computed in
# fp32 (~20 dependent roundings: projection, 1/Z, Jacobian, weight), summed in fp32 over at most ~40 terms per
# thread / warp tree before the fp64 accumulation, and the oracle rounds each edge's block to fp32.  Relative to
# the sum of |terms| that is <= ~64 * 2^-24 ~ 4e-6; by Cauchy-Schwarz the sum of |terms| of H_ab is at most
# sqrt(A_aa A_bb) with A the pose-block Hessian, and the Schur complement cancels part of A's diagonal, so
# tau_H = 2^-24 * 2^10 on sqrt(|H_aa| |H_bb|) of the REDUCED H (measured on an H100: <= 6e-8 motion-only).
# b sums residual-weighted terms of random sign (sum of |terms| >> |b|), hence the looser tau_b on max|b|.
TAU_H = 2.0 ** -14
TAU_B = 2.0 ** -10
# split form against the fused kernel: same arithmetic per pixel, only the reduction trees differ
# (system_items<256> against <128>): fp32 sums in a different order, nothing else
SPLIT_TOL = 1e-5


def dev():
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)


def _report(*args):
    print("[ba-window]", *args)


_cache = {}


# ------------------------------------------------------------------------------------------ A. solve kernels
def _solver_backend(P):
    """CudaBackend whose graph tables come from a one-edge motion-only phase 1 with this (t0, t1)."""
    if P not in _cache:
        from goslam_b200 import parallel, synthetic
        t0, t1, ht, wd = 1, 1 + P, 4, 8
        num = t1 + 2
        poses = torch.zeros(num, 7)
        poses[:, 6] = 1.0
        poses[:t1] = synthetic.make_poses(t1, torch.Generator().manual_seed(5))
        disps = torch.ones(num, ht, wd, device=dev())
        be = parallel.CudaBackend(poses.to(dev()), disps, torch.tensor([3.6, 3.6, 4.0, 2.0], device=dev()),
                                  torch.zeros_like(disps), t0, t1)
        ii = torch.tensor([t0], dtype=torch.int64, device=dev())
        jj = torch.tensor([t0 + 1 if P > 1 else t0 - 1], dtype=torch.int64, device=dev())
        z = torch.zeros(1, 2, ht, wd, device=dev())
        be.phase1(z, z, torch.zeros(num, ht, wd, device=dev()), ii, jj, True)
        _cache[P] = (be, poses)
    return _cache[P]


def _phase2(P, H, b, lm, ep):
    be, poses0 = _solver_backend(P)
    be.poses.copy_(poses0.to(dev()))
    system = torch.from_numpy(np.concatenate([H.ravel(), b])).to(dev())
    dx, st = be.phase2(system, lm, ep, True, 0, be.num, return_status=True)
    return dx.cpu().numpy(), int(st.item()), be.poses.cpu(), poses0, be.t0, be.t1


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("P", SOLVE_P)
def test_solve_kernels_on_crafted_systems(P, pattern):
    n = 6 * P
    worst, worst_pose = 0.0, 0.0
    for kappa in KAPPAS:
        H, _ = crafted_system(P, pattern, kappa)
        for lm, ep in LM_EP:
            b, Hd = crafted_rhs(H, lm, ep)
            ref, rst = ba_oracle.solve(H, b, H, lm, ep)
            assert rst == 0
            dx, st, poses, poses0, t0, t1 = _phase2(P, H, b, lm, ep)
            assert st == 0, (kappa, lm)
            # one fp32 rounding of the fp64 solution on each side, plus the backward error of an fp64 Cholesky
            # (both sides factor in fp64, in different orders)
            k = np.linalg.cond(Hd)
            bound = (2.0 ** -22 + 16 * n * k * 2.0 ** -53) * np.abs(ref).max()
            err = np.abs(dx.reshape(P, 6) - ref).max()
            worst = max(worst, err / bound)
            assert err <= bound, (kappa, lm, k, err, bound)
            # both sides retract in fp32 with different sinf/cosf; the pose entries are O(1), so a few ulps of 1
            tn, qn = geom_oracle.retr_se3(ref, poses0[t0:t1, :3].numpy(), poses0[t0:t1, 3:].numpy())
            perr = np.abs(poses[t0:t1].numpy() - np.concatenate([tn, qn], 1)).max()
            worst_pose = max(worst_pose, perr)
            assert perr <= 4e-6, (kappa, lm, perr)
            assert torch.equal(poses[:t0], poses0[:t0]) and torch.equal(poses[t1:], poses0[t1:])
    _report("A P=%d %s kernel=%s dx err/bound %.3g pose err %.3g (bound 4e-6)" % (
        P, pattern, solve_kernel(P), worst, worst_pose))


FAILURES = ["indefinite_first", "indefinite_mid", "indefinite_last", "nan_b", "nan_lower"]


@pytest.mark.parametrize("kind", FAILURES)
@pytest.mark.parametrize("P", [7, 16, 17, 99, 100])
def test_solve_kernels_report_a_failed_factorisation(P, kind):
    """status 1, dx exactly 0 and the poses untouched, in every solve kernel."""
    n = 6 * P
    lm, ep = 1e-4, 0.1
    H, _ = crafted_system(P, "banded", 1e4)
    b, Hd = crafted_rhs(H, lm, ep)
    if kind.startswith("indefinite"):
        col = {"first": 0, "mid": P // 2, "last": P - 1}[kind.split("_")[1]]
        j = 6 * col + 3
        H[j, j] = -max(1.0, abs(H[j, j]))
        np.linalg.cholesky(Hd[:j, :j])                 # so the factorisation fails exactly at column j
    elif kind == "nan_b":
        b[n // 2] = np.nan
    else:
        H[n - 1, 0] = np.nan                           # lower triangle only: the upper one is never read
    assert ba_oracle.solve(H, b, H, lm, ep)[1] == 1
    dx, st, poses, poses0, _, _ = _phase2(P, H, b, lm, ep)
    assert st == 1
    assert np.all(dx == 0.0)
    assert torch.equal(poses, poses0)


# ------------------------------------------------------------------------------------------ window scenes
def _case(name):
    if ("case", name) not in _cache:
        _cache[("case", name)] = window_case(name)
    return _cache[("case", name)]


def _dev_inputs(name):
    """device copies of the constant inputs, made once (a CUDA graph capture cannot contain the copies)"""
    if ("dev", name) not in _cache:
        sc, tg, wg, eta = _case(name)
        _cache[("dev", name)] = dict(
            intr=sc["intrinsics"][0].to(dev()).contiguous(), sens=sc["disps_sens"].to(dev()), tg=tg.to(dev()),
            wg=wg.to(dev()), eta=eta.to(dev()), ii=sc["ii"].to(dev()), jj=sc["jj"].to(dev()))
    return _cache[("dev", name)]


def _eta_by_frame(name):
    sc, _, _, eta = _case(name)
    num, ht, wd = sc["disps"].shape
    kx = torch.unique(torch.cat([torch.arange(sc["t0"], sc["t1"]), sc["ii"]]))
    e = torch.zeros(num, ht, wd)
    e[kx] = eta
    return e


def _oracle_trace(name, motion_only):
    """ba_oracle.ba in fp64, keeping the state after each of the first MAX_ITERS iterations."""
    key = ("trace", name, motion_only)
    if key not in _cache:
        sc, tg, wg, eta = _case(name)
        t0, t1 = sc["t0"], sc["t1"]
        poses = np.array(sc["poses"].numpy(), np.float32, copy=True)
        disps = np.array(sc["disps"].numpy(), np.float32, copy=True)
        status, out = [], {}
        for it in range(1, MAX_ITERS + 1):
            st = ba_oracle.phase1(poses, disps, sc["intrinsics"][0].numpy(), sc["disps_sens"].numpy(), tg.numpy(),
                                  wg.numpy(), eta.numpy(), sc["ii"].numpy(), sc["jj"].numpy(), t0, t1, motion_only,
                                  np.float64)
            dx, fail = ba_oracle.solve(st["Hred"], st["bred"], st["A"], WIN_LM, WIN_EP)
            status.append(fail)
            dz = ba_oracle.phase2(st, dx, poses, disps, t0, t1, motion_only)
            out[it] = dict(p=poses.copy(), d=disps.copy(), dx=dx, dz=dz, status=list(status), H=st["Hred"],
                           b=st["bred"], A=st["A"])
        _cache[key] = out
    return _cache[key]


def _fused(name, motion_only, iters):
    key = ("fused", name, motion_only, iters)
    if key not in _cache:
        from goslam_b200 import droid_backends
        sc = _case(name)[0]
        a = _dev_inputs(name)
        poses, disps = sc["poses"].clone().to(dev()), sc["disps"].clone().to(dev())
        dx, dz, status = droid_backends.ba(poses, disps, a["intr"], a["sens"], a["tg"], a["wg"], a["eta"], a["ii"],
                                           a["jj"], sc["t0"], sc["t1"], iters, WIN_LM, WIN_EP, motion_only,
                                           return_status=True)
        _cache[key] = dict(p=poses.cpu(), d=disps.cpu(), dx=dx.cpu(), dz=None if dz is None else dz.cpu(),
                           status=status.cpu().tolist())
    return _cache[key]


# ------------------------------------------------------------------------------------------ B. reduced system
@pytest.mark.parametrize("motion_only", [False, True])
@pytest.mark.parametrize("name", list(WINDOW_CASES))
def test_reduced_system_vs_oracle(name, motion_only):
    from goslam_b200 import parallel
    sc, _, _, _ = _case(name)
    t0, t1 = sc["t0"], sc["t1"]
    P, n = t1 - t0, 6 * (t1 - t0)
    a = _dev_inputs(name)
    be = parallel.CudaBackend(sc["poses"].clone().to(dev()), sc["disps"].clone().to(dev()), a["intr"], a["sens"],
                              t0, t1)
    sysd = be.phase1(a["tg"], a["wg"], _eta_by_frame(name).to(dev()), a["ii"], a["jj"], motion_only).cpu().numpy()
    Hd, bd = sysd[:n * n].reshape(n, n), sysd[n * n:]
    ref = _oracle_trace(name, motion_only)[1]
    H, b = ref["H"], ref["b"]
    # Schur pair tables (entry_code / pair_ptr): exactly the same structural zeros
    want = expected_blocks(sc["ii"].numpy(), sc["jj"].numpy(), t0, t1, motion_only)
    assert np.array_equal(block_nonzero(H, P), want)
    assert np.array_equal(block_nonzero(Hd, P), want)
    dg = np.sqrt(np.abs(np.diag(H)))
    scale = dg[:, None] * dg[None, :]
    # blocks (a, b) and (b, a), a != b, receive the same fp64 addends, possibly in another order; inside a diagonal
    # block, entries (r, c) and (c, r) are different fp32 pixel sums (sum E_r Q E_c against sum E_c Q E_r)
    asym = np.abs(Hd - Hd.T) / scale
    diag_blk = np.kron(np.eye(P, dtype=bool), np.ones((6, 6), bool))
    sym = asym[~diag_blk].max() if P > 1 else 0.0
    assert sym <= 1e-12, sym
    assert asym[diag_blk].max() <= TAU_H
    eh = (np.abs(Hd - H) / scale).max()
    eb = np.abs(bd - b).max() / np.abs(b).max()
    _report("B %s motion_only=%d |dH|/sqrt(HaaHbb) %.3g (tau %.3g) |db|/max|b| %.3g (tau %.3g) asym %.3g" % (
        name, motion_only, eh, TAU_H, eb, TAU_B, sym))
    assert eh <= TAU_H
    assert eb <= TAU_B


# ------------------------------------------------------------------------------------------ C. end to end
def _dx_bound(ref):
    """First-order perturbation bound on the step when the reduced system is known to TAU_H / TAU_B (as in B):
    H_d dx = b with H -> H + D E D (|E_ab| <= TAU_H, D = diag sqrt|H_aa|) and |db| <= TAU_B max|b| gives
    |d dx|_2 <= |H_d^-1 D|_2 n TAU_H |D dx|_2 + |H_d^-1|_2 sqrt(n) TAU_B max|b|, plus one fp32 rounding."""
    H, b = ref["H"], ref["b"]
    n = H.shape[0]
    Hd = H.copy()
    Hd[np.diag_indices(n)] += np.float64(np.float32(WIN_EP)) + np.float64(np.float32(WIN_LM)) * np.diag(H)
    x = np.linalg.solve(Hd, b)
    D = np.sqrt(np.abs(np.diag(H)))
    Hinv = np.linalg.inv(Hd)
    return (np.linalg.norm(Hinv * D[None, :], 2) * n * TAU_H * np.linalg.norm(D * x)
            + np.linalg.norm(Hinv, 2) * np.sqrt(n) * TAU_B * np.abs(b).max() + 2.0 ** -23 * np.abs(x).max())


@pytest.mark.parametrize("iters", [1, 2, 5])
@pytest.mark.parametrize("motion_only", [False, True])
@pytest.mark.parametrize("name", list(WINDOW_CASES))
def test_window_ba_vs_oracle(name, motion_only, iters):
    sc, _, _, _ = _case(name)
    t0, t1 = sc["t0"], sc["t1"]
    assert solve_kernel(t1 - t0) == EXPECTED_KERNEL[name]
    got = _fused(name, motion_only, iters)
    ref = _oracle_trace(name, motion_only)[iters]
    assert got["status"] == ref["status"] == [0] * iters
    assert _rel(got["p"], ref["p"]) < 1e-4                      # 1e-4 relative on the state, as everywhere
    # after 5 iterations a motion-only window has converged: the step is ~1e-7 of O(1) poses, i.e. fp32 noise of
    # the state, so the relative check gets an absolute floor of ~16 ulps of 1
    assert np.abs(got["dx"].numpy() - ref["dx"]).max() < 5e-3 * np.abs(ref["dx"]).max() + 1e-6
    if not motion_only:
        assert _rel(got["d"], ref["d"]) < 1e-4
        assert np.abs(got["dz"].numpy() - ref["dz"]).max() < 1e-4 * max(np.abs(ref["d"]).max(), 1.0)
    else:
        assert torch.equal(got["d"], sc["disps"]) and got["dz"] is None
    assert torch.equal(got["p"][:t0], sc["poses"][:t0]) and torch.equal(got["p"][t1:], sc["poses"][t1:])
    if iters == 1:
        err = np.abs(got["dx"].numpy() - ref["dx"]).max()
        bound = _dx_bound(ref)
        _report("C %s motion_only=%d dx err %.3g bound %.3g (max|dx| %.3g) pose rel %.3g" % (
            name, motion_only, err, bound, np.abs(ref["dx"]).max(), _rel(got["p"], ref["p"])))
        assert err <= bound


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("motion_only", [False, True])
@pytest.mark.parametrize("name", list(WINDOW_CASES))
def test_window_split_form_matches_the_fused_kernel(name, motion_only, world):
    """goslam_ba_phase1/2 (for P <= 16 the solve is ba_solve_warp_kernel) with `world` emulated ranks, as in
    test_gpu_ba_large.test_ba_split_form_vs_oracle, against goslam_ba on the same inputs."""
    from goslam_b200 import parallel
    iters = 2
    sc, _, _, _ = _case(name)
    t0, t1 = sc["t0"], sc["t1"]
    num = sc["disps"].shape[0]
    D = _dev_inputs(name)
    eta_f = _eta_by_frame(name).to(dev())
    bounds = parallel.shard_frames_by_edges(sc["ii"], num, world)
    ranks = []
    for lo, hi in bounds:
        p, d = sc["poses"].clone().to(dev()), sc["disps"].clone().to(dev())
        sel = parallel.local_edges(D["ii"], lo, hi)
        ranks.append(dict(be=parallel.CudaBackend(p, d, D["intr"], D["sens"], t0, t1), p=p, d=d, lo=lo, hi=hi,
                          tg=D["tg"][sel].contiguous(), wg=D["wg"][sel].contiguous(),
                          ii=D["ii"][sel].contiguous(), jj=D["jj"][sel].contiguous()))
    for _ in range(iters):
        total = None
        for r in ranks:
            s = r["be"].phase1(r["tg"], r["wg"], eta_f, r["ii"], r["jj"], motion_only)
            total = s if total is None else total + s
        for r in ranks:
            r["dx"], st = r["be"].phase2(total, WIN_LM, WIN_EP, motion_only, r["lo"], r["hi"], return_status=True)
            assert int(st.item()) == 0
        if not motion_only:
            merged = torch.cat([r["d"][r["lo"]:r["hi"]] for r in ranks])
            for r in ranks:
                r["d"].copy_(merged)
    fused = _fused(name, motion_only, iters)
    ep_, ed_, edx = _rel(ranks[0]["p"].cpu(), fused["p"]), _rel(ranks[0]["d"].cpu(), fused["d"]), \
        _rel(ranks[0]["dx"].cpu(), fused["dx"])
    _report("C split %s motion_only=%d world=%d rel poses %.3g disps %.3g dx %.3g (tol %.3g, dx %.3g)" % (
        name, motion_only, world, ep_, ed_, edx, SPLIT_TOL, 100 * SPLIT_TOL))
    for r in ranks:
        assert torch.equal(r["p"], ranks[0]["p"])
    assert ep_ <= SPLIT_TOL and ed_ <= SPLIT_TOL
    assert edx <= 100 * SPLIT_TOL                        # the step is ~1e-2 of the state


def test_window_failed_factorisation_inside_the_cooperative_kernel():
    """Weights of the edges into one pose scaled by -1e6 make the reduced system indefinite: every iteration
    reports status 1 and takes dx = 0, the poses stay bit-identical, and the depths still take the
    back-substitution with dx = 0 (dz = Q w), as the reference does."""
    from goslam_b200 import droid_backends
    name, iters = "P16", 2
    sc, tg, wg, eta = _case(name)
    t0, t1 = sc["t0"], sc["t1"]
    wbad = wg.clone()
    wbad[sc["jj"] == t0 + 8] *= -1e6
    a = _dev_inputs(name)
    poses, disps = sc["poses"].clone().to(dev()), sc["disps"].clone().to(dev())
    dx, dz, status = droid_backends.ba(poses, disps, a["intr"], a["sens"], a["tg"], wbad.to(dev()), a["eta"],
                                       a["ii"], a["jj"], t0, t1, iters, WIN_LM, WIN_EP, False, return_status=True)
    rp, rd, rdx, rdz, rst = ba_oracle.ba(
        sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy(), sc["disps_sens"].numpy(), tg.numpy(),
        wbad.numpy(), eta.numpy(), sc["ii"].numpy(), sc["jj"].numpy(), t0, t1, iters, WIN_LM, WIN_EP, False,
        dtype=np.float64)
    assert status.cpu().tolist() == rst.tolist() == [1] * iters
    assert float(dx.abs().max()) == 0.0
    assert torch.equal(poses.cpu(), sc["poses"])
    d = disps.cpu().numpy()
    assert not np.array_equal(d, sc["disps"].numpy())
    # negative weights can drive the depth term C towards 0 (Q = 1/C): compare where the oracle is finite
    fin = np.isfinite(rd)
    assert np.array_equal(np.isfinite(d), fin)
    err = (np.abs(d[fin] - rd[fin]) / np.maximum(np.abs(rd[fin]), 1.0)).max()
    _report("C failure P16 disps rel err %.3g (tol 1e-4), finite %d/%d" % (err, fin.sum(), fin.size))
    assert err < 1e-4


# ------------------------------------------------------------------------------------------ D. reuse, graphs
def _ba_call(name, poses, disps, iters=2, motion_only=False):
    from goslam_b200 import droid_backends
    sc = _case(name)[0]
    a = _dev_inputs(name)
    return droid_backends.ba(poses, disps, a["intr"], a["sens"], a["tg"], a["wg"], a["eta"], a["ii"], a["jj"],
                             sc["t0"], sc["t1"], iters, WIN_LM, WIN_EP, motion_only, return_status=True)


def test_cached_workspace_reuse_at_another_size_gives_the_same_result():
    """The cooperative kernel's barrier / arrival / solved counters live in the grow-only workspace, at an offset
    that depends on the frame count: a call with another `num` leaves its values where the next call's
    counters are.  ba_prep_kernel must reset them."""
    sc = _case("P12")[0]
    other = _case("P16")[0]
    assert other["disps"].shape[0] != sc["disps"].shape[0]
    outs = []
    for k in range(2):
        p, d = sc["poses"].clone().to(dev()), sc["disps"].clone().to(dev())
        dx, _, st = _ba_call("P12", p, d)
        outs.append((p.cpu(), d.cpu(), dx.cpu(), st.cpu().tolist()))
        if k == 0:
            _ba_call("P16", other["poses"].clone().to(dev()), other["disps"].clone().to(dev()), iters=3)
    (p1, d1, x1, s1), (p2, d2, x2, s2) = outs
    assert s1 == s2 == [0, 0]
    assert _rel(p2, p1) <= 1e-6 and _rel(d2, d1) <= 1e-6 and _rel(x2, x1) <= 1e-6     # fp64 atomics may reorder


def test_cuda_graph_replay_matches_eager():
    """The update step is replayed as a CUDA graph (bench.py): table kernel + cooperative kernel, replayed from
    restored inputs, must give the eager result each time."""
    sc = _case("P12")[0]
    p0, d0 = sc["poses"].to(dev()), sc["disps"].to(dev())
    p, d = p0.clone(), d0.clone()
    ex, _, est = _ba_call("P12", p, d)
    eager = (p.cpu(), d.cpu(), ex.cpu())
    assert est.cpu().tolist() == [0, 0]
    sp, sd = p0.clone(), d0.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _ba_call("P12", sp, sd)                          # warm-up off the capture: workspaces, attributes
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    try:
        with torch.cuda.graph(g):
            gx, _, gst = _ba_call("P12", sp, sd)
    except Exception as e:  # noqa: BLE001
        pytest.skip("CUDA graph capture of the BA call failed: %s: %s" % (type(e).__name__, e))
    for _ in range(2):
        sp.copy_(p0)
        sd.copy_(d0)
        g.replay()
        torch.cuda.synchronize()
        assert gst.cpu().tolist() == [0, 0]
        assert _rel(sp.cpu(), eager[0]) <= 1e-6 and _rel(sd.cpu(), eager[1]) <= 1e-6
        assert _rel(gx.cpu(), eager[2]) <= 1e-6
