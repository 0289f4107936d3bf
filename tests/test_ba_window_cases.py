"""Generators for the local-window bundle-adjustment tests (tests/test_gpu_ba_window.py), and CPU checks that
they produce what those tests claim: the pose count P of each case and the solve kernel it selects, the
frontend's edge budget, fixed source frames before t0, more than 32 depth slots where the binary-search
branch of the Schur pair lookup is wanted, crafted matrices at their target condition numbers, and the
zero-block pattern of the fp64 oracle's reduced camera system.

Local BA in the reference configs runs a window of 25 keyframes with up to 75 edges (mono: 50 / 100), so
P = t1 - t0 from 8 to ~20 is the frontend's normal range."""
import numpy as np
import torch

from oracle import ba_oracle, geom_oracle

# Solve-path thresholds of goslam_ba / goslam_ba_phase2 (go-slam_b200/csrc/ba.cu):
WARP_SOLVE_MAX_N = 96     # kWarpSolveMaxN: 6P <= 96 -> cooperative kernel / ba_solve_warp_kernel (solve_small)
CLUSTER_MAX_P = 99        # cl_smem_bytes(P) <= kClusterSmemMax up to P = 99 -> ba_solve_cluster_kernel
MAX_FACTORS = 75          # frontend edge budget of the reference configs (max_factors: 75)


def solve_kernel(P):
    if 6 * P <= WARP_SOLVE_MAX_N:
        return "small"        # solve_small: inside ba_persistent_kernel, or ba_solve_warp_kernel in the split form
    if P <= CLUSTER_MAX_P:
        return "cluster"
    return "global"


# ------------------------------------------------------------------------------------------ window cases
# radius: neighbourhood edges |i - j| <= radius inside [t0, t1); old: source frames before t0 (fixed poses,
# variable depths) with `per_old` edges each into the window; stereo: offsets in the window of stereo self-edges.
WINDOW_CASES = {
    "P8": dict(P=8, ht=40, wd=80, radius=3),
    "P12": dict(P=12, ht=40, wd=80, radius=3),
    "P16": dict(P=16, ht=40, wd=80, radius=2),              # radius 3 would give 84 > 75 edges
    "P16_60x80": dict(P=16, ht=60, wd=80, radius=2),        # hw = 4800: ragged last 128-pixel tile
    "P12_9x13": dict(P=12, ht=9, wd=13, radius=3),          # hw = 117: not a multiple of 32
    "P11_stereo": dict(P=11, ht=24, wd=32, radius=3, stereo=(1, 6), rgbd=False),
    "P12_M52": dict(P=12, ht=24, wd=32, radius=1, t0=40, old=40, per_old=1),   # 52 depth slots
    "P17": dict(P=17, ht=24, wd=32, radius=2),              # first cluster size
}
EXPECTED_KERNEL = {name: ("cluster" if name == "P17" else "small") for name in WINDOW_CASES}


def window_edges(P, t0, radius, old=3, per_old=2, stereo=()):
    """Frontend-like local window: neighbourhood edges inside [t0, t1), edges from the `old` frames before t0
    into the window (and one back out of it, to a fixed pose), and a few long-range edges."""
    t1 = t0 + P
    ii, jj = [], []
    for i in range(t0, t1):
        for j in range(t0, t1):
            if 0 < abs(i - j) <= radius:
                ii.append(i)
                jj.append(j)
    for s in range(t0 - old, t0):
        for m in range(per_old):
            ii.append(s)
            jj.append(t0 + (s + m) % min(P, 3) if per_old > 1 else t0 + s % P)
    ii.append(t0)
    jj.append(t0 - 1)                                   # target pose fixed: only the source's pose blocks
    for a, b in ((t0, t1 - 1), (t1 - 1, t0), (t0 + 1, t1 - 2)):
        if abs(a - b) > radius:
            ii.append(a)
            jj.append(b)
    for s in stereo:
        ii.append(t0 + s)
        jj.append(t0 + s)
    return torch.tensor(ii, dtype=torch.int64), torch.tensor(jj, dtype=torch.int64)


def window_case(name, seed=43):
    """Returns (scene, targets, weights, eta) with scene["ii"], ["jj"], ["t0"], ["t1"] set; deterministic."""
    from goslam_b200 import synthetic
    c = WINDOW_CASES[name]
    P, ht, wd = c["P"], c["ht"], c["wd"]
    t0 = c.get("t0", 4)
    t1 = t0 + P
    sc, g = synthetic.make_scene(num_kf=t1, ht=ht, wd=wd, rgbd=c.get("rgbd", True), seed=seed, with_fmaps=False,
                                 buffer=t1 + 2)
    ii, jj = window_edges(P, t0, c["radius"], c.get("old", 3), c.get("per_old", 2), c.get("stereo", ()))
    sc.update(ii=ii, jj=jj, t0=t0, t1=t1)
    coords, _ = geom_oracle.reproject(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"].numpy(),
                                      ii.numpy(), jj.numpy())
    targets, weights, eta = synthetic.make_update(sc, torch.from_numpy(coords[0]), g, noise=0.7)
    sc["poses"][t0:t1, :3] += 0.01 * torch.randn(P, 3, generator=g)
    sc["disps"][:t1] *= 1 + 0.03 * torch.randn(t1, ht, wd, generator=g)
    return sc, targets, weights, eta


def depth_slots(ii, t0, t1):
    return np.unique(np.concatenate([np.arange(t0, t1), np.asarray(ii)]))


def expected_blocks(ii, jj, t0, t1, motion_only):
    """[P, P] bool: which 6x6 blocks of the reduced camera system are structurally non-zero.  Pose blocks of
    every edge with an optimised end; Schur blocks between every two entries of a depth slot (its own pose if
    optimised, and the target pose of each of its outgoing edges that is optimised)."""
    P = t1 - t0
    nz = np.zeros((P, P), bool)
    ii, jj = np.asarray(ii), np.asarray(jj)
    for i, j in zip(ii, jj):
        a, b = i - t0, j - t0
        if 0 <= a < P:
            nz[a, a] = True
        if 0 <= b < P:
            nz[b, b] = True
        if 0 <= a < P and 0 <= b < P:
            nz[a, b] = nz[b, a] = True
    if not motion_only:
        for f in depth_slots(ii, t0, t1):
            ent = ([f - t0] if t0 <= f < t1 else []) + [j - t0 for i, j in zip(ii, jj) if i == f and t0 <= j < t1]
            for a in ent:
                for b in ent:
                    nz[a, b] = True
    return nz


def block_nonzero(H, P):
    return np.abs(H.reshape(P, 6, P, 6)).max(axis=(1, 3)) != 0


# ------------------------------------------------------------------------------------------ crafted systems
SOLVE_P = [1, 2, 7, 8, 15, 16, 17, 18, 23, 24, 25, 33, 99, 100]
PATTERNS = ["banded", "dense", "zero_blocks"]
KAPPAS = [1e1, 1e4, 1e7]


def block_pattern(P, pattern, rng):
    idx = np.arange(P)
    if pattern == "dense":
        return np.ones((P, P), bool)
    if pattern == "banded":                             # a local window (radius 3) plus a few long-range blocks
        m = np.abs(idx[:, None] - idx[None, :]) <= 3
        for _ in range(max(1, P // 8)):
            a, b = rng.integers(0, P, 2)
            m[a, b] = m[b, a] = True
        return m
    # blocks that are exactly zero: ~20 % of the off-diagonal blocks present, and pose P//2 coupled to nothing
    m = rng.random((P, P)) < 0.2
    m = m | m.T
    m[P // 2, :] = m[:, P // 2] = False
    m[idx, idx] = True
    return m


def crafted_system(P, pattern, kappa, seed=0):
    """Symmetric positive definite H [6P, 6P] with the block pattern and eigenvalues in [1, kappa] (exactly
    those ends).  Dense: a geometric spectrum Q diag(lam) Q^T.  Sparse patterns: a random symmetric matrix on the
    pattern, its spectrum shifted and scaled onto [1, kappa] (that touches only the diagonal, so the pattern is
    kept).  Also returns the block mask."""
    rng = np.random.default_rng(seed * 1000 + P)
    n = 6 * P
    mask = block_pattern(P, pattern, rng)
    if pattern == "dense":
        Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
        lam = np.geomspace(1.0, kappa, n)
        H = (Q * lam) @ Q.T
        H = 0.5 * (H + H.T)
    else:
        R = rng.standard_normal((n, n)) * np.kron(mask, np.ones((6, 6)))
        S = 0.5 * (R + R.T)
        lo, hi = np.linalg.eigvalsh(S)[[0, -1]]
        H = (kappa - 1.0) / (hi - lo) * (S - lo * np.eye(n)) + np.eye(n)
    return H, mask


def crafted_rhs(H, lm, ep, seed=0):
    """b = H_damped x with x ~ 0.02 N(0, 1): steps of the size a BA iteration takes."""
    n = H.shape[0]
    rng = np.random.default_rng(seed + 7)
    Hd = H.copy()
    Hd[np.diag_indices(n)] += np.float64(np.float32(ep)) + np.float64(np.float32(lm)) * np.diag(H)
    return Hd @ (0.02 * rng.standard_normal(n)), Hd


# ------------------------------------------------------------------------------------------ tests
def test_window_cases_reach_the_intended_solve_paths():
    for name, c in WINDOW_CASES.items():
        sc, _, _, _ = window_case(name)
        P = sc["t1"] - sc["t0"]
        assert P == c["P"], name
        assert solve_kernel(P) == EXPECTED_KERNEL[name], name
        assert sc["ii"].numel() <= MAX_FACTORS, (name, sc["ii"].numel())
        assert sc["t1"] + 2 == sc["poses"].shape[0]      # frames after the window too: they must stay put
    assert [solve_kernel(P) for P in (16, 17, 99, 100)] == ["small", "cluster", "cluster", "global"]


def test_window_cases_have_fixed_sources_before_t0():
    for name in WINDOW_CASES:
        sc, _, _, _ = window_case(name)
        ii, jj, t0, t1 = sc["ii"].numpy(), sc["jj"].numpy(), sc["t0"], sc["t1"]
        assert t0 >= 4, name
        old = ii < t0
        assert old.sum() >= 3, name                              # inactive-style edges: fixed pose, variable depth
        assert np.all((jj[old] >= t0) & (jj[old] < t1)), name
        assert np.any((ii >= t0) & (jj < t0)), name              # an edge into a fixed pose
        assert np.any(np.abs(ii - jj) > WINDOW_CASES[name]["radius"]), name   # long-range edges
    sc, _, _, _ = window_case("P11_stereo")
    assert int((sc["ii"] == sc["jj"]).sum()) == 2


def test_binary_search_case_has_more_than_32_depth_slots():
    sc, _, _, _ = window_case("P12_M52")
    M = len(depth_slots(sc["ii"].numpy(), sc["t0"], sc["t1"]))
    assert M > 32, M
    for name in ("P8", "P12", "P16"):
        sc, _, _, _ = window_case(name)
        assert len(depth_slots(sc["ii"].numpy(), sc["t0"], sc["t1"])) <= 32      # the ballot branch


def test_crafted_matrices_hit_their_condition_numbers():
    for P in (2, 16, 17):
        for pattern in PATTERNS:
            for kappa in KAPPAS:
                H, mask = crafted_system(P, pattern, kappa)
                assert np.array_equal(H, H.T)
                lam = np.linalg.eigvalsh(H)
                assert lam[0] > 0
                assert 0.5 * kappa <= lam[-1] / lam[0] <= 2.0 * kappa, (P, pattern, kappa, lam[-1] / lam[0])
                assert np.array_equal(block_nonzero(H, P), mask), (P, pattern)
    _, mask = crafted_system(16, "zero_blocks", 1e4)
    assert not mask.all() and mask[8].sum() == 1


def test_oracle_reduced_system_is_symmetric_with_the_graph_zero_pattern():
    sc, tg, wg, eta = window_case("P12_9x13")
    t0, t1 = sc["t0"], sc["t1"]
    P = t1 - t0
    for motion_only in (False, True):
        st = ba_oracle.phase1(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy(),
                              sc["disps_sens"].numpy(), tg.numpy(), wg.numpy(), eta.numpy(), sc["ii"].numpy(),
                              sc["jj"].numpy(), t0, t1, motion_only, dtype=np.float64)
        H = st["Hred"]
        d = np.sqrt(np.abs(np.diag(H)))
        assert np.abs(H - H.T).max() <= 1e-12 * (d[:, None] * d[None, :]).max()
        want = expected_blocks(sc["ii"].numpy(), sc["jj"].numpy(), t0, t1, motion_only)
        assert np.array_equal(block_nonzero(H, P), want), motion_only
        assert not want.all()                                    # there are zero blocks to get right
    # the Schur pairs add blocks the pose blocks alone do not have (two targets of one depth slot)
    assert not np.array_equal(expected_blocks(sc["ii"].numpy(), sc["jj"].numpy(), t0, t1, False),
                              expected_blocks(sc["ii"].numpy(), sc["jj"].numpy(), t0, t1, True))
