"""CPU tests of the host-side mirror of the reference interface (no kernels are launched)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import geom_oracle


def test_install_registers_reference_module_names():
    import goslam_b200
    saved = {k: sys.modules.get(k) for k in ("droid_backends", "lietorch")}
    try:
        db, lt = goslam_b200.install()
        import droid_backends
        import lietorch
        assert droid_backends is db and lietorch is lt
        # the nine functions of src/lib/droid.cpp:237-250
        for fn in ("ba", "frame_distance", "projmap", "depth_filter", "iproj", "altcorr_forward",
                   "altcorr_backward", "corr_index_forward", "corr_index_backward"):
            assert callable(getattr(droid_backends, fn)), fn
        assert hasattr(lietorch, "SE3") and hasattr(lietorch, "Sim3") and hasattr(lietorch, "cat")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_contiguity_and_device_errors_mirror_the_reference():
    from goslam_b200 import droid_backends as db
    vol = torch.zeros(1, 4, 4, 4, 4)
    coords = torch.zeros(1, 2, 4, 4)
    with pytest.raises(RuntimeError, match="must be contiguous"):
        db.corr_index_forward(vol.transpose(1, 2), coords, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        db.corr_index_forward(vol, coords, 3)             # CPU tensors: no fallback
    with pytest.raises(RuntimeError, match="training-only"):
        db.corr_index_backward(vol, coords, vol, 3)
    with pytest.raises(RuntimeError, match="training-only"):
        db.altcorr_backward(vol, vol, coords, vol, 3)
    poses = torch.zeros(4, 7)
    with pytest.raises(RuntimeError, match="CUDA"):
        db.frame_distance(poses, torch.ones(4, 4, 4), torch.ones(4), torch.zeros(2).long(), torch.ones(2).long(), 0.3)


def test_no_cpu_fallback_in_mirror_classes():
    from goslam_b200.modules import CorrBlock
    from goslam_b200 import neus, synthetic
    f = torch.zeros(1, 1, 128, 16, 16).half()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        CorrBlock(f, f)
    net = neus.InstantNeuS(synthetic.NEUS_CFG, [[-1.0, 1.0]] * 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        net(torch.zeros(2, 3), torch.ones(2, 3), torch.ones(2, 8), torch.ones(2, 8))


def test_oracle_only_in_timing_arms_and_bench_baseline():
    import os
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "go-slam_b200")
    for dp, _, fns in os.walk(root):
        for fn in fns:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, fn)).read()
                assert "import oracle" not in src and "from oracle" not in src, os.path.join(dp, fn)
    # among the developer tools, exactly the timing scripts whose comparison arm is the oracle import it; bench.py
    # imports it only inside its CPU-baseline leg
    top = os.path.dirname(root)
    oracle_arms = {"time_encoder.py", "time_graph.py", "time_mapper.py", "time_mesh_eval.py", "time_obb.py",
                   "time_refining_mapper.py", "time_render.py"}
    importers = set()
    for fn in os.listdir(os.path.join(top, "tools")):
        if fn.endswith(".py"):
            src = open(os.path.join(top, "tools", fn)).read()
            if "import oracle" in src or "from oracle" in src:
                importers.add(fn)
    assert importers == oracle_arms, importers ^ oracle_arms
    bench_src = open(os.path.join(top, "bench.py")).read()
    uses = [i for i in range(len(bench_src)) if bench_src.startswith("from oracle", i)]
    start = bench_src.index("def cpu_reference_step")
    end = bench_src.index("\ndef ", start + 10)
    assert uses and all(start < i < end for i in uses)


def _rand_se3(n, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(n, 4, generator=g)
    q = q / q.norm(dim=-1, keepdim=True)
    return torch.cat([torch.randn(n, 3, generator=g), q], dim=-1)


def test_lietorch_shim_group_axioms_and_oracle_agreement():
    from goslam_b200.lietorch import SE3
    A, B = SE3(_rand_se3(5, 0)), SE3(_rand_se3(5, 1))
    I = (A * A.inv()).data
    assert torch.allclose(I[:, :3], torch.zeros(5, 3), atol=1e-5) and torch.allclose(I[:, 3:].abs(), torch.tensor([0, 0, 0, 1.0]).expand(5, 4), atol=1e-5)
    X = torch.randn(5, 4)
    # (A*B)*X == A*(B*X)
    assert torch.allclose((A * B) * X, A * (B * X), atol=1e-5)
    # relative pose == the CUDA twin relSE3 (src/lib/droid_kernels.cu:96-107)
    rel = (B * A.inv()).data.numpy()
    t, q = geom_oracle.rel_se3(A.data[:, :3].numpy(), A.data[:, 3:].numpy(), B.data[:, :3].numpy(), B.data[:, 3:].numpy())
    assert np.allclose(rel[:, :3], t, atol=1e-5) and np.allclose(rel[:, 3:], q, atol=1e-5)
    # act / adjT == actSE3 / adjSE3
    Y = (A * X).numpy()
    assert np.allclose(Y, geom_oracle.act_se3(A.data[:, :3].numpy(), A.data[:, 3:].numpy(), X.numpy()), atol=1e-5)
    J = torch.randn(5, 6)
    assert np.allclose(A.adjT(J).numpy(), geom_oracle.adj_se3(A.data[:, :3].numpy(), A.data[:, 3:].numpy(), J.numpy()), atol=1e-5)
    # matrix() is the homogeneous form of act
    M = A.matrix()
    P = torch.randn(5, 3)
    assert torch.allclose((M[:, :3, :3] @ P[..., None])[..., 0] + M[:, :3, 3], A * P, atol=1e-5)
    # retraction == retrSE3 (left multiplication by exp)
    xi = 0.1 * torch.randn(5, 6)
    r = A.retr(xi).data.numpy()
    t1, q1 = geom_oracle.retr_se3(xi.numpy(), A.data[:, :3].numpy(), A.data[:, 3:].numpy())
    assert np.allclose(r[:, :3], t1, atol=1e-5) and np.allclose(r[:, 3:], q1, atol=1e-5)
    assert np.allclose(SE3.exp(torch.zeros(2, 6)).data.numpy(), [[0, 0, 0, 0, 0, 0, 1]] * 2)


def test_lietorch_shim_log_is_the_inverse_of_exp():
    """ADVICE r01: PoseTrajectoryFiller calls dP.log() (src/trajectory_filler.py:53); exp(log(T)) == T and
    log(exp(xi)) == xi for rotations below pi, through the small-angle branches and for qw < 0."""
    from goslam_b200.lietorch import SE3
    g = torch.Generator().manual_seed(0)
    xi = torch.randn(4000, 6, generator=g, dtype=torch.float64) * torch.tensor([1, 1, 1, .8, .8, .8], dtype=torch.float64)
    xi[:10, 3:] *= 1e-6
    xi[10:20, 3:] *= 1e-3
    xi[20:25, 3:] *= 0.99e-4 / xi[20:25, 3:].norm(dim=-1, keepdim=True)     # either side of the switch-over (exp
    xi[25:30, 3:] *= 1.01e-4 / xi[25:30, 3:].norm(dim=-1, keepdim=True)     # itself jumps by ~theta/2 * |tau| there)
    xi[30, 3:] = 0.0
    xi = xi[xi[:, 3:].norm(dim=-1) < 3.0]
    T = SE3.exp(xi)
    assert (T.log() - xi).abs().max() < 1e-9
    assert (SE3.exp(T.log()).data - T.data).abs().max() < 1e-9
    neg = SE3(torch.cat([T.data[:, :3], -T.data[:, 3:]], dim=-1))           # same rotation, qw < 0
    assert (neg.log() - xi).abs().max() < 1e-9
    # float32: (1 - cos t) / t^2 of the reference's expSE3 cancels completely for t ~ 1e-4 .. 3e-4 (cos t rounds
    # to 1), so exp itself is off by ~t/2 * |tau| there; away from that band the round trip is float-accurate
    xf = xi.float()
    err = (SE3.exp(xf).log() - xf).abs().max(dim=-1)[0]
    band = (xf[:, 3:].norm(dim=-1) > 0.9e-4) & (xf[:, 3:].norm(dim=-1) < 2e-2)
    assert err[~band].max() < 2e-5 and err.max() < 5e-4
    # the interpolation PoseTrajectoryFiller does with it
    P0, P1 = SE3.exp(0.4 * xi[100:150]), SE3.exp(0.4 * xi[150:200])      # relative rotation stays below pi
    v = (P1 * P0.inv()).log()
    assert ((SE3.exp(v) * P0).data - P1.data).abs().max() < 1e-9


def test_lietorch_shim_indexing_like_the_reference_call_sites():
    from goslam_b200.lietorch import SE3, cat
    G = SE3(_rand_se3(6, 2)[None])                 # [1, 6, 7] like DepthVideo.reproject
    jj = torch.tensor([1, 2, 5])
    assert G[:, jj].data.shape == (1, 3, 7)
    assert G[:, :, None, None].data.shape == (1, 6, 1, 1, 7)
    assert cat([G, G], 1).data.shape == (1, 12, 7)
    assert SE3.Identity(1).data.tolist() == [[0, 0, 0, 0, 0, 0, 1]]
    assert G.to(torch.float64).data.dtype == torch.float64


def test_synthetic_graph_matches_reference_neighbourhood_rule():
    from goslam_b200 import synthetic
    ii, jj = synthetic.neighborhood_edges(0, 8, 3)
    assert ii.numel() == 36                              # BASELINE.md §5 config 2
    assert ((ii - jj).abs() <= 3).all() and (ii != jj).all()
    sc, _ = synthetic.make_scene(8, 40, 80, with_fmaps=False)
    sc2, _ = synthetic.make_scene(8, 40, 80, with_fmaps=False)
    assert torch.equal(sc["poses"], sc2["poses"]) and torch.equal(sc["disps"], sc2["disps"])   # deterministic
    assert abs(float(sc["poses"][:, 3:].norm(dim=-1).mean()) - 1.0) < 1e-5


def test_tiled_corr_pool_slot_bookkeeping():
    """CorrPool is host-side bookkeeping only: allocation order, release, exhaustion."""
    from goslam_b200.modules.corr import CorrPool
    pool = CorrPool(5, 8, 8, num_levels=2, device="cpu", layout="tiled")
    assert [tuple(l.shape) for l in pool.levels] == [(5, 64, 2 * 2 * 16), (5, 64, 1 * 1 * 16)]
    with pytest.raises(ValueError):
        CorrPool(5, 8, 8, num_levels=2, device="cpu", layout="rowmajor")      # the build writes the tiled layout only
    # tiled planes are padded to whole 4x4 tiles on levels 0/1 (same formula as the C helper)
    tiled = CorrPool(2, 30, 40, num_levels=4, device="cpu")
    assert tiled.plane_elems == [8 * 10 * 16, 4 * 5 * 16, 4 * 32, 4 * 16]      # 4 bands, 3 x-blocks
    from goslam_b200 import _lib
    if os.path.exists(_lib.lib_path()):
        lib = _lib.load(build_if_missing=False)
        assert [lib.goslam_corr_level_plane_elems(i, 1, 30, 40) for i in range(4)] == tiled.plane_elems
    # de-tiling is the inverse of the kernel's tile order
    lvl = tiled.levels[1]
    lvl.copy_(torch.arange(lvl.numel(), dtype=torch.float32).reshape(lvl.shape) % 1024)
    rm = tiled.level_rowmajor(1)
    assert rm.shape == (2, 30, 40, 15, 20)
    y, x = 6, 13                      # element (y, x) lives in tile (1, 3), position (2, 1)
    assert rm[1, 7, 9, y, x] == lvl[1, 7 * 40 + 9, ((1 * 5) + 3) * 16 + 2 * 4 + 1]
    a = pool.alloc(3)
    assert a == [0, 1, 2] and pool.free_slots == 2
    pool.release([1])
    assert pool.alloc(2) == [1, 3]
    with pytest.raises(RuntimeError):
        pool.alloc(2)
    pool.release([0, 2, 1, 3])
    assert pool.free_slots == 5 and sorted(pool.alloc(5)) == [0, 1, 2, 3, 4]


def test_filter_repeated_edges_matches_python_set():
    """graph.filter_repeated_edges is device-agnostic torch plumbing: check it on CPU tensors against
    the reference's Python-set formulation (src/factor_graph.py:44-54)."""
    from goslam_b200 import graph
    from oracle import graph_oracle
    g = torch.Generator().manual_seed(4)
    ii, jj = torch.randint(0, 12, (60,), generator=g), torch.randint(0, 12, (60,), generator=g)
    ia, ja = torch.randint(0, 12, (25,), generator=g), torch.randint(0, 12, (25,), generator=g)
    ib, jb = torch.randint(0, 12, (10,), generator=g), torch.randint(0, 12, (10,), generator=g)
    got = graph.filter_repeated_edges(ii, jj, ia, ja, ib, jb)
    want = graph_oracle.filter_repeated_edges(ii.numpy(), jj.numpy(), ia.numpy(), ja.numpy(), ib.numpy(), jb.numpy())
    assert got[0].tolist() == want[0].tolist() and got[1].tolist() == want[1].tolist()
    e = torch.zeros(0, dtype=torch.long)
    assert graph.filter_repeated_edges(ii, jj, e, e, e, e)[0].tolist() == ii.tolist()


def test_synthetic_true_reprojection_matches_oracle():
    """the plain-torch setup helper that seeds bench.py's flow targets == the oracle's DepthVideo.reproject
    (incl. the stereo baseline for i == j)."""
    from goslam_b200 import synthetic
    for kw in (dict(num_kf=6, ht=12, wd=16, seed=43), dict(num_kf=5, ht=9, wd=13, seed=2, stereo_edges=3)):
        sc, _ = synthetic.make_scene(rgbd=True, with_fmaps=False, **kw)
        ref, _ = geom_oracle.reproject(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"].numpy(),
                                       sc["ii"].numpy(), sc["jj"].numpy())
        np.testing.assert_allclose(synthetic.true_reprojection(sc).numpy(), ref, rtol=1e-6, atol=1e-5)


def test_data_parallel_helpers_are_no_ops_without_a_process_group():
    """bench.py's mapping leg calls them at N = 1 without torch.distributed initialised"""
    import torch
    from goslam_b200 import parallel
    assert parallel.ray_slice(10) == (0, 10)
    p = torch.nn.Parameter(torch.ones(3))
    p.grad = torch.full((3,), 2.0)
    parallel.broadcast_parameters([p])
    parallel.allreduce_gradients([p])
    assert torch.equal(p.grad, torch.full((3,), 2.0))
