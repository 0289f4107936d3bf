"""Pin the CPU oracle (and the host-side mirrors) against golden vectors produced by the
REFERENCE'S OWN PYTHON (tests/golden/make_golden.py, run where /root/reference exists).
These run on the CPU box; the GPU parity tests then compare the kernels with the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import ba_oracle, corr_oracle, geom_oracle, neus_oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    p = os.path.join(GOLD, name)
    if not os.path.exists(p):
        pytest.skip("golden fixture %s missing" % name)
    return np.load(p)


def _rel(a, b):
    return np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max() / max(np.abs(b).max(), 1e-12)


@pytest.mark.parametrize("tag", ["f32", "f16"])
def test_corr_build_and_lookup_vs_reference_corrblock(tag):
    g = _load("corr_block.npz")
    f1, f2 = torch.from_numpy(g[tag + "_fmap1"])[0], torch.from_numpy(g[tag + "_fmap2"])[0]
    pyr = corr_oracle.corr_build(f1, f2, 4)
    for i in range(4):
        want = g["%s_level%d" % (tag, i)]
        got = pyr[i].numpy()
        assert got.shape == want.shape and got.dtype == want.dtype
        if tag == "f32":
            np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5)
        else:
            # the reference's CPU half matmul rounds differently from fp32-accumulate-then-round
            np.testing.assert_allclose(got.astype(np.float32), want.astype(np.float32), rtol=2e-3, atol=2e-3)
    # CorrBlock.__call__ plumbing (permute, /2**i, level-major concat) on the reference's own pyramid
    pyr_ref = [g["%s_level%d" % (tag, i)] for i in range(4)]
    out = corr_oracle.corr_pyramid_lookup(pyr_ref, g[tag + "_coords"][0], 3)
    np.testing.assert_array_equal(out.astype(np.float32), g[tag + "_sampled"][0].astype(np.float32))


def test_lookup_oracle_equals_grid_sample():
    rng = np.random.default_rng(0)
    vol = rng.standard_normal((2, 6, 8, 6, 8)).astype(np.float32)
    coords = (rng.uniform(-3, 10, (2, 2, 6, 8))).astype(np.float32)
    a = corr_oracle.corr_index_forward(vol, coords, 3)
    b = corr_oracle.corr_index_forward_grid_sample(vol, coords, 3)
    np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-5)


def test_lookup_oracle_edge_cases():
    vol = np.ones((1, 2, 2, 4, 4), np.float16)
    far = np.full((1, 2, 2, 2), 1000.0, np.float32)         # everything out of bounds -> zeros
    assert not corr_oracle.corr_index_forward(vol, far, 3).any()
    centre = np.full((1, 2, 2, 2), 1.5, np.float32)
    out = corr_oracle.corr_index_forward(vol, centre, 3)
    assert out.dtype == np.float16 and out.max() == 1.0 and out.min() == 0.0
    empty = corr_oracle.corr_index_forward(np.zeros((0, 2, 2, 4, 4), np.float32), np.zeros((0, 2, 2, 2), np.float32), 3)
    assert empty.shape == (0, 7, 7, 2, 2)


def test_reproject_vs_reference_projective_ops():
    g = _load("reproject.npz")
    c, v = geom_oracle.reproject(g["poses"], g["disps"], g["intrinsics"], g["ii"], g["jj"])
    np.testing.assert_allclose(c, g["coords"], rtol=1e-5, atol=2e-4)
    np.testing.assert_array_equal(v, g["valid"])
    # stereo edges (ii == jj) use the fixed baseline: x shifts by -0.1 * fx * disp
    s = g["ii"] == g["jj"]
    assert s.sum() == 2


def test_ba_oracle_vs_reference_dense_torch_ba():
    """src/geom/ba.py (the reference's pure-torch dense BA) on a scene where it and the CUDA
    formulation coincide (no sensor prior, nothing behind the camera, no stereo edges)."""
    g = _load("ba_torch.npz")
    t0 = int(g["t0"])
    num = g["poses"].shape[0]
    sens = np.zeros_like(g["disps"])
    _, _, dx, dz, st, dbg = ba_oracle.ba(g["poses"], g["disps"], g["intrinsics"][0], sens, g["targets"], g["weights"],
                                         g["eta"], g["ii"], g["jj"], t0, num, 1, 1e-4, 0.1, False,
                                         dtype=np.float64, return_debug=True, damping="pose_block")
    assert st.tolist() == [0]
    # same algebra in float64 (reference run with float64 tensors) and against its stock fp32 run
    assert _rel(dx, g["dx64"]) < 1e-5, _rel(dx, g["dx64"])
    assert _rel(dx, g["dx"]) < 2e-4, _rel(dx, g["dx"])
    # the reference torch BA does NOT drop the first optimised pose in the back-substitution
    # (the CUDA path does, :1105); undo the quirk to compare dz: dz_ref = Q (w - E^T dx) with all poses
    E, Q, w = dbg["E"], dbg["Q"], dbg["w"]
    P = num - t0
    ii_exp = np.concatenate([np.arange(t0, num), g["ii"]])
    jj_exp = np.concatenate([np.arange(t0, num), g["jj"]])
    kx, kk = np.unique(ii_exp, return_inverse=True)
    acc = np.zeros_like(Q)
    for a in range(len(jj_exp)):
        p = jj_exp[a] - t0
        if 0 <= p < P:
            acc[kk[a]] += (E[a] * dx[p].astype(np.float64)[:, None]).sum(0)
    dz_full = Q * (w - acc)
    assert _rel(dz_full, g["dz64"]) < 1e-5, _rel(dz_full, g["dz64"])


def test_ba_oracle_properties():
    from goslam_b200 import synthetic
    sc, g = synthetic.make_scene(6, 12, 16, with_fmaps=False)
    coords, _ = geom_oracle.reproject(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"].numpy(), sc["ii"].numpy(), sc["jj"].numpy())
    tg, wg, eta = synthetic.make_update(sc, torch.from_numpy(coords[0]), g, noise=0.0)
    # zero residual + matching sensor depth: BA must not move anything (dx = 0, dz ~ prior only)
    sens = sc["disps"].numpy().copy()
    p, d, dx, dz, st = ba_oracle.ba(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy(), sens,
                                    tg.numpy(), wg.numpy(), eta.numpy(), sc["ii"].numpy(), sc["jj"].numpy(), 1, 6, 2, 1e-4, 0.1, False)
    assert np.abs(dx).max() < 1e-4 and np.abs(d - sc["disps"].numpy()).max() < 1e-4
    # noisy targets: the weighted reprojection cost decreases
    tg, wg, eta = synthetic.make_update(sc, torch.from_numpy(coords[0]), g, noise=1.0)
    pose0 = sc["poses"].numpy().copy()
    pose0[1:6, :3] += 0.02
    c0 = ba_oracle.reprojection_cost(pose0, sc["disps"].numpy(), sc["intrinsics"][0].numpy(), tg.numpy(), wg.numpy(), sc["ii"].numpy(), sc["jj"].numpy())
    p, d, dx, dz, st = ba_oracle.ba(pose0, sc["disps"].numpy(), sc["intrinsics"][0].numpy(), np.zeros_like(sens),
                                    tg.numpy(), wg.numpy(), eta.numpy(), sc["ii"].numpy(), sc["jj"].numpy(), 1, 6, 3, 1e-4, 0.1, False)
    c1 = ba_oracle.reprojection_cost(p, d, sc["intrinsics"][0].numpy(), tg.numpy(), wg.numpy(), sc["ii"].numpy(), sc["jj"].numpy())
    assert c1 < c0
    # motion-only leaves the depths alone; fixed poses stay fixed
    p2, d2, _, _, _ = ba_oracle.ba(pose0, sc["disps"].numpy(), sc["intrinsics"][0].numpy(), sens, tg.numpy(), wg.numpy(), eta.numpy(),
                                   sc["ii"].numpy(), sc["jj"].numpy(), 2, 6, 1, 1e-4, 0.1, True)
    assert np.array_equal(d2, sc["disps"].numpy()) and np.array_equal(p2[:2], pose0[:2])


def test_frame_distance_oracle_properties():
    from goslam_b200 import synthetic
    sc, _ = synthetic.make_scene(5, 12, 16, with_fmaps=False)
    ii = np.arange(5)
    d = geom_oracle.frame_distance(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy(), ii, ii, 0.3)
    assert np.abs(d).max() < 1e-4                         # a frame is at distance 0 from itself
    # points pushed behind the camera -> the 1000 sentinel (src/lib/droid_kernels.cu:655)
    poses = sc["poses"].numpy().copy()
    poses[1, 2] = -100.0
    d = geom_oracle.frame_distance(poses, sc["disps"].numpy(), sc["intrinsics"][0].numpy(), np.array([0]), np.array([1]), 0.3)
    assert d[0] == 1000.0


def test_neus_oracle_vs_reference_forward():
    """oracle.neus_oracle.forward == the reference's InstantNeuS.forward (its own torch code, with
    only the tcnn modules replaced by the restatement)."""
    g = _load("neus.npz")
    from goslam_b200 import synthetic
    metas, entries = neus_oracle.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [entries * 2]
    w = synthetic.make_neus_weights(seed=int(g["weights_seed"]), total_grid_params=entries * 2,
                                    layout=(offs, [m["res"] for m in metas]))
    args = (w["grid"].half().numpy(), w["sdf_w"].numpy(), w["sdf_b"].numpy(), w["color_B"].numpy(),
            w["mlp"].half().numpy(), g["bound"], g["rt_bound"], 0.2, 10.0)
    out = neus_oracle.forward(*args, g["rays_o"], g["rays_d"], g["z_vals_in"], g["dists"])
    ulp = neus_oracle.forward(*args, np.nextafter(g["rays_o"], np.float32(10)), g["rays_d"], g["z_vals_in"], g["dists"])
    for k in ("z_vals", "sdf", "sdf_variance"):
        assert _rel(out[k], g["out_" + k].reshape(out[k].shape)) < 2e-5, k
    for k in ("color", "depth", "depth_variance", "normal", "weight_sum", "gradient_error"):
        want = g["out_" + k].reshape(out[k].shape)
        sens = _rel(ulp[k], out[k])
        assert _rel(out[k], want) < max(2e-4, 4 * sens), (k, _rel(out[k], want), sens)


@pytest.mark.parametrize("tag", ["s24", "s48", "s72", "fallback"])
def test_neus_oracle_vs_reference_training_forward_cases(tag):
    """oracle.neus_oracle.forward == the forward outputs stored in neus_grad_cases.npz: the reference's InstantNeuS.forward
    under enable_grad with the differentiable tcnn restatements, at S = 24, 48, 72 and on a batch with nothing inside
    realtime_bound (the reference then forces its first 100 samples in).  The restatements accumulate the encoding in
    fp32 where the oracle rounds to fp16 per corner, as the golden neus_grad comparison on the GPU allows: 2e-3."""
    g = _load("neus_grad_cases.npz")
    from goslam_b200 import synthetic
    metas, entries = neus_oracle.hashgrid_meta()
    offs = [m["offset"] * 2 for m in metas] + [entries * 2]
    w = synthetic.make_neus_weights(seed=int(g["weights_seed"]), total_grid_params=entries * 2,
                                    layout=(offs, [m["res"] for m in metas]))
    c = {k[len(tag) + 1:]: g[k] for k in g.files if k.startswith(tag + "_")}
    out = neus_oracle.forward(w["grid"].half().numpy(), w["sdf_w"].numpy(), w["sdf_b"].numpy(), w["color_B"].numpy(),
                              w["mlp"].half().numpy(), g["bound"], c["rt_bound"], 0.2, 10.0,
                              c["rays_o"], c["rays_d"], c["z_vals_in"], c["dists"])
    inb = c["out_sdf"] != 100.0
    assert np.array_equal(inb, out["sdf"] != 100.0)
    if tag == "fallback":
        assert np.array_equal(inb.reshape(-1), np.arange(inb.size) < 100)
    assert np.abs(out["sdf"][inb] - c["out_sdf"][inb]).max() <= 2e-3 * np.abs(c["out_sdf"][inb]).max()
    for k in ("color", "depth", "depth_variance", "normal", "weight_sum", "z_vals", "gradient_error"):
        want = c["out_" + k].reshape(out[k].shape)
        assert np.abs(out[k] - want).max() <= 2e-3 * max(1.0, np.abs(want).max()), (k, np.abs(out[k] - want).max())
    assert (c["out_weight_sum"] > 1e-3).sum() >= 3, "degenerate case: nothing is rendered"


def test_neus_oracle_edge_cases():
    from goslam_b200 import synthetic
    metas, entries = neus_oracle.hashgrid_meta()
    w = synthetic.make_neus_weights(seed=1, total_grid_params=entries * 2, trained_like=False)
    b = np.array([[-1.0, 1.0]] * 3, np.float32)
    ro = np.full((4, 3), 50.0, np.float32)                  # every sample out of bound
    rd = np.tile(np.array([[0.0, 0.0, 1.0]], np.float32), (4, 1))
    zv = np.tile(np.linspace(0.1, 1, 40, dtype=np.float32), (4, 1))
    ds = np.full((4, 40), 0.02, np.float32)
    out = neus_oracle.forward(w["grid"].half().numpy(), w["sdf_w"].numpy(), w["sdf_b"].numpy(), w["color_B"].numpy(),
                              w["mlp"].half().numpy(), b, b, 0.2, 10.0, ro, rd, zv, ds)
    # the reference forces mask[:100] = True when nothing is in bound (src/InstantNeuS.py:311-312)
    assert (out["sdf"].reshape(-1)[:100] != 100.0).all() and (out["sdf"].reshape(-1)[100:] == 100.0).all()
    assert out["weight_sum"][3, 0] == 0.0 and out["weight_sum"][0, 0] > 0.0


def test_render_z_sampling_oracle_bit_exact():
    g = _load("render_z.npz")
    from oracle.render_oracle import sample_z
    torch.manual_seed(int(g["torch_seed"]))
    bound = torch.tensor([[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]])
    z, d = sample_z(torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"]), bound,
                    torch.from_numpy(g["gt_depth"]), 24, 48, perturb=1.0, lindisp=False)
    np.testing.assert_array_equal(z.numpy(), g["z_vals"])
    np.testing.assert_array_equal(d.numpy(), g["dists"])


def test_cvx_upsample_oracle_matches_reference_function():
    """oracle/upsample_oracle.py against outputs of the reference's own cvx_upsample (src/droid_net.py:9-23)."""
    from oracle import upsample_oracle
    g = _load("cvx_upsample.npz")
    for tag in ("disp", "flow"):
        data, mask = torch.from_numpy(g[tag + "_data"]), torch.from_numpy(g[tag + "_mask"])
        np.testing.assert_allclose(upsample_oracle.cvx_upsample(data, mask).numpy(), g[tag + "_out_f32"], rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(upsample_oracle.cvx_upsample(data, mask.half()).numpy(), g[tag + "_out_f16mask"],
                                   rtol=1e-6, atol=1e-7)


def test_proximity_edges_oracle_matches_reference_method():
    """oracle/graph_oracle.py against the edges FactorGraph.add_proximity_factors itself produced
    (src/factor_graph.py:384-450, run by tests/golden/make_golden.py with a stub video)."""
    from oracle import graph_oracle
    g = _load("proximity.npz")
    for n in range(int(g["n_cases"])):
        t0, t1, t, rad, nms, maxf, st = [int(x) for x in g["c%d_params" % n]]
        old = g["c%d_old" % n]
        es = graph_oracle.proximity_edges(g["c%d_dist" % n], t0, t1, t, rad, nms, float(g["c%d_thresh" % n]), maxf,
                                          bool(st), old[:, 0], old[:, 1])
        np.testing.assert_array_equal(es, g["c%d_es" % n])


def test_backend_edges_oracle_matches_reference_method():
    """oracle/graph_oracle.backend_edges against Backend.ba's own edge list (src/backend.py:25-99; dense and loop-closure modes)."""
    from oracle import graph_oracle
    g = _load("backend_edges.npz")
    for n in range(int(g["n_cases"])):
        ts, te, rad, nms, maxf, st, tsl, loop = [int(x) for x in g["b%d_params" % n]]
        es = graph_oracle.backend_edges(g["b%d_dist" % n], ts, te, rad, nms, float(g["b%d_thresh" % n]), maxf, bool(st),
                                        None if tsl < 0 else tsl, bool(loop))
        if int(g["b%d_early" % n]):
            assert es is None
        else:
            np.testing.assert_array_equal(es, g["b%d_es" % n])


def test_altcorr_block_pyramid_matches_reference_constructor():
    """goslam_b200.modules.AltCorrBlock.__init__ is torch-only: its pyramid must equal the reference
    constructor's (src/modules/corr.py:97-111) bit for bit."""
    from goslam_b200.modules.corr import AltCorrBlock
    g = _load("altcorr_pyramid.npz")
    blk = AltCorrBlock(torch.from_numpy(g["fmaps"]))
    assert len(blk.pyramid) == 4
    for i, lvl in enumerate(blk.pyramid):
        assert torch.equal(lvl, torch.from_numpy(g["level%d" % i]))
