"""GPU parity tests (run on an H100): every kernel of the hot path, called through the
C-ABI (via the droid_backends / CorrBlock / InstantNeuS shims), against the CPU oracle on the
same seeded inputs.  Tolerances are written next to each assertion."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ba_oracle, corr_oracle, geom_oracle, neus_oracle  # noqa: E402


def dev():
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)


# ------------------------------------------------------------------------------ lookup
def _lookup_case(dtype, N, h1, w1, h2, w2, seed):
    g = torch.Generator().manual_seed(seed)
    vol = torch.randn(N, h1, w1, h2, w2, generator=g)
    vol = vol.half() if dtype == "f16" else vol
    base = torch.stack(torch.meshgrid(torch.arange(w1).float(), torch.arange(h1).float(), indexing="xy"), 0)
    coords = base[None].repeat(N, 1, 1, 1) * (w2 / w1) + 3.0 * torch.randn(N, 2, h1, w1, generator=g)
    coords[0, :, 0, 0] = torch.tensor([-7.5, -9.25])           # fully outside
    coords[0, :, 0, 1] = torch.tensor([w2 + 2.5, h2 + 1.0])
    coords[0, :, 1, 0] = torch.tensor([-0.5, 0.5])             # straddling the border
    coords[0, :, 1, 1] = torch.tensor([float(w2 - 1), float(h2 - 1)])   # integer coords (dx = 0)
    return vol, coords.contiguous()


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("shape", [(3, 12, 16, 12, 16), (2, 9, 11, 7, 10), (2, 6, 8, 3, 5)])
def test_corr_index_forward(dtype, shape):
    from goslam_b200 import droid_backends
    vol, coords = _lookup_case(dtype, *shape, seed=1)
    out, = droid_backends.corr_index_forward(vol.to(dev()), coords.to(dev()), 3)
    ref = corr_oracle.corr_index_forward(vol.numpy(), coords.numpy(), 3)
    got = out.cpu().numpy()
    assert got.shape == ref.shape and got.dtype == ref.dtype
    if dtype == "f16":
        # the half instantiation is a fixed sequence of correctly-rounded half ops: bit-exact
        np.testing.assert_array_equal(got.astype(np.float32), ref.astype(np.float32))
    else:
        # chained FMAs in the reference's order; the oracle emulates FMA in float64: <= 1 ulp
        np.testing.assert_allclose(got, ref, rtol=2e-7, atol=1e-7)


def test_corr_index_forward_vs_grid_sample():
    from goslam_b200 import droid_backends
    vol, coords = _lookup_case("f32", 2, 12, 16, 12, 16, seed=2)
    out, = droid_backends.corr_index_forward(vol.to(dev()), coords.to(dev()), 3)
    ref = corr_oracle.corr_index_forward_grid_sample(vol.numpy(), coords.numpy(), 3)
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-5, atol=2e-5)


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("hw", [(16, 16), (12, 20), (30, 40)])
def test_corr_block_build_and_lookup(dtype, hw):
    """CorrBlock(fmap1, fmap2)(coords): build (auto impl) + fused 4-level lookup."""
    from goslam_b200.modules import CorrBlock
    h, w = hw
    N = 2
    g = torch.Generator().manual_seed(3)
    f1 = torch.randn(1, N, 128, h, w, generator=g)
    f2 = torch.randn(1, N, 128, h, w, generator=g)
    if dtype == "f16":
        f1, f2 = f1.half(), f2.half()
    blk = CorrBlock(f1.to(dev()), f2.to(dev()))
    ref = corr_oracle.corr_build(f1[0], f2[0], 4)
    for i in range(4):
        got = blk.corr_pyramid[i].float().cpu().numpy()
        want = ref[i].float().numpy()
        assert got.shape == want.shape
        if dtype == "f16":
            # fp32 accumulate in a different order, one rounding to half: <= 1 half-ulp
            np.testing.assert_allclose(got, want, rtol=1.5e-3, atol=1e-3)
            assert (got == want).mean() > 0.97
        else:
            np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-4)
    coords = torch.stack(torch.meshgrid(torch.arange(w).float(), torch.arange(h).float(), indexing="xy"), -1)
    coords = coords[None, None].repeat(1, N, 1, 1, 1) + 2.5 * torch.randn(1, N, h, w, 2, generator=g)
    out = blk(coords.to(dev()))
    pyr = [p.cpu().numpy() for p in blk.corr_pyramid]
    want = corr_oracle.corr_pyramid_lookup(pyr, coords[0].numpy(), 3)
    got = out[0].cpu().numpy()
    assert got.shape == want.shape
    if dtype == "f16":
        np.testing.assert_array_equal(got.astype(np.float32), want.astype(np.float32))
    else:
        np.testing.assert_allclose(got, want, rtol=2e-7, atol=1e-7)


def _simt_pyramid(f1, f2, num_levels=4):
    """goslam_corr_build, the CUDA-core row-major build, called directly on half feature maps [N, D, h, w]."""
    import ctypes
    from goslam_b200 import _lib
    N, D, h, w = f1.shape
    levels = [torch.empty((N, h, w, h >> i, w >> i), dtype=torch.float16, device=f1.device) for i in range(num_levels)]
    ptrs = (ctypes.c_void_p * num_levels)(*[t.data_ptr() for t in levels])
    rc = _lib.load().goslam_corr_build(_lib.ptr(f1), _lib.ptr(f2), 1, ptrs, num_levels, N, D, h, w, _lib.stream_ptr())
    _lib.check(rc, "corr_build")
    return levels


def _rowmajor_lookup(pyramid, coords):
    """goslam_corr_pyramid_lookup on row-major f16 levels [N, h, w, h>>i, w>>i]; coords [1, N, h, w, 2]."""
    import ctypes
    from goslam_b200 import _lib
    N, h, w = pyramid[0].shape[:3]
    L = len(pyramid)
    out = torch.empty((1, N, L * 49, h, w), dtype=torch.float16, device=coords.device)
    c = coords.reshape(N, h, w, 2).float().contiguous()
    ptrs = (ctypes.c_void_p * L)(*[t.data_ptr() for t in pyramid])
    rc = _lib.load().goslam_corr_pyramid_lookup(ptrs, 1, L, _lib.ptr(c), _lib.ptr(out), N, h, w, h, w, 3,
                                                _lib.stream_ptr())
    _lib.check(rc, "corr_pyramid_lookup")
    return out


@pytest.mark.parametrize("hw", [(40, 80), (30, 40), (12, 20)])
def test_corr_build_tc_matches_simt(hw):
    """the tensor-core kernel (CorrBlock on half inputs) and its CUDA-core twin (goslam_corr_build) share
    one numerics contract; they may differ only where fp32 summation order flips a half rounding."""
    from goslam_b200.modules import CorrBlock
    h, w = hw
    g = torch.Generator().manual_seed(4)
    f1 = torch.randn(1, 3, 128, h, w, generator=g).half().to(dev())
    f2 = torch.randn(1, 3, 128, h, w, generator=g).half().to(dev())
    a = CorrBlock(f1, f2)
    assert a.pool is not None
    b = _simt_pyramid(f1[0], f2[0])
    for i in range(4):
        x, y = a.corr_pyramid[i].float(), b[i].float()
        assert x.shape == y.shape
        assert torch.isfinite(x).all()
        assert (x - y).abs().max().item() <= 2e-3 * max(1.0, y.abs().max().item())
        assert (x == y).float().mean().item() > 0.97
    # cuBLAS-style check of level 0 against torch on the device
    want = torch.matmul((f1[0] / 4).reshape(3, 128, h * w).transpose(1, 2).float(),
                        (f2[0] / 4).reshape(3, 128, h * w).float()).half().float()
    got = a.corr_pyramid[0].reshape(3, h * w, h * w).float()
    assert (got - want).abs().max().item() <= 2e-3 * max(1.0, want.abs().max().item())


def test_corr_block_from_video_matches_gathered_build():
    """video-level indexed build (K-major per-frame feature maps, edge->frame indirection on the
    device, stereo slot rule) == CorrBlock(fmaps[ii,0], fmaps[jj,c])."""
    from goslam_b200.modules import CorrBlock
    from goslam_b200.modules.corr import fmaps_to_kmajor
    g = torch.Generator().manual_seed(6)
    h, w = 24, 32
    for rig in (1, 2):
        fmaps = torch.randn(5, rig, 128, h, w, generator=g).half().to(dev())
        ii = torch.tensor([0, 1, 2, 4, 3, 2], device=dev())
        jj = torch.tensor([1, 0, 4, 2, 3 if rig == 2 else 0, 1], device=dev())
        c = (ii == jj).long() if rig == 2 else torch.zeros_like(ii)
        a = CorrBlock(fmaps[ii, 0][None], fmaps[jj, c][None])
        km = fmaps_to_kmajor(fmaps)
        assert km.shape == (5 * rig, h * w, 128)
        b = CorrBlock.from_video(km, ii, jj, h, w, rig=rig)
        for x, y in zip(a.corr_pyramid, b.corr_pyramid):
            assert torch.equal(x, y)


@pytest.mark.parametrize("hw", [(24, 32), (30, 40), (22, 26), (8, 16), (37, 45), (20, 128)])
def test_corr_pool_add_remove_matches_cat_and_mask(hw):
    """FactorGraph's add_factors / rm_factors sequence (src/factor_graph.py:114,149) on a slot pool:
    cat() and [mask] edit the slot table only, and the pooled pyramid and lookup equal, bit for bit, the
    reference's torch.cat / mask of the one-block pyramids and the row-major lookup on that."""
    from goslam_b200.modules import CorrBlock
    from goslam_b200.modules.corr import CorrPool, fmaps_to_kmajor
    g = torch.Generator().manual_seed(16)
    h, w = hw
    fmaps = torch.randn(6, 1, 128, h, w, generator=g).half().to(dev())
    km = fmaps_to_kmajor(fmaps)
    pool = CorrPool(10, h, w, device=dev())
    ptrs = [lvl.data_ptr() for lvl in pool.levels]

    def edges(pairs):
        t = torch.tensor(pairs, device=dev())
        return t[:, 0].contiguous(), t[:, 1].contiguous()

    def coords_for(n):
        base = torch.stack(torch.meshgrid(torch.arange(w).float(), torch.arange(h).float(), indexing="xy"), -1)
        c = base[None, None] + 3 * torch.randn(1, n, h, w, 2, generator=g)
        c[0, :, 0, :3] = torch.tensor([-5.5, 2.25])           # windows hanging over every border
        c[0, :, 1, :3] = torch.tensor([w + 1.5, h - 2.0])
        c[0, :, 2, :3] = torch.tensor([w / 2.0, -3.75])
        c[0, :, 3, :3] = torch.tensor([1.0, h + 2.5])
        return c.to(dev())

    i1, j1 = edges([(0, 1), (1, 0), (1, 2), (2, 1)])
    i2, j2 = edges([(2, 3), (3, 2), (0, 3)])
    i3, j3 = edges([(4, 5), (5, 4), (3, 5), (5, 3), (4, 2)])
    def one_block(i, j):
        return CorrBlock.from_video(km, i, j, h, w).gather_pyramid()

    def check(plain, pooled, n):
        for x, y in zip(plain, pooled.gather_pyramid()):
            assert torch.equal(x, y)
        c = coords_for(n)
        assert torch.equal(_rowmajor_lookup(plain, c), pooled(c))

    plain = one_block(i1, j1)                                # the reference's row-major pyramid, edited by copies
    pooled = CorrBlock.from_video(km, i1, j1, h, w, pool=pool)
    assert pool.free_slots == 6
    # add
    plain = [torch.cat([x, y]) for x, y in zip(plain, one_block(i2, j2))]
    pooled = pooled.cat(CorrBlock.from_video(km, i2, j2, h, w, pool=pool))
    assert pool.free_slots == 3 and len(pooled._slots_host) == 7
    check(plain, pooled, 7)
    # remove (boolean keep-mask, as rm_factors passes ~mask)
    keep = torch.tensor([True, False, True, True, False, True, False], device=dev())
    plain, pooled = [x[keep] for x in plain], pooled[keep]
    assert pool.free_slots == 6
    check(plain, pooled, 4)
    # add again: freed slots are reused, nothing was reallocated or moved
    plain = [torch.cat([x, y]) for x, y in zip(plain, one_block(i3, j3))]
    pooled = pooled.cat(CorrBlock.from_video(km, i3, j3, h, w, pool=pool))
    assert pool.free_slots == 1 and sorted(pooled._slots_host) == sorted(set(pooled._slots_host))
    check(plain, pooled, 9)
    assert [lvl.data_ptr() for lvl in pool.levels] == ptrs
    with pytest.raises(RuntimeError):
        CorrBlock.from_video(km, i1, j1, h, w, pool=pool)      # 4 edges, 1 free slot
    pooled.free()
    assert pool.free_slots == 10


# ------------------------------------------------------------------------------ altcorr
def test_altcorr_forward():
    from goslam_b200 import droid_backends
    g = torch.Generator().manual_seed(5)
    B, H, W, C, S = 3, 10, 12, 128, 2
    f1 = torch.randn(B, H, W, C, generator=g)
    f2 = torch.randn(B, H // 2, W // 2, C, generator=g)
    base = torch.stack(torch.meshgrid(torch.arange(W).float(), torch.arange(H).float(), indexing="xy"), -1)
    coords = (base[None, None].repeat(B, S, 1, 1, 1) + 2 * torch.randn(B, S, H, W, 2, generator=g)) / 2
    coords[0, 0, 0, 0] = torch.tensor([-20.0, 3.0])
    out, = droid_backends.altcorr_forward(f1.to(dev()), f2.to(dev()), coords.to(dev()).contiguous(), 3)
    ref = corr_oracle.altcorr_forward(f1.numpy(), f2.numpy(), coords.numpy(), 3)
    # fp32 dot products of 128 terms in a different order: 1e-5 relative to the value scale
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-4, atol=1e-4)


def _altcorr_per_level_twin(blk, coords, ii, jj):
    """test twin of AltCorrBlock: one drop-in `altcorr_forward` launch per level on gathered fp32 maps — the
    shape of the reference's own path (src/modules/corr.py:113-131), kept HERE as a checker only."""
    from goslam_b200 import droid_backends
    b, n, h, w, s, _ = coords.shape
    pts = coords.permute(0, 1, 4, 2, 3, 5)
    src = blk.pyramid[0][0, ii].float().contiguous()
    outs = []
    for lvl, maps in enumerate(blk.pyramid):
        tgt = maps[0, jj].float().contiguous()
        c, = droid_backends.altcorr_forward(src, tgt, (pts / float(1 << lvl)).reshape(n, s, h, w, 2).contiguous(), blk.radius)
        outs.append(c.view(b, n, s, -1, h, w).permute(0, 1, 3, 4, 5, 2))
    return torch.cat(outs, dim=2)


def test_altcorr_block_fused_matches_per_level_path():
    """AltCorrBlock(fmaps)(coords, ii, jj): fused indexed half-precision tensor-core launch == per-level
    drop-in altcorr_forward launches on gathered fp32 maps == the oracle; 5-D and 6-D (S sets) coords."""
    from goslam_b200.modules import AltCorrBlock
    g = torch.Generator().manual_seed(8)
    F, H, W, N = 6, 30, 40, 9
    fm = torch.randn(1, F, 128, H, W, generator=g).half().to(dev())
    blk = AltCorrBlock(fm)
    ii = torch.randint(0, F, (N,), generator=g).to(dev())
    jj = torch.randint(0, F, (N,), generator=g).to(dev())
    base = torch.stack(torch.meshgrid(torch.arange(W).float(), torch.arange(H).float(), indexing="xy"), -1)
    coords = (base[None, None].repeat(1, N, 1, 1, 1) + 3 * torch.randn(1, N, H, W, 2, generator=g)).to(dev())
    fused = blk(coords, ii, jj)
    slow = _altcorr_per_level_twin(blk, coords.unsqueeze(-2), ii, jj).squeeze(-1).contiguous()
    assert fused.shape == slow.shape == (1, N, 196, H, W)
    assert (fused - slow).abs().max().item() < 1e-4 * max(1.0, slow.abs().max().item())
    lvl = 2
    ref = corr_oracle.altcorr_forward(blk.pyramid[0][0, ii].float().cpu().numpy(), blk.pyramid[lvl][0, jj].float().cpu().numpy(),
                                      (coords[0] / 2 ** lvl).unsqueeze(1).cpu().numpy(), 3)
    np.testing.assert_allclose(fused[0, :, 49 * lvl:49 * (lvl + 1)].cpu().numpy(), ref[:, 0], rtol=1e-4, atol=1e-4)
    c6 = torch.stack([coords, coords + torch.tensor([0.25, -0.5], device=dev())], dim=-2)      # S = 2
    out6 = blk(c6, ii, jj)
    want6 = _altcorr_per_level_twin(blk, c6, ii, jj)
    assert out6.shape == want6.shape == (1, N, 196, H, W, 2)
    assert torch.equal(out6[..., 0], fused)
    assert (out6 - want6).abs().max().item() < 1e-4 * max(1.0, want6.abs().max().item())


def test_altcorr_block_vs_reference_class_golden():
    """outputs of the REFERENCE AltCorrBlock class (src/modules/corr.py:113-145; golden made with the oracle
    standing in for its CUDA op, fp32 maps): gather per edge, coords / 2^l, channel order, 5-D and 6-D coords.
    The per-level twin on the drop-in fp32 kernel reproduces it to fp32 summation order; the fused
    half-precision launch to the half rounding of the pooled maps."""
    from goslam_b200.modules import AltCorrBlock
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "altcorr_block.npz"))
    fm = torch.from_numpy(g["fmaps"]).to(dev())
    ii, jj = torch.from_numpy(g["ii"]).to(dev()), torch.from_numpy(g["jj"]).to(dev())
    c5, c6 = torch.from_numpy(g["coords"]).to(dev()), torch.from_numpy(g["coords6"]).to(dev())
    blk32 = AltCorrBlock(fm)
    out5 = _altcorr_per_level_twin(blk32, c5.unsqueeze(-2), ii, jj).squeeze(-1)
    out6 = _altcorr_per_level_twin(blk32, c6, ii, jj)
    np.testing.assert_allclose(out5[:, :, ::7].cpu().numpy(), g["out5"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(out6[:, :, ::7].cpu().numpy(), g["out6"], rtol=1e-4, atol=1e-4)
    blk16 = AltCorrBlock(fm.half())
    f5, f6 = blk16(c5, ii, jj), blk16(c6, ii, jj)
    assert f5.shape == (1, 3, 196, 16, 24) and f6.shape == (1, 3, 196, 16, 24, 2)
    scale = float(np.abs(g["out5"]).max())
    assert np.abs(f5[:, :, ::7].cpu().numpy() - g["out5"]).max() < 4e-3 * scale      # fp16 inputs (2^-11 each)
    assert np.abs(f6[:, :, ::7].cpu().numpy() - g["out6"]).max() < 4e-3 * scale


# ------------------------------------------------------------------------------ geometry
def _scene(num_kf=6, ht=12, wd=16, **kw):
    from goslam_b200 import synthetic
    return synthetic.make_scene(num_kf=num_kf, ht=ht, wd=wd, **kw)


def _to_dev(sc, *keys):
    return [sc[k].to(dev()).contiguous() for k in keys]


@pytest.mark.parametrize("size", [(6, 12, 16), (8, 40, 80)])
def test_frame_distance(size):
    from goslam_b200 import droid_backends
    sc, g = _scene(*size, with_fmaps=False)
    n = size[0]
    ii, jj = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
    ii, jj = ii.reshape(-1), jj.reshape(-1)
    poses, disps, intr = _to_dev(sc, "poses", "disps", "intrinsics")
    for beta in (0.3, 0.75):
        d = droid_backends.frame_distance(poses, disps, intr[0].contiguous(), ii.to(dev()), jj.to(dev()), beta)
        ref = geom_oracle.frame_distance(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy(),
                                         ii.numpy(), jj.numpy(), beta)
        got = d.cpu().numpy()
        # same summation tree; remaining differences are FMA contraction inside the projection
        np.testing.assert_allclose(got, ref, rtol=2e-5, atol=1e-6)
        # the edge set the frontend derives from it (distance < thresh) must be identical
        for thresh in (2.0, 8.0, 16.0):
            assert ((got < thresh) == (ref < thresh)).all()
        assert (np.argsort(got, kind="stable") == np.argsort(ref, kind="stable")).mean() > 0.95


def test_frame_distance_bidirectional_equals_two_launches():
    """goslam_frame_distance_bidir == 0.5 * (d(ii,jj) + d(jj,ii)) of the one-way kernel, bit for bit."""
    from goslam_b200 import droid_backends
    sc, _ = _scene(7, 30, 40, seed=3, with_fmaps=False)
    poses, disps, intr = _to_dev(sc, "poses", "disps", "intrinsics")
    ii, jj = torch.meshgrid(torch.arange(7), torch.arange(7), indexing="ij")
    ii, jj = ii.reshape(-1).to(dev()), jj.reshape(-1).to(dev())
    d1 = droid_backends.frame_distance(poses, disps, intr[0].contiguous(), ii, jj, 0.3)
    d2 = droid_backends.frame_distance(poses, disps, intr[0].contiguous(), jj, ii, 0.3)
    both = droid_backends.frame_distance_bidirectional(poses, disps, intr[0].contiguous(), ii, jj, 0.3)
    assert torch.equal(both, 0.5 * (d1 + d2))


def test_projmap_iproj_depth_filter_reproject():
    from goslam_b200 import droid_backends
    sc, g = _scene(7, 12, 16, with_fmaps=False)
    poses, disps, intr = _to_dev(sc, "poses", "disps", "intrinsics")
    ii, jj = sc["ii"], sc["jj"]
    c, v = droid_backends.projmap(poses, disps, intr[0].contiguous(), ii.to(dev()), jj.to(dev()))
    rc, rv = geom_oracle.projmap(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy(), ii.numpy(), jj.numpy())
    np.testing.assert_allclose(c.cpu().numpy(), rc, rtol=1e-5, atol=1e-4)
    np.testing.assert_array_equal(v.cpu().numpy(), rv)
    pts = droid_backends.iproj(poses, disps, intr[0].contiguous())
    np.testing.assert_allclose(pts.cpu().numpy(), geom_oracle.iproj(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy()),
                               rtol=1e-5, atol=1e-5)
    ix = torch.arange(7)
    th = torch.full((7,), 0.05)
    cnt = droid_backends.depth_filter(poses, disps, intr[0].contiguous(), ix.to(dev()), th.to(dev()))
    ref = geom_oracle.depth_filter(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy(), ix.numpy(), th.numpy())
    assert (cnt.cpu().numpy() == ref).mean() > 0.995     # counts are integers; borderline |.|<t may flip
    co, va = droid_backends.reproject(poses, disps, intr, ii.to(dev()), jj.to(dev()))
    rco, rva = geom_oracle.reproject(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"].numpy(), ii.numpy(), jj.numpy())
    np.testing.assert_allclose(co.cpu().numpy(), rco, rtol=1e-5, atol=1e-4)
    np.testing.assert_array_equal(va.cpu().numpy(), rva)


# ------------------------------------------------------------------------------ bundle adjustment
def _ba_case(num_kf, ht, wd, rgbd, stereo_edges=0, seed=43, t0=1):
    from goslam_b200 import synthetic
    sc, g = synthetic.make_scene(num_kf=num_kf, ht=ht, wd=wd, rgbd=rgbd, seed=seed, with_fmaps=False,
                                 stereo_edges=stereo_edges, buffer=num_kf + 3)
    sc["t0"] = t0
    coords, _ = geom_oracle.reproject(sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"].numpy(),
                                      sc["ii"].numpy(), sc["jj"].numpy())
    targets, weights, eta = synthetic.make_update(sc, torch.from_numpy(coords[0]), g, noise=0.7)
    # perturb the state so that BA has something to do
    sc["poses"][1:num_kf, :3] += 0.01 * torch.randn(num_kf - 1, 3, generator=g)
    sc["disps"][:num_kf] *= 1 + 0.03 * torch.randn(num_kf, ht, wd, generator=g)
    return sc, targets, weights, eta


@pytest.mark.parametrize("case", [
    dict(num_kf=6, ht=12, wd=16, rgbd=True),
    dict(num_kf=6, ht=12, wd=16, rgbd=False),
    dict(num_kf=5, ht=9, wd=13, rgbd=True, stereo_edges=3),
    dict(num_kf=8, ht=40, wd=80, rgbd=True),
    dict(num_kf=8, ht=40, wd=80, rgbd=False, t0=2),
])
@pytest.mark.parametrize("motion_only", [False, True])
def test_ba(case, motion_only):
    from goslam_b200 import droid_backends
    sc, targets, weights, eta = _ba_case(**case)
    t0, t1 = sc["t0"], sc["t1"]
    iters, lm, ep = 3, 1e-4, 0.1
    poses = sc["poses"].clone().to(dev())
    disps = sc["disps"].clone().to(dev())
    dx, dz, status = droid_backends.ba(
        poses, disps, sc["intrinsics"][0].to(dev()).contiguous(), sc["disps_sens"].to(dev()),
        targets.to(dev()), weights.to(dev()), eta.to(dev()), sc["ii"].to(dev()), sc["jj"].to(dev()),
        t0, t1, iters, lm, ep, motion_only, return_status=True)
    rp, rd, rdx, rdz, rst = ba_oracle.ba(
        sc["poses"].numpy(), sc["disps"].numpy(), sc["intrinsics"][0].numpy(), sc["disps_sens"].numpy(),
        targets.numpy(), weights.numpy(), eta.numpy(), sc["ii"].numpy(), sc["jj"].numpy(),
        t0, t1, iters, lm, ep, motion_only, dtype=np.float64)
    assert status.cpu().numpy().tolist() == rst.tolist() == [0] * iters
    # north_star tolerance: 1e-4 relative (fp32) on the updated state and the last step
    assert _rel(poses.cpu().numpy(), rp) < 1e-4
    assert _rel(dx.cpu().numpy(), rdx) < 2e-3          # dx is the *difference* of two ~equal iterates' worth
    if not motion_only:
        assert _rel(disps.cpu().numpy(), rd) < 1e-4
        assert np.abs(dz.cpu().numpy() - rdz).max() < 1e-4 * max(np.abs(rd).max(), 1.0)
    else:
        assert torch.equal(disps.cpu(), sc["disps"])
        assert dz is None
    # frames outside [t0,t1) keep their pose
    assert torch.equal(poses[:t0].cpu(), sc["poses"][:t0])
    assert torch.equal(poses[t1:].cpu(), sc["poses"][t1:])


def test_ba_failed_factorisation_gives_zero_step():
    """negative weights make the reduced system indefinite: the reference falls back to dx = 0
    (src/lib/droid_kernels.cu:1207-1210)."""
    from goslam_b200 import droid_backends
    sc, targets, weights, eta = _ba_case(num_kf=5, ht=9, wd=13, rgbd=False)
    poses = sc["poses"].clone().to(dev())
    disps = sc["disps"].clone().to(dev())
    dx, dz, status = droid_backends.ba(
        poses, disps, sc["intrinsics"][0].to(dev()).contiguous(), sc["disps_sens"].to(dev()),
        targets.to(dev()), (-1e6 * weights).to(dev()), eta.to(dev()), sc["ii"].to(dev()), sc["jj"].to(dev()),
        1, 5, 1, 1e-4, 0.1, True, return_status=True)
    assert status.cpu().tolist() == [1]
    assert float(dx.abs().max()) == 0.0
    assert torch.equal(poses.cpu(), sc["poses"])


# ------------------------------------------------------------------------------ renderer
@pytest.mark.parametrize("R", [37, 256, 1500])
def test_neus_forward(R):
    from goslam_b200 import neus, synthetic
    offs, ress, _, total = neus.hashgrid_layout()
    metas, tot_entries = neus_oracle.hashgrid_meta()
    assert total == 2 * tot_entries
    w = synthetic.make_neus_weights(seed=7, total_grid_params=total, layout=(offs, ress))
    bound = [[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]]
    net = neus.InstantNeuS(synthetic.NEUS_CFG, bound)
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to(dev())
    net.update_bound(torch.tensor([[-1.8, 1.9], [-2.0, 2.0], [-1.5, 2.0]]))
    ro, rd, zv, ds = synthetic.make_rays(R, S=72, seed=11)
    out = net(ro.to(dev()), rd.to(dev()), zv.to(dev()), ds.to(dev()), debug=True)
    ref = neus_oracle.forward(
        w["grid"].half().numpy(), w["sdf_w"].numpy(), w["sdf_b"].numpy(), w["color_B"].numpy(),
        w["mlp"].half().numpy(), np.array(bound, np.float32), net.realtime_bound.cpu().numpy(),
        0.2, 10.0, ro.numpy(), rd.numpy(), zv.numpy(), ds.numpy(), debug=True)
    assert set(out.keys()) == set(k for k in ref.keys() if not k.startswith("_"))
    got = {k: v.cpu().numpy() for k, v in out.items()}
    assert (ref["weight_sum"] > 1e-3).mean() > 0.2, "degenerate test scene: nothing is rendered"
    # per-sample quantities before the NeuS alpha: 1e-4 relative (north_star)
    for k in ("z_vals", "sdf", "sdf_variance"):
        assert got[k].shape == ref[k].shape, k
        assert _rel(got[k], ref[k]) < 1e-4, (k, _rel(got[k], ref[k]))
    inb = ref["sdf"] != 100.0                 # the 100 sentinel would hide errors in a max-norm
    assert np.array_equal(inb, got["sdf"] != 100.0)
    assert np.abs(got["sdf"][inb] - ref["sdf"][inb]).max() < 1e-4 * np.abs(ref["sdf"][inb]).max()
    # per-sample intermediates that drive the compositing (test-only outputs of the kernel)
    dbg = net.last_debug
    assert np.abs(dbg["alpha"].cpu().numpy() - ref["_alpha"]).max() < 1e-5
    assert np.abs(dbg["grad"].cpu().numpy().reshape(-1, 3) - ref["_grad"]).max() < 1e-5 * max(1.0, np.abs(ref["_grad"]).max())
    assert np.array_equal(dbg["pos"].cpu().numpy().reshape(-1, 3)[ref["_mask"]], ref["_xn"])     # bit-identical positions
    # Composited outputs, EVERY ray: 1e-4 relative (north_star).  (Round 1 needed a loose bound here: the
    # oracle's level scales were 1 ulp off the library's at levels 3/6/8/11, which put samples on those levels'
    # cell faces into the neighbouring cell — a different piecewise-constant normal.  Scales are now bit-exact,
    # tests/test_abi.py, and the measured worst ray of 16k was 5e-6.)
    for k in ("depth", "weight_sum", "normal", "depth_variance"):
        assert got[k].shape == ref[k].shape, k
        assert _rel(got[k], ref[k]) < 1e-4, (k, _rel(got[k], ref[k]))
    # colour passes through fp16 activations and an fp16 sigmoid output per sample (tcnn's contract): one fp16
    # rounding flip of one sample moves the composited colour by at most weight * 2^-11.  Bound: half an fp16 ulp
    # of a value in [0.5, 1) in absolute terms for every ray, 1e-4 relative for 99 % of the rays.
    assert got["color"].shape == ref["color"].shape
    cerr = np.abs(got["color"] - ref["color"]).max(1)
    assert cerr.max() < 2.5e-4, float(cerr.max())
    assert (cerr / max(np.abs(ref["color"]).max(), 1e-12) < 1e-4).mean() >= 0.99
    assert abs(float(got["gradient_error"][0]) - float(ref["gradient_error"][0])) < 2e-3 * abs(float(ref["gradient_error"][0]))


def test_neus_forward_vs_reference_golden():
    """tests/golden/neus.npz = the REFERENCE's own InstantNeuS.forward (src/InstantNeuS.py:295-370, imported from
    /root/reference by make_golden.py with only the tcnn modules restated): all 9 outputs, 1e-4 (colour: fp16 bound)."""
    from goslam_b200 import neus, synthetic
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "neus.npz"))
    offs, ress, _, total = neus.hashgrid_layout()
    w = synthetic.make_neus_weights(seed=int(g["weights_seed"]), total_grid_params=total, layout=(offs, ress))
    net = neus.InstantNeuS(synthetic.NEUS_CFG, g["bound"].tolist())
    with torch.no_grad():
        net.sdf_network.encoding.encoding.params.copy_(w["grid"])
        net.sdf_network.sdf_layer.weight.copy_(w["sdf_w"])
        net.sdf_network.sdf_layer.bias.copy_(w["sdf_b"])
        net.color_network._B.copy_(w["color_B"])
        net.color_network.network.params.copy_(w["mlp"])
    net = net.to(dev())
    net.update_bound(torch.from_numpy(g["rt_bound"]))
    with torch.no_grad():        # rendering runs under no_grad in the reference too; with grad enabled see test_gpu_neus_train.py
        out = net(*[torch.from_numpy(g[k]).to(dev()) for k in ("rays_o", "rays_d", "z_vals_in", "dists")])
    assert set(out.keys()) == set(k[4:] for k in g.files if k.startswith("out_"))
    for k, v in out.items():
        want = g["out_" + k]
        got = v.cpu().numpy().reshape(want.shape)
        if k == "color":
            assert np.abs(got - want).max() < 2.5e-4
        elif k == "sdf":
            inb = want != 100.0
            assert np.array_equal(inb, got != 100.0)
            assert np.abs(got[inb] - want[inb]).max() < 1e-4 * np.abs(want[inb]).max()
        elif k == "gradient_error":
            assert abs(float(got.reshape(-1)[0]) - float(want.reshape(-1)[0])) < 1e-4 * abs(float(want.reshape(-1)[0]))
        else:
            assert _rel(got, want) < 1e-4, (k, _rel(got, want))


# ------------------------------------------------------------------------------ z sampling
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["rgbd", "mono", "lindisp", "noperturb"])
def test_sample_z_matches_oracle(case, monkeypatch):
    """goslam_sample_z (one launch) == the eager restatement of src/render.py:99-171, bit for bit on
    z_vals (same linspace tables, same shared perturb_rand); the last dists column — a mean over
    n_samples copies of one number in the reference — to 1e-6."""
    from goslam_b200 import synthetic
    from goslam_b200.render import sample_z
    from oracle import render_oracle
    g = torch.Generator().manual_seed(31)
    R = 3000
    ro, rd, _, _ = synthetic.make_rays(R, S=72, seed=9)
    depth = 0.5 + 2.5 * torch.rand(R, generator=g)
    depth[::11] = 0.0                                   # no sensor reading
    ro[5::97] = torch.tensor([1.999, 0.0, 0.5])         # about to leave the box: far < near, the stratified
    rd[5::97] = torch.tensor([1.0, 0.0, 0.0])           # list is DEscending -> the general sort path
    ns, nf = (24, 48)
    if case == "mono":
        depth, ns, nf = None, 48, 24
    fixed = torch.rand(ns, generator=g)
    monkeypatch.setattr(torch, "rand", lambda n, device=None: fixed.to(device))
    bound = torch.tensor([[-2.0, 2.0], [-2.5, 1.5], [-1.0, 3.0]])
    kw = dict(perturb=0.0 if case == "noperturb" else 1.0, lindisp=case == "lindisp")
    z, d = sample_z(ro.to(dev()), rd.to(dev()), bound, None if depth is None else depth.to(dev()), ns, nf, **kw)
    zo, do = render_oracle.sample_z(ro.to(dev()), rd.to(dev()), bound, None if depth is None else depth.to(dev()),
                                    ns, nf, **kw)
    S = ns + (nf if depth is not None else 0)
    assert z.shape == (R, S) and d.shape == (R, S)
    # lindisp with a missing depth gives near = 0 -> inf/NaN samples, in the reference too: NaN == NaN here
    torch.testing.assert_close(z, zo, rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(d[:, :-1], do[:, :-1], rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(d[:, -1], do[:, -1], rtol=1e-6, atol=0, equal_nan=True)
    # and against the all-CPU run of the restatement (CPU linspace / CPU kernels)
    zc, dc = render_oracle.sample_z(ro, rd, bound, depth, ns, nf, **kw)
    torch.testing.assert_close(z.cpu(), zc, rtol=2e-6, atol=1e-7, equal_nan=True)


@pytest.mark.gpu
def test_sample_z_golden_from_reference_renderer(monkeypatch):
    """tests/golden/render_z.npz holds z_vals/dists captured from the reference's own
    Renderer.render_batch_ray (CPU, seed 1234)."""
    from goslam_b200.render import sample_z
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "render_z.npz"))
    torch.manual_seed(int(gold["torch_seed"]))
    fixed = torch.rand(24)                               # the reference's perturb_rand for that seed
    monkeypatch.setattr(torch, "rand", lambda n, device=None: fixed.to(device))
    bound = torch.tensor([[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]])
    z, d = sample_z(torch.from_numpy(gold["rays_o"]).to(dev()), torch.from_numpy(gold["rays_d"]).to(dev()), bound,
                    torch.from_numpy(gold["gt_depth"]).to(dev()), 24, 48, perturb=1.0, lindisp=False)
    np.testing.assert_allclose(z.cpu().numpy(), gold["z_vals"], rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(d.cpu().numpy(), gold["dists"], rtol=1e-4, atol=2e-6)


# ------------------------------------------------------------------------------ convex upsampling
@pytest.mark.parametrize("shape", [(2, 40, 80, 1), (1, 30, 40, 1), (2, 7, 45, 2), (1, 5, 33, 4)])
@pytest.mark.parametrize("mask_dtype", [torch.float32, torch.float16])
def test_cvx_upsample(shape, mask_dtype):
    """goslam_cvx_upsample == softmax/unfold/sum of src/droid_net.py:9-23 (oracle); 1e-6 relative: the
    9-term softmax and dot product are fp32 in both, only the summation order differs."""
    from goslam_b200 import droid_net
    from oracle import upsample_oracle
    b, ht, wd, dim = shape
    g = torch.Generator().manual_seed(b * 1000 + wd)
    data = torch.rand(b, ht, wd, dim, generator=g) + 0.1
    mask = (3.0 * torch.randn(b, 576, ht, wd, generator=g)).to(mask_dtype)
    out = droid_net.cvx_upsample(data.to(dev()), mask.to(dev()))
    ref = upsample_oracle.cvx_upsample(data, mask)
    assert out.shape == (b, 8 * ht, 8 * wd, dim)
    if mask_dtype == torch.float32:
        torch.testing.assert_close(out.cpu(), ref, rtol=2e-6, atol=2e-7)
    else:
        # torch.softmax(half) rounds the 9 weights to half: a 1-ulp fp32 difference before that
        # rounding can flip one weight by half an ulp (2^-11 relative) in a few of the 10^5 outputs
        diff = (out.cpu() - ref).abs()
        assert diff.max().item() <= 2.0 ** -11 * float(data.max()) * 1.01
        assert (diff > 2e-6).float().mean().item() < 5e-2
    if dim == 1:
        up = droid_net.upsample_disp(data[..., 0][None].to(dev()), mask[None].to(dev()))
        assert torch.equal(up[0], out[..., 0])


def test_cvx_upsample_golden_from_reference():
    from goslam_b200 import droid_net
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "cvx_upsample.npz"))
    for tag in ("disp", "flow"):
        data, mask = torch.from_numpy(gold[tag + "_data"]).to(dev()), torch.from_numpy(gold[tag + "_mask"]).to(dev())
        np.testing.assert_allclose(droid_net.cvx_upsample(data, mask).cpu().numpy(), gold[tag + "_out_f32"], rtol=2e-6, atol=2e-7)
        np.testing.assert_allclose(droid_net.cvx_upsample(data, mask.half()).cpu().numpy(), gold[tag + "_out_f16mask"],
                                   rtol=0, atol=2.0 ** -11 * 1.2)


# ------------------------------------------------------------------------------ graph bookkeeping
def _prox_case(rng, t0, t1, t, n_old, frac_big=0.1, ties=False):
    ilen, jlen = t - t0, t - t1
    dist = (rng.random(ilen * jlen) * 40).astype(np.float32)
    if ties:
        dist = np.round(dist)                               # many equal distances
    dist[rng.random(ilen * jlen) < frac_big] = 150.0
    old = rng.integers(0, t, size=(n_old, 2)).astype(np.int64)
    return dist, old


@pytest.mark.parametrize("case", [
    dict(t0=7, t1=0, t=12, rad=2, nms=2, thresh=16.0, maxf=48, stereo=False, n_old=6),
    dict(t0=0, t1=0, t=9, rad=2, nms=2, thresh=16.0, maxf=60, stereo=False, n_old=0),
    dict(t0=10, t1=3, t=22, rad=3, nms=1, thresh=20.0, maxf=40, stereo=True, n_old=9),
    dict(t0=4, t1=0, t=10, rad=2, nms=2, thresh=12.0, maxf=14, stereo=False, n_old=3),
    dict(t0=0, t1=0, t=120, rad=2, nms=2, thresh=16.0, maxf=1200, stereo=False, n_old=300),   # global-BA sized
    dict(t0=5, t1=9, t=30, rad=2, nms=2, thresh=25.0, maxf=200, stereo=True, n_old=20),       # t1 > t0: negative columns
    dict(t0=3, t1=0, t=14, rad=2, nms=3, thresh=30.0, maxf=-1, stereo=False, n_old=0),        # max_factors = -1
    dict(t0=2, t1=0, t=40, rad=1, nms=0, thresh=18.0, maxf=500, stereo=False, n_old=10, ties=True),
])
def test_proximity_edges_match_reference_loops(case):
    """goslam_proximity_edges == the reference's Python loops (oracle, itself pinned to the reference method):
    same edges in the same order — edge-index parity, bit-exact."""
    from goslam_b200 import graph
    from oracle import graph_oracle
    c = dict(case)
    rng = np.random.default_rng(c["t"] * 31 + c["t0"])
    dist, old = _prox_case(rng, c["t0"], c["t1"], c["t"], c["n_old"], ties=c.pop("ties", False))
    want = graph_oracle.proximity_edges(dist, c["t0"], c["t1"], c["t"], c["rad"], c["nms"], c["thresh"], c["maxf"],
                                        c["stereo"], old[:, 0], old[:, 1])
    ii, jj = graph.proximity_edges(torch.from_numpy(dist).to(dev()), c["t0"], c["t1"], c["t"], c["rad"], c["nms"],
                                   c["thresh"], c["maxf"], c["stereo"], torch.from_numpy(old[:, 0]).to(dev()),
                                   torch.from_numpy(old[:, 1]).to(dev()))
    got = torch.stack([ii, jj], 1).cpu().numpy()
    np.testing.assert_array_equal(got, want)


def test_proximity_edges_golden_from_reference_method():
    from goslam_b200 import graph
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "proximity.npz"))
    for n in range(int(g["n_cases"])):
        t0, t1, t, rad, nms, maxf, st = [int(x) for x in g["c%d_params" % n]]
        old = g["c%d_old" % n]
        ii, jj = graph.proximity_edges(torch.from_numpy(g["c%d_dist" % n]).to(dev()), t0, t1, t, rad, nms,
                                       float(g["c%d_thresh" % n]), maxf, bool(st),
                                       torch.from_numpy(old[:, 0].copy()).to(dev()), torch.from_numpy(old[:, 1].copy()).to(dev()))
        np.testing.assert_array_equal(torch.stack([ii, jj], 1).cpu().numpy(), g["c%d_es" % n])


def test_backend_edges_golden_and_oracle():
    """Backend.ba's edge selection (dense and loop-closure modes): device == the reference method (golden) == the oracle,
    including the early return with fewer than 3 edges."""
    from goslam_b200 import graph
    from oracle import graph_oracle
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "backend_edges.npz"))
    for n in range(int(g["n_cases"])):
        ts, te, rad, nms, maxf, st, tsl, loop = [int(x) for x in g["b%d_params" % n]]
        got = graph.backend_edges(torch.from_numpy(g["b%d_dist" % n]).to(dev()), ts, te, rad, nms,
                                  float(g["b%d_thresh" % n]), maxf, bool(st), None if tsl < 0 else tsl, bool(loop))
        if int(g["b%d_early" % n]):
            assert got is None
        else:
            np.testing.assert_array_equal(torch.stack(got, 1).cpu().numpy(), g["b%d_es" % n])
    rng = np.random.default_rng(8)
    dist = (rng.random(90 * 90) * 50).astype(np.float32)
    want = graph_oracle.backend_edges(dist, 10, 100, 2, 2, 22.0, 700, False)
    got = graph.backend_edges(torch.from_numpy(dist).to(dev()), 10, 100, 2, 2, 22.0, 700, False)
    np.testing.assert_array_equal(torch.stack(got, 1).cpu().numpy(), want)
    assert graph.backend_edges(torch.from_numpy(dist[:1]).to(dev()), 4, 5, 2, 2, 22.0, 10, False) is None
    # loop-closure mode on a larger smooth field
    ilen, jlen = 60, 100
    field = (rng.random((ilen, jlen)) * 8 + 30.0 * np.abs(np.sin(np.arange(ilen)[:, None] * 0.3 + np.arange(jlen)[None] * 0.2))).astype(np.float32)
    want = graph_oracle.backend_edges(field.reshape(-1), 0, 100, 2, 2, 20.0, 900, False, 40, True)
    got = graph.backend_edges(torch.from_numpy(field.reshape(-1)).to(dev()), 0, 100, 2, 2, 20.0, 900, False, 40, True)
    np.testing.assert_array_equal(torch.stack(got, 1).cpu().numpy(), want)


# ------------------------------------------------------------------------------ degenerate inputs
def test_degenerate_inputs_do_not_crash():
    """empty edge lists / ray batches and all-masked graphs go through every entry point cleanly."""
    from goslam_b200 import droid_backends, graph, render
    from goslam_b200.modules import CorrBlock
    from goslam_b200.modules.corr import CorrPool, fmaps_to_kmajor
    sc, targets, weights, eta = _ba_case(num_kf=5, ht=9, wd=13, rgbd=True)
    e = torch.zeros(0, dtype=torch.long, device=dev())
    poses, disps = sc["poses"].clone().to(dev()), sc["disps"].clone().to(dev())
    # BA with no edges: the damped system is diagonal with a zero right-hand side -> zero pose step, and the
    # depth update is the pure sensor-prior step
    dx, dz, status = droid_backends.ba(poses, disps, sc["intrinsics"][0].to(dev()).contiguous(), sc["disps_sens"].to(dev()),
                                       torch.zeros(0, 2, 9, 13, device=dev()), torch.zeros(0, 2, 9, 13, device=dev()),
                                       eta[:4].to(dev()).contiguous(), e, e, 1, 5, 2, 1e-4, 0.1, False, return_status=True)
    assert status.cpu().tolist() == [0, 0] and float(dx.abs().max()) == 0.0
    assert torch.equal(poses.cpu(), sc["poses"]) and torch.isfinite(disps).all()
    # correlation: empty blocks
    fm = torch.randn(3, 1, 128, 16, 16).half().to(dev())
    km = fmaps_to_kmajor(fm)
    pool = CorrPool(4, 16, 16, device=dev())
    blk = CorrBlock.from_video(km, e, e, 16, 16, pool=pool)
    assert blk(torch.zeros(1, 0, 16, 16, 2, device=dev())).shape == (1, 0, 196, 16, 16) and pool.free_slots == 4
    assert droid_backends.frame_distance(poses, disps, sc["intrinsics"][0].to(dev()).contiguous(), e, e, 0.3).numel() == 0
    # renderer: empty ray batch
    z, d = render.sample_z(torch.zeros(0, 3, device=dev()), torch.zeros(0, 3, device=dev()),
                           torch.tensor([[-1.0, 1.0]] * 3), torch.zeros(0, device=dev()), 24, 48)
    assert z.shape == (0, 72) and d.shape == (0, 72)
    # graph: nothing below the threshold -> only the local-window edges
    ii, jj = graph.proximity_edges(torch.full((36,), 1e9, device=dev()), 0, 0, 6, 2, 2, 16.0, 48, False, e, e)
    assert ii.numel() == graph.local_edge_count(0, 6, 2, False)
