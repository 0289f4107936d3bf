"""GPU parity of the wgmma correlation build + pooled lookup on EVERY shape BASELINE.json names
(SURVEY §8 head: cfg1 48x64, Replica 40x80, ScanNet 30x40, EuRoC 40x60 stereo, 640x480 -> 60x80)
against the CPU oracle — not only against the SIMT twin.  The irregular ones are what matters:
40x60 has w % 16 != 0 (ragged x-tile + padded tiles), 60x80 has h % 8 == 4 (ragged last band)
and 4800 / 128 = 37.5 (ragged last m-tile), 48x64 is the one CPU-shaped config."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import corr_oracle  # noqa: E402

SHAPES = [(48, 64), (40, 80), (30, 40), (40, 60), (60, 80)]


def dev():
    return torch.device("cuda:0")


def _coords(N, h, w, g):
    base = torch.stack(torch.meshgrid(torch.arange(w).float(), torch.arange(h).float(), indexing="xy"), -1)
    c = base[None, None].repeat(1, N, 1, 1, 1) + 3.0 * torch.randn(1, N, h, w, 2, generator=g)
    c[0, :, 0, :3] = torch.tensor([-5.5, 2.25])                  # windows hanging over every border
    c[0, :, 1, :3] = torch.tensor([w + 1.5, h - 2.0])
    c[0, :, 2, :3] = torch.tensor([w / 2.0, -3.75])
    c[0, :, 3, :3] = torch.tensor([w - 1.0, h - 1.0])            # integer coordinates at the last pixel
    return c


def _check_pyramid(got_levels, want_levels):
    for i, (got, want) in enumerate(zip(got_levels, want_levels)):
        got = got.float().cpu().numpy()
        want = want.float().numpy()
        assert got.shape == want.shape, (i, got.shape, want.shape)
        # fp32 accumulation in a different order, one rounding to half per level: <= 1 half-ulp,
        # and identical almost everywhere
        np.testing.assert_allclose(got, want, rtol=1.5e-3, atol=1e-3, err_msg="level %d" % i)
        assert (got == want).mean() > 0.97, (i, (got == want).mean())


@pytest.mark.parametrize("hw", SHAPES)
def test_corr_block_build_vs_oracle(hw):
    """CorrBlock(fmap1, fmap2) — the tensor-core build into a private pool — and the fused lookup on
    it, against the oracle (bit-exact for the half-precision lookup)."""
    from goslam_b200.modules import CorrBlock
    h, w = hw
    N = 2
    g = torch.Generator().manual_seed(100 + h)
    f1 = torch.randn(1, N, 128, h, w, generator=g).half()
    f2 = torch.randn(1, N, 128, h, w, generator=g).half()
    blk = CorrBlock(f1.to(dev()), f2.to(dev()))
    _check_pyramid(blk.corr_pyramid, corr_oracle.corr_build(f1[0], f2[0], 4))
    coords = _coords(N, h, w, g)
    out = blk(coords.to(dev()))
    want = corr_oracle.corr_pyramid_lookup([p.cpu().numpy() for p in blk.corr_pyramid], coords[0].numpy(), 3)
    np.testing.assert_array_equal(out[0].cpu().numpy().astype(np.float32), want.astype(np.float32))


@pytest.mark.parametrize("num_levels", [4, 1])
@pytest.mark.parametrize("hw,rig", [((48, 64), 1), ((40, 80), 1), ((30, 40), 1), ((40, 60), 2), ((60, 80), 1)])
def test_pool_build_and_lookup_vs_oracle(hw, rig, num_levels):
    """FactorGraph's path: video-level K-major maps -> pooled tensor-core build -> pooled lookup of every
    level; stereo rigs use the right image for self-edges (src/factor_graph.py:108-111).  num_levels = 1
    leaves the stores of levels 1-3 out of the build."""
    from goslam_b200.modules import CorrBlock
    from goslam_b200.modules.corr import CorrPool, fmaps_to_kmajor
    h, w = hw
    g = torch.Generator().manual_seed(200 + h + rig)
    fmaps = torch.randn(4, rig, 128, h, w, generator=g).half()
    if rig == 2:
        ii = torch.tensor([0, 1, 2, 3, 1])
        jj = torch.tensor([1, 0, 2, 1, 1])            # (2,2) and (1,1) are stereo self-edges
    else:
        ii = torch.tensor([0, 1, 3])
        jj = torch.tensor([1, 0, 2])
    N = ii.numel()
    c = (ii == jj).long() if rig == 2 else torch.zeros_like(ii)
    want_pyr = corr_oracle.corr_build(fmaps[ii, 0], fmaps[jj, c], num_levels)
    km = fmaps_to_kmajor(fmaps.to(dev()))
    pool = CorrPool(N + 3, h, w, num_levels, device=dev())
    pool.alloc(2)                                       # edges do not start at slot 0
    blk = CorrBlock.from_video(km, ii.to(dev()), jj.to(dev()), h, w, rig=rig, num_levels=num_levels, pool=pool)
    got_pyr = blk.gather_pyramid()
    assert len(got_pyr) == num_levels
    _check_pyramid(got_pyr, want_pyr)
    coords = _coords(N, h, w, g)
    out = blk(coords.to(dev()))
    want = corr_oracle.corr_pyramid_lookup([p.cpu().numpy() for p in got_pyr], coords[0].numpy(), 3)
    np.testing.assert_array_equal(out[0].cpu().numpy().astype(np.float32), want.astype(np.float32))


@pytest.mark.parametrize("hw", SHAPES)
def test_corr_level0_vs_oracle(hw):
    """CorrBlock.corr (level 0 only): the tensor-core build with one level."""
    from goslam_b200.modules import CorrBlock
    h, w = hw
    g = torch.Generator().manual_seed(400 + h)
    f1 = torch.randn(1, 2, 128, h, w, generator=g).half()
    f2 = torch.randn(1, 2, 128, h, w, generator=g).half()
    got = CorrBlock.corr(f1.to(dev()), f2.to(dev()))
    assert got.shape == (1, 2, h, w, h, w)
    _check_pyramid([got[0]], corr_oracle.corr_build(f1[0], f2[0], 1))


def test_cat_of_two_private_pool_blocks():
    """the reference's cat for any two blocks: two CorrBlock(f1, f2) live in different private pools, and
    their cat holds both pyramids, edge order kept, and looks up like one block built from all edges."""
    from goslam_b200.modules import CorrBlock
    h, w = 40, 60
    g = torch.Generator().manual_seed(500)
    f1 = torch.randn(1, 5, 128, h, w, generator=g).half().to(dev())
    f2 = torch.randn(1, 5, 128, h, w, generator=g).half().to(dev())
    a = CorrBlock(f1[:, :2], f2[:, :2])
    b = CorrBlock(f1[:, 2:], f2[:, 2:])
    want = [torch.cat([x, y]) for x, y in zip(a.corr_pyramid, b.corr_pyramid)]
    whole = CorrBlock(f1, f2)
    ab = a.cat(b)
    assert ab is a and a.pool is not b.pool and len(a._slots_host) == 5
    for x, y, z in zip(ab.corr_pyramid, want, whole.corr_pyramid):
        assert torch.equal(x, y) and torch.equal(x, z)
    coords = _coords(5, h, w, g).to(dev())
    assert torch.equal(ab(coords), whole(coords))
    assert len(b._slots_host) == 3                      # `b` keeps its own edges
