"""The correlation build over a whole update window: 36 edges, so every CTA of the persistent kernel runs
many work items in a row and the double-buffered band staging (levels 2 and 3) cycles through its buffers many
times.  A one-edge build runs few items per CTA (40x80: 125 items, at most one per CTA on 132 SMs), and the
items of an edge do the same arithmetic whatever CTA runs them, so the window build must equal 36 one-edge
builds of the same pairs bit for bit; every edge is also checked against the CPU oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import corr_oracle  # noqa: E402


@pytest.mark.parametrize("hw", [(40, 80), (60, 80)])
def test_window_build_matches_one_edge_builds(hw):
    from goslam_b200.modules import CorrBlock
    from goslam_b200.modules.corr import CorrPool, fmaps_to_kmajor
    h, w = hw
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(300 + h)
    fmaps = torch.randn(8, 1, 128, h, w, generator=g).half()
    N = 36
    ii = torch.arange(N) % 8
    jj = (torch.arange(N) * 3 + 1) % 8
    km = fmaps_to_kmajor(fmaps.to(dev))
    pool = CorrPool(N + 3, h, w, device=dev)
    pool.alloc(3)                                       # edges do not start at slot 0
    for lvl in pool.levels:
        lvl.fill_(float("nan"))                         # padding the build fails to write shows up below
    blk = CorrBlock.from_video(km, ii.to(dev), jj.to(dev), h, w, pool=pool)
    pyr = blk.gather_pyramid()
    # each level-2 piece is written whole, its padding as zeros
    n_yb, n_xb = (h + 7) // 8, (w + 15) // 16
    raw = pool.levels[2][blk.slots.long()].view(N, h * w, n_yb, -1)
    n_bands = ((h >> 2) + 1) // 2
    assert torch.equal(raw[:, :, :n_bands, 2 * n_xb * 4:].float().cpu(),
                       torch.zeros_like(raw[:, :, :n_bands, 2 * n_xb * 4:].float().cpu()))
    for e in range(N):
        one = CorrBlock.from_video(km, ii[e:e + 1].to(dev), jj[e:e + 1].to(dev), h, w)
        for i, (a, b) in enumerate(zip(pyr, one.gather_pyramid())):
            assert torch.equal(a[e:e + 1], b), "edge %d level %d" % (e, i)
    for e0 in range(0, N, 6):                           # the CPU oracle in chunks of 6 edges (memory)
        want = corr_oracle.corr_build(fmaps[ii[e0:e0 + 6], 0], fmaps[jj[e0:e0 + 6], 0], 4)
        for i, (got, ref) in enumerate(zip(pyr, want)):
            np.testing.assert_allclose(got[e0:e0 + 6].float().cpu().numpy(), ref.float().numpy(), rtol=1.5e-3,
                                       atol=1e-3, err_msg="edges %d.. level %d" % (e0, i))
