"""The tiled correlation build over a whole update window: 36 edges, so every CTA of the persistent kernel runs
many work items in a row and the double-buffered band staging (levels 2 and 3) cycles through its buffers many
times.  The row-major instance does the same arithmetic with its own write-out, so the two layouts must give the
same pyramid bit for bit; a few edges are also checked against the CPU oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import corr_oracle  # noqa: E402


@pytest.mark.parametrize("hw", [(40, 80), (60, 80)])
def test_tiled_window_build_matches_rowmajor(hw):
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
    pyr = {}
    for layout in ("tiled", "rowmajor"):
        pool = CorrPool(N + 3, h, w, device=dev, layout=layout)
        pool.alloc(3)                                   # edges do not start at slot 0
        if layout == "tiled":
            for lvl in pool.levels:
                lvl.fill_(float("nan"))                 # padding the build fails to write shows up below
        blk = CorrBlock.from_video(km, ii.to(dev), jj.to(dev), h, w, pool=pool)
        pyr[layout] = blk.gather_pyramid()
        if layout == "tiled":
            # each level-2 piece is written whole, its padding as zeros
            n_yb, n_xb = (h + 7) // 8, (w + 15) // 16
            raw = pool.levels[2][blk.slots.long()].view(N, h * w, n_yb, -1)
            n_bands = ((h >> 2) + 1) // 2
            assert torch.equal(raw[:, :, :n_bands, 2 * n_xb * 4:].float().cpu(),
                               torch.zeros_like(raw[:, :, :n_bands, 2 * n_xb * 4:].float().cpu()))
    for i, (a, b) in enumerate(zip(pyr["tiled"], pyr["rowmajor"])):
        assert torch.equal(a, b), "level %d" % i
    want = corr_oracle.corr_build(fmaps[ii[-2:], 0], fmaps[jj[-2:], 0], 4)
    for i, (got, ref) in enumerate(zip(pyr["tiled"], want)):
        got = got[-2:].float().cpu().numpy()
        np.testing.assert_allclose(got, ref.float().numpy(), rtol=1.5e-3, atol=1e-3, err_msg="level %d" % i)
