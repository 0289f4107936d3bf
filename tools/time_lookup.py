"""pooled 4-level lookup time per shape (36 edges), CUDA events around 20 back-to-back lookups, 5 samples:
python tools/time_lookup.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_lookup.py")
import torch  # noqa: E402
from goslam_b200.modules import CorrBlock  # noqa: E402
from goslam_b200.modules.corr import CorrPool, fmaps_to_kmajor  # noqa: E402
dev = torch.device("cuda:0")
measure.emit({})
for (h, w, rig) in ((40, 80, 1), (40, 60, 1), (40, 60, 2), (48, 64, 1), (60, 80, 1), (30, 40, 1)):
    g = torch.Generator().manual_seed(0)
    fm = torch.randn(8, rig, 128, h, w, generator=g).half().to(dev)
    km = fmaps_to_kmajor(fm)
    N = 36
    ii = (torch.arange(N) % 8).to(dev)
    jj = ((torch.arange(N) * 3 + 1) % 8).to(dev)
    pool = CorrPool(N, h, w, device=dev)
    blk = CorrBlock.from_video(km, ii, jj, h, w, rig=rig, pool=pool)
    gx, gy = torch.meshgrid(torch.arange(w), torch.arange(h), indexing="xy")
    for name, off in (("identity+1.7", 1.7), ("random", None)):
        if off is None:
            coords = torch.stack([torch.rand(N, h, w, generator=g) * w, torch.rand(N, h, w, generator=g) * h], dim=-1)[None].to(dev)
        else:
            coords = (torch.stack([gx, gy], dim=-1).float()[None, None].expand(1, N, h, w, 2) + off).contiguous().to(dev)
        t = measure.cuda_time(lambda: blk(coords), reps=5, batch=20)
        print("%dx%d rig %d %-13s lookup %7.1f us (%.1f-%.1f)" % (h, w, rig, name, 1e3 * t["median_ms"], 1e3 * t["min_ms"],
                                                                  1e3 * t["max_ms"]), flush=True)
