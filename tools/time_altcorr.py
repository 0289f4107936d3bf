"""AltCorrBlock at 384 edges, 30x40, 4 levels: CUDA events around 5 back-to-back calls, 5 samples.
usage: python tools/time_altcorr.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_altcorr.py")
import torch  # noqa: E402
from goslam_b200.modules import AltCorrBlock  # noqa: E402
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
F, H, W, N = 66, 30, 40, 384
fm = torch.randn(1, F, 128, H, W, generator=g).half().to(dev)
blk = AltCorrBlock(fm)
ii = torch.randint(0, 64, (N,), generator=g).to(dev)
jj = torch.randint(0, 64, (N,), generator=g).to(dev)
base = torch.stack(torch.meshgrid(torch.arange(W).float(), torch.arange(H).float(), indexing="xy"), -1)
coords = (base[None, None].repeat(1, N, 1, 1, 1) + 2 * torch.randn(1, N, H, W, 2, generator=g)).to(dev)
measure.emit({})
t = measure.cuda_time(lambda: blk(coords, ii, jj), reps=5, warmup=2, batch=5)
print("AltCorrBlock(384 edges, 30x40, 4 levels): %.3f ms (%.3f-%.3f)  (%.1f GFLOP/s fp32 useful)" % (
    t["median_ms"], t["min_ms"], t["max_ms"], N * H * W * 65536 / t["median_ms"] / 1e6), blk(coords, ii, jj).shape)
