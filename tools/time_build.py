"""time the correlation build for several edge counts (L2-resident vs DRAM-streaming outputs).
usage: time_build.py [h w]   (default 40 80)"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
if os.environ.get("TOOL_VARIANT"):            # an A/B build made by tools/build_variant.py
    from tools.build_variant import use_variant
    use_variant(os.environ["TOOL_VARIANT"])
from goslam_b200.modules import CorrBlock
from goslam_b200.modules.corr import CorrPool, fmaps_to_kmajor
dev = torch.device("cuda:0")
h, w = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (40, 80)
g = torch.Generator().manual_seed(0)
fm = torch.randn(16, 1, 128, h, w, generator=g).half().to(dev)
km = fmaps_to_kmajor(fm)
for N in ((36,) if os.environ.get("TOOL_VARIANT") else (2, 36, 72)):
    ii = torch.arange(N, device=dev) % 16
    jj = (torch.arange(N, device=dev) * 7 + 3) % 16
    pool = CorrPool(N, h, w, device=dev)

    def run():
        c = CorrBlock.from_video(km, ii, jj, h, w, pool=pool)
        c.free()
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        run()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    lvl = sum((h >> i) * (w >> i) for i in range(4))
    gb = N * h * w * lvl * 2 / 1e9
    print(f"{h}x{w} {'build':8s} N={N:3d} {ms*1e3:8.1f} us  {ms*1e3/N:7.2f} us/edge  out={gb*1e3:7.1f} MB (algorithmic)  {gb/ms*1e3:7.1f} GB/s")
    # the card's write ceiling beside it: a plain device fill of the same byte count
    buf = torch.empty(int(gb * 1e9) // 2, dtype=torch.half, device=dev)
    for _ in range(3):
        buf.zero_()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(20):
        buf.zero_()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    print(f"{h}x{w} {'fill':8s} N={N:3d} {ms*1e3:8.1f} us  {'':20s}out={gb*1e3:7.1f} MB  {gb/ms*1e3:7.1f} GB/s")
    del buf
