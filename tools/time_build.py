"""time the correlation build for several edge counts (L2-resident vs DRAM-streaming outputs), and for the
benchmark's |i - j| <= 3 window, whose 36 edges are 18 reverse pairs that store level 0 once per pair.
"written" is what the build stores (a reader edge's level 0 is its partner's, transposed), "algorithmic" what
the same edges would store unpaired; the rate is over the written bytes.  CUDA events around 20 back-to-back builds,
5 samples.
usage: time_build.py [h w]   (default 40 80)"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_build.py")
import torch  # noqa: E402
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
measure.emit({})


def readers(ii, jj):
    """edges whose level 0 the build does not store: the later edge of a reverse pair (CorrPool)"""
    e = list(zip(ii.tolist(), jj.tolist()))
    return sum(1 for r, (a, b) in enumerate(e)
               if a != b and e.count((a, b)) == 1 and e.count((b, a)) == 1 and e.index((b, a)) < r)


fwd = [(i, j) for i in range(8) for j in range(8) if 0 < j - i <= 3]
window = (torch.tensor([i for i, _ in fwd] + [j for _, j in fwd]), torch.tensor([j for _, j in fwd] + [i for i, _ in fwd]))
cases = [("no pairs", N, torch.arange(N) % 16, (torch.arange(N) * 7 + 3) % 16) for N in
         ((36,) if os.environ.get("TOOL_VARIANT") else (2, 36, 72))] + [("window", 36) + window]
for tag, N, ii, jj in cases:
    n_rd = readers(ii, jj)
    ii, jj = ii.to(dev), jj.to(dev)
    pool = CorrPool(N, h, w, device=dev)

    def run():
        c = CorrBlock.from_video(km, ii, jj, h, w, pool=pool)
        c.free()
    t = measure.cuda_time(run, reps=5, batch=20)
    ms = t["median_ms"]
    lvl = sum((h >> i) * (w >> i) for i in range(4))
    alg = N * h * w * lvl * 2 / 1e9
    gb = alg - n_rd * (h * w) ** 2 * 2 / 1e9
    print(f"{h}x{w} {'build':8s} N={N:3d} {ms*1e3:8.1f} us  {ms*1e3/N:7.2f} us/edge  out={gb*1e3:7.1f} MB written "
          f"({alg*1e3:.1f} MB algorithmic, {tag}: {n_rd} readers)  {gb/ms*1e3:7.1f} GB/s  "
          f"({t['min_ms']*1e3:.1f}-{t['max_ms']*1e3:.1f} us)")
    # the card's write ceiling beside it: a plain device fill of the same byte count
    buf = torch.empty(int(gb * 1e9) // 2, dtype=torch.half, device=dev)
    t = measure.cuda_time(buf.zero_, reps=5, batch=20)
    ms = t["median_ms"]
    print(f"{h}x{w} {'fill':8s} N={N:3d} {ms*1e3:8.1f} us  {'':20s}out={gb*1e3:7.1f} MB  {gb/ms*1e3:7.1f} GB/s  "
          f"({t['min_ms']*1e3:.1f}-{t['max_ms']*1e3:.1f} us)")
    del buf
