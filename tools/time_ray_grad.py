"""Time the renderer's forward + backward with and without ray gradients at the mapping batch shapes bench.py uses
(2^16 and 2^12 rays x 72 samples, the mapping loss of src/mapping.py:97-128), alternating the two variants, and print
the card's name and power limit beside the numbers.  Each sample is one event pair around 20 (2^16 rays) or 100
(2^12 rays) calls.  Run on the GPU:  python tools/time_ray_grad.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_ray_grad.py")
import torch  # noqa: E402

import bench  # noqa: E402
from goslam_b200 import parallel, synthetic  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    net, _, _ = bench.make_renderer(dev, 43)
    measure.emit({})
    for R in (1 << 16, 1 << 12):
        ro, rd, zv, ds = [t.to(dev) for t in synthetic.make_rays(R, S=bench.SAMPLES, seed=47)]
        g = torch.Generator().manual_seed(5)
        rc = torch.rand(R, 3, generator=g).to(dev)
        depth = (0.5 + 2.5 * torch.rand(R, 1, generator=g)).to(dev)

        def fwd_bwd(rays_grad):
            for p in net.parameters():
                p.grad = None
            o_, d_ = (ro.clone().requires_grad_(True), rd.clone().requires_grad_(True)) if rays_grad else (ro, rd)
            with torch.enable_grad():
                o = net(o_, d_, zv, ds)
                total = parallel.mapping_loss_local(net, o, rc, depth, R, 2.0, 2.0, 0.1)
            total.backward()

        for v in (False, True):                            # warm-up of both shapes and paths
            for _ in range(3):
                fwd_bwd(v)
        torch.cuda.synchronize()
        n = 20 if R > 4096 else 100
        res = {False: [], True: []}
        for _ in range(5):                                 # alternate: the two variants see the same machine state
            for v in (False, True):
                res[v] += measure.cuda_time(lambda: fwd_bwd(v), 1, warmup=0, batch=n)["samples_ms"]
        med = {v: sorted(x)[len(x) // 2] for v, x in res.items()}
        print("R=%6d S=%d  forward+backward  params only %.3f ms (%.3f-%.3f)  + rays %.3f ms (%.3f-%.3f)  extra %.3f ms (%.1f %%)" % (
            R, bench.SAMPLES, med[False], min(res[False]), max(res[False]), med[True], min(res[True]), max(res[True]),
            med[True] - med[False], 100.0 * (med[True] - med[False]) / med[False]))


if __name__ == "__main__":
    main()
