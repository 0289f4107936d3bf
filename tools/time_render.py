"""in-stream timing of the renderer pieces: z-sampling kernel, marcher on bench rays vs sampled rays.  CUDA events
around 10 back-to-back calls (5 for the eager oracle), 5 samples.  usage: python tools/time_render.py"""
import os, sys, time, types
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_render.py")
import torch  # noqa: E402
torch.set_grad_enabled(False)      # inference tools
import bench  # noqa: E402
from goslam_b200 import render as render_mod  # noqa: E402

dev = torch.device("cuda:0")
net, rays, _ = bench.make_renderer(dev, 43)
rd = [r.to(dev) for r in rays]
R = rd[0].shape[0]
gt = (0.5 + 2.5 * torch.rand(R, generator=torch.Generator().manual_seed(43))).to(dev)


def t(fn, n=10):
    r = measure.cuda_time(fn, reps=5, batch=n)
    return "%8.3f ms (%.3f-%.3f)" % (r["median_ms"], r["min_ms"], r["max_ms"])


S = rd[2].shape[1]
measure.emit({})
print("marcher, bench rays            %s" % t(lambda: net(*rd)))
print("sample_z kernel (24+48)        %s" % t(lambda: render_mod.sample_z(rd[0], rd[1], net.bound, gt, 24, S - 24)))
z, d = render_mod.sample_z(rd[0], rd[1], net.bound, gt, 24, S - 24)
print("marcher, sampled z             %s" % t(lambda: net(rd[0], rd[1], z, d)))
print("z stats: bench z [%.3f, %.3f] mean %.3f; sampled z [%.3f, %.3f] mean %.3f" % (
    rd[2].min().item(), rd[2].max().item(), rd[2].mean().item(), z.min().item(), z.max().item(), z.mean().item()))
print("dists:   bench mean %.4f; sampled mean %.4f" % (rd[3].mean().item(), d.mean().item()))
from oracle import render_oracle
print("eager torch sample_z (oracle)  %s" % t(lambda: render_oracle.sample_z(rd[0], rd[1], net.bound, gt, 24, S - 24), n=5))

# ---- end-to-end pieces, as bench.py's render_e2e does them ----
rcfg = {"rendering": {"lindisp": False, "perturb": 1.0, "N_samples": 24, "N_surface": S - 24}}
renderer = render_mod.Renderer(rcfg, None, types.SimpleNamespace(H=512, W=512, fx=460.8, fy=460.8, cx=256.0, cy=256.0))
gth = (0.5 + 2.5 * torch.rand(R, generator=torch.Generator().manual_seed(43)))
hp = [rays[0].pin_memory(), rays[1].pin_memory(), gth.pin_memory()]
keep = {}
pinned_out = {k: torch.empty((R, 3 if k == "color" else 1), dtype=torch.float32).pin_memory() for k in ("color", "depth")}


def e2e(h2d=True, d2h="pageable"):
    ro, rdir, gd = [x.to(dev, non_blocking=True) for x in hp] if h2d else (rd[0], rd[1], gt)
    out = renderer.render_batch_ray(ro, rdir, net, None, device=dev, gt_depth=gd)
    for k in ("color", "depth"):
        if d2h == "pageable":
            keep[k] = out[k].to("cpu", non_blocking=True)
        elif d2h == "pinned":
            pinned_out[k].copy_(out[k].reshape(pinned_out[k].shape), non_blocking=True)


print("e2e full (pageable d2h)        %s" % t(lambda: e2e()))
print("e2e pinned d2h                 %s" % t(lambda: e2e(d2h="pinned")))
print("e2e no d2h                     %s" % t(lambda: e2e(d2h=None)))
print("e2e no h2d, no d2h             %s" % t(lambda: e2e(h2d=False, d2h=None)))
# the enqueue cost: a host clock read before the device drains, which no timer in measure does
torch.cuda.synchronize(); t0 = time.perf_counter()
for _ in range(5):
    e2e(h2d=False, d2h=None)
t1 = time.perf_counter(); torch.cuda.synchronize(); t2 = time.perf_counter()
print("host time per call %.3f ms, drained after %.3f ms" % ((t1 - t0) / 5 * 1e3, (t2 - t0) / 5 * 1e3))
