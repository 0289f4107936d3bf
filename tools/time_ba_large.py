"""CUDA-event timing of droid_backends.ba on global-BA-sized systems (config 4: 64 kf, 30x40, ~384 edges,
P = 63) and of its phases through the split entry points: 5 samples of 20 back-to-back calls.
usage: python tools/time_ba_large.py [num_kf ht wd]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_ba_large.py")
import torch  # noqa: E402
from goslam_b200 import droid_backends, parallel, synthetic  # noqa: E402

dev = torch.device("cuda:0")
num_kf, ht, wd = (int(a) for a in sys.argv[1:4]) if len(sys.argv) >= 4 else (64, 30, 40)
sc, g = synthetic.make_scene(num_kf=num_kf, ht=ht, wd=wd, rgbd=True, seed=43, with_fmaps=False, buffer=num_kf + 2)
sc["t0"], sc["t1"] = 1, num_kf
coords = synthetic.true_reprojection(sc)
tg, wg, eta = synthetic.make_update(sc, coords[0], g, noise=0.7)
D = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in sc.items()}
tg, wg, eta = tg.to(dev), wg.to(dev), eta.to(dev)
intr = D["intrinsics"][0].contiguous()
p0, d0 = D["poses"].clone(), D["disps"].clone()


def t(fn):
    r = measure.cuda_time(fn, reps=5, warmup=3, batch=20)
    return "%9.1f us (%.1f-%.1f)" % (1e3 * r["median_ms"], 1e3 * r["min_ms"], 1e3 * r["max_ms"])


def ba(iters, motion_only=False):
    D["poses"].copy_(p0); D["disps"].copy_(d0)
    droid_backends.ba(D["poses"], D["disps"], intr, D["disps_sens"], tg, wg, eta, D["ii"], D["jj"], 1, num_kf, iters,
                      1e-5, 1e-2, motion_only)


measure.emit({})
print("edges %d, P %d, 6P %d, %dx%d" % (D["ii"].numel(), num_kf - 1, 6 * (num_kf - 1), ht, wd))
for it in (1, 2):
    print("ba iters=%d              %s" % (it, t(lambda: ba(it))))
print("ba motion_only iters=2   %s" % t(lambda: ba(2, True)))
num = D["disps"].shape[0]
kx = torch.unique(torch.cat([torch.arange(1, num_kf, device=dev), D["ii"]]))
eta_f = torch.zeros(num, ht, wd, device=dev)
eta_f[kx] = eta
be = parallel.CudaBackend(D["poses"], D["disps"], intr, D["disps_sens"], 1, num_kf)
sysm = be.phase1(tg, wg, eta_f, D["ii"], D["jj"], False)
print("phase1 (prep+lin+system) %s" % t(lambda: be.phase1(tg, wg, eta_f, D["ii"], D["jj"], False)))


def p2():
    D["poses"].copy_(p0); D["disps"].copy_(d0)
    be.phase2(sysm, 1e-5, 1e-2, False, 0, num)


print("phase2 (solve+backsub)   %s" % t(p2))
