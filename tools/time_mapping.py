"""kernel-level breakdown of one mapping iteration (forward under grad + loss + backward + AdamW): device us per
iteration by kernel name, from one profiler pass (measure.kernel_times) over 3 iterations.
usage: time_mapping.py [log2_rays]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_mapping.py")
import torch  # noqa: E402
import bench  # noqa: E402
from goslam_b200 import synthetic  # noqa: E402

dev = torch.device("cuda:0")
R = 1 << (int(sys.argv[1]) if len(sys.argv) > 1 else 16)
net, _, _ = bench.make_renderer(dev, 43)
ro, rd, zv, ds = [t.to(dev) for t in synthetic.make_rays(R, S=bench.SAMPLES, seed=47)]
g = torch.Generator().manual_seed(5)
rc = torch.rand(R, 3, generator=g).to(dev)
depth = (0.5 + 2.5 * torch.rand(R, 1, generator=g)).to(dev)
opt = torch.optim.AdamW([{"params": net.get_training_parameters(), "lr": 1e-4}, {"params": net.get_volume_parameters(), "lr": 1e-3}])
params = net.get_training_parameters() + net.get_volume_parameters()


def step():
    opt.zero_grad()
    with torch.enable_grad():
        o = net(ro, rd, zv, ds)
        unc = 1.0 / torch.sqrt(o["depth_variance"].detach() + 1e-10)
        sl, spl = net.compute_sdf_error(sdf=o["sdf"], z_vals=o["z_vals"], gt_depth=depth)
        total = 2.0 * torch.abs(o["color"] - rc).mean() + (torch.abs(o["depth"] - depth) * unc).mean() + 2.0 * (sl + spl) + 0.1 * o["gradient_error"].mean()
    total.backward()
    torch.nn.utils.clip_grad_norm_(params, max_norm=35.0)
    opt.step()


for _ in range(3):
    step()
us = measure.kernel_times(step, steps=3)
measure.emit({})
for name, t in sorted(us.items(), key=lambda kv: -kv[1])[:28]:
    print("%9.1f us  %5.1f launches  %s" % (t, us.launches[name], name[:70]))
print("%9.1f us  total kernel time per iteration" % sum(us.values()))
