"""per-kernel device time of the main leg's update step (36 edges, 40x80, tiled, 8 keyframes) under torch.profiler.
usage: profile_step.py [steps]   (TOOL_VARIANT=name: an A/B build made by tools/build_variant.py)"""
import collections, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
if os.environ.get("TOOL_VARIANT"):
    from tools.build_variant import use_variant
    use_variant(os.environ["TOOL_VARIANT"])
import bench

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
print(torch.cuda.get_device_name(0))
win = bench.Window(bench.make_window(43), torch.device("cuda:0"))
for _ in range(5):
    win.step()
torch.cuda.synchronize()
acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
with torch.profiler.profile(activities=acts) as prof:
    for _ in range(steps):
        win.step()
    torch.cuda.synchronize()
us = collections.Counter()
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
        us[ev.name] += ev.device_time_total / steps
for name, t in us.most_common():
    print("%9.1f us  %s" % (t, name[:110]))
print("%9.1f us  total kernel time per step" % sum(us.values()))
