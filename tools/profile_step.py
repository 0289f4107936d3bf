"""per-kernel device time of the main leg's update step (36 edges, 40x80, tiled, 8 keyframes), from
measure.kernel_times.
usage: profile_step.py [steps]   (TOOL_VARIANT=name: an A/B build made by tools/build_variant.py)"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("profile_step.py")
import torch  # noqa: E402
if os.environ.get("TOOL_VARIANT"):
    from tools.build_variant import use_variant
    use_variant(os.environ["TOOL_VARIANT"])
import bench  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
measure.emit({})
win = bench.Window(bench.make_window(43), torch.device("cuda:0"))
for _ in range(5):
    win.step()
us = measure.kernel_times(win.step, steps)
for name, t in sorted(us.items(), key=lambda kv: -kv[1]):
    print("%9.1f us  %s" % (t, name[:110]))
print("%9.1f us  total kernel time per step" % sum(us.values()))
