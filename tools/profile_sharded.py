"""torchrun --nproc-per-node N tools/profile_sharded.py : kernel-level summary (measure.kernel_times, rank 0) of the
sharded-graph leg of bench.py with both exchanges (NCCL collectives, peer memory): how long the all-reduce / all-gather
kernels take per BA iteration, what the peer path launches instead."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("profile_sharded.py")
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import bench  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
from goslam_b200 import _lib
_lib.load()
steps, warm = 20, 3
recs = []
us = measure.kernel_times(lambda: recs.append(bench.sharded_graph_leg(dev, steps, warm, lambda: dist.barrier(), world,
                                                                      rank)))
if rank == 0:
    measure.emit({})
    print("exchanges:", {k: {a: b for a, b in v.items() if a != "poses"} for k, v in recs[0]["exchanges"].items()})
    rows = sorted(((k, us.launches[k], t / 1e3) for k, t in us.items() if t > 0), key=lambda r: -r[2])
    per_variant_updates = steps + warm
    print("| kernel | launches | total ms | avg us |")
    print("|---|---|---|---|")
    for k, c, t in rows[:22]:
        print("| `%s` | %d | %.2f | %.1f |" % (k[:90], c, t, 1e3 * t / c))
    print("(each exchange variant ran %d updates x 2 BA iterations)" % per_variant_updates)
dist.barrier()
dist.destroy_process_group()
