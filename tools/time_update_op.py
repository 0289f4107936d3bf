"""goslam_b200.droid_net.UpdateModule at the config-2 update size (36 edges, 40x80) against the reference forward in
torch / cuDNN under autocast.  GPU: CUDA events around 20 back-to-back calls, 5 samples; wall: host clock around the
same 20 calls and a device synchronise.  Per-kernel times: tools/measure.py's kernel_times, as tools/profile_step.py
uses it."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_update_op.py")
import torch  # noqa: E402
from goslam_b200.droid_net import UpdateModule  # noqa: E402

dev = torch.device("cuda:0")
B, h, w = 36, 40, 80
torch.manual_seed(11)
m = UpdateModule().to(dev).eval()
g = torch.Generator().manual_seed(1)
net = torch.tanh(torch.randn(1, B, 128, h, w, generator=g)).half().to(dev)
inp = torch.relu(torch.randn(1, B, 128, h, w, generator=g)).half().to(dev)
corr = (0.7 * torch.randn(1, B, 196, h, w, generator=g)).half().to(dev)
flow = (4 * torch.randn(1, B, 4, h, w, generator=g)).to(dev)
ii = (torch.arange(B) // 5).to(dev)
jj = ((torch.arange(B) + 1) % 8).to(dev)


def t(name, fn, n=20):
    gpu = measure.cuda_time(fn, reps=5, batch=n)
    wall = measure.host_time(lambda: [fn() for _ in range(n)], reps=5, warmup=0)
    print("%-38s GPU %8.1f us (%.1f-%.1f)   wall %8.1f us (%.1f-%.1f)" % (
        name, 1e3 * gpu["median_ms"], 1e3 * gpu["min_ms"], 1e3 * gpu["max_ms"],
        1e3 * wall["median_ms"] / n, 1e3 * wall["min_ms"] / n, 1e3 * wall["max_ms"] / n))


measure.emit({})
t("whole forward (one library call)", lambda: m(net, inp, corr, flow, ii, jj))


def torch_reference_forward():
    """the reference UpdateModule.forward, op for op, in torch under autocast (cuDNN): src/droid_net.py:107-140"""
    with torch.no_grad(), torch.autocast("cuda", enabled=True):
        n_, i_, c_, f_ = [x.view(B, -1, h, w) for x in (net, inp, corr, flow)]
        c_ = m.corr_encoder(c_)
        f_ = m.flow_encoder(f_)
        gru = m.gru
        x = torch.cat([i_, c_, f_], dim=1)
        net_inp = torch.cat([n_, x], dim=1)
        glo = (torch.sigmoid(gru.w(n_)) * n_).view(B, 128, h * w).mean(dim=-1, keepdim=True).view(B, 128, 1, 1)
        z = torch.sigmoid(gru.convz(net_inp) + gru.convz_glo(glo))
        r = torch.sigmoid(gru.convr(net_inp) + gru.convr_glo(glo))
        q = torch.tanh(gru.convq(torch.cat([r * n_, x], dim=1)) + gru.convq_glo(glo))
        n2 = (1 - z) * n_ + z * q
        delta = m.delta(n2).view(1, B, -1, h, w).permute(0, 1, 3, 4, 2)[..., :2].contiguous()
        weight = m.weight(n2).view(1, B, -1, h, w).permute(0, 1, 3, 4, 2)[..., :2].contiguous()
        eta, upmask = m.agg(n2.view(1, B, 128, h, w), ii)
        return n2, delta, weight, eta, upmask


t("torch/cuDNN autocast reference forward", torch_reference_forward)
