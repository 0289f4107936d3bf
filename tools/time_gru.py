"""ConvGRU at the config-2 update size (36 edges, 40x80): the wgmma kernel (NHWC in/out, and through the
reference's NCHW call) against the same module evaluated by torch/cuDNN under autocast (what the reference runs).
CUDA events around 20 back-to-back calls, 5 samples.
usage: python tools/time_gru.py [B h w]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import measure  # noqa: E402
measure.require_cuda("time_gru.py")
import torch  # noqa: E402
from goslam_b200.modules.gru import ConvGRU, to_nhwc  # noqa: E402

dev = torch.device("cuda:0")
B, h, w = (int(a) for a in sys.argv[1:4]) if len(sys.argv) >= 4 else (36, 40, 80)
torch.manual_seed(77)
m = ConvGRU(128, 320).to(dev)
g = torch.Generator().manual_seed(1)
net = torch.tanh(torch.randn(B, 128, h, w, generator=g)).to(dev).half()
inp, corr = [torch.relu(torch.randn(B, 128, h, w, generator=g)).to(dev).half() for _ in range(2)]
flow = torch.relu(torch.randn(B, 64, h, w, generator=g)).to(dev).half()


def cudnn_gru():
    """the reference's ConvGRU.forward, op for op (src/modules/gru.py:21-39), under autocast"""
    with torch.no_grad(), torch.autocast("cuda", enabled=True):
        x = torch.cat([inp, corr, flow], dim=1)
        net_inp = torch.cat([net, x], dim=1)
        b, c, hh, ww = net.shape
        glo = torch.sigmoid(m.w(net)) * net
        glo = glo.view(b, c, hh * ww).mean(dim=-1, keepdim=True).view(b, c, 1, 1)
        z = torch.sigmoid(m.convz(net_inp) + m.convz_glo(glo))
        r = torch.sigmoid(m.convr(net_inp) + m.convr_glo(glo))
        q = torch.tanh(m.convq(torch.cat([r * net, x], dim=1)) + m.convq_glo(glo))
        return (1 - z) * net + z * q


nh = [to_nhwc(x) for x in (net, inp, corr, flow)]
flops = 2.0 * B * h * w * (3 * 9 * 448 * 128 + 128 * 128)
ours = m.forward_nhwc(*nh)
ref = cudnn_gru()
measure.emit({})
print("max |ours - cuDNN autocast| = %.3e" % (ours.permute(0, 3, 1, 2).float() - ref.float()).abs().max().item())
for name, fn in (("wgmma ConvGRU, NHWC in/out", lambda: m.forward_nhwc(*nh)),
                 ("wgmma ConvGRU, reference NCHW call (+5 layout kernels)", lambda: m(net, inp, corr, flow)),
                 ("torch / cuDNN autocast (reference path)", cudnn_gru)):
    t = measure.cuda_time(fn, reps=5, batch=20)
    us = 1e3 * t["median_ms"]
    print("%-58s %9.1f us (%.1f-%.1f)  %7.1f TFLOP/s" % (name, us, 1e3 * t["min_ms"], 1e3 * t["max_ms"], flops / us / 1e6))
