"""Float64 restatement of the update operator: UpdateModule.forward (src/droid_net.py:107-140) with its ConvGRU
(src/modules/gru.py:21-39) and GraphAgg (src/droid_net.py:51-67), from an `UpdateModule` state dict.  Plain torch,
device-agnostic; only tests import it.

round16=False: the reference's arithmetic in float64.

round16=True: the same, but every value goslam_update_op (csrc/conv_tc.cu) stores as fp16 is rounded to fp16 at the
point where the kernels store it; all other arithmetic stays float64.  The rounding points:
  operands      the convolution weights (not the fp32 `*_glo` 1x1s on the pooled vector, not any bias);
                net, inp and corr on input; flow inside the 7x7 im2col
  encoders      c1, c2 (corr), f1, f2 (flow)
  ConvGRU       z, r*net and net' (not the pooled glo, r or q)
  heads         the hidden layer (delta.0 | weight.0), a1 = relu(agg.conv1), the scatter-mean, a2 = relu(agg.conv2)
                and upmask
  never         delta, weight and eta (written as fp32)
What is left between this and the kernels is fp32 accumulation order, which can flip an fp16 rounding."""
import torch
import torch.nn.functional as F


def _round16(x):
    return x.to(torch.float16).to(torch.float64)


def _keep(x):
    return x


class _Params:
    """conv layers of a state dict in float64: weights optionally fp16-rounded, biases exact"""

    def __init__(self, sd, prefix, r):
        self.sd, self.prefix, self.r = sd, prefix, r

    def conv(self, x, name, rounded=True):
        w = self.sd[self.prefix + name + ".weight"].detach().to(device=x.device, dtype=torch.float64)
        b = self.sd[self.prefix + name + ".bias"].detach().to(device=x.device, dtype=torch.float64)
        return F.conv2d(x, self.r(w) if rounded else w, b, padding=w.shape[-1] // 2)


def conv_gru(sd, net, inp, corr, flow, round16=False, prefix=""):
    """ConvGRU.forward: net, inp, corr [B,128,h,w], flow [B,64,h,w] (any float dtype) -> net' [B,128,h,w] float64.
    `sd` holds the ConvGRU's parameters under `prefix` (e.g. "gru." inside an UpdateModule state dict)."""
    r = _round16 if round16 else _keep
    p = _Params(sd, prefix, r)
    net = r(net.double())
    x = torch.cat([r(inp.double()), r(corr.double()), r(flow.double())], dim=1)
    glo = (torch.sigmoid(p.conv(net, "w")) * net).mean(dim=(2, 3), keepdim=True)
    zin = torch.cat([net, x], dim=1)
    z = r(torch.sigmoid(p.conv(zin, "convz") + p.conv(glo, "convz_glo", rounded=False)))
    rr = torch.sigmoid(p.conv(zin, "convr") + p.conv(glo, "convr_glo", rounded=False))
    q = torch.tanh(p.conv(torch.cat([r(rr * net), x], dim=1), "convq") + p.conv(glo, "convq_glo", rounded=False))
    return r((1 - z) * net + z * q)


def update_forward(sd, net, inp, corr, flow=None, ii=None, round16=False):
    """UpdateModule.forward.  net, inp [batch, num, 128, h, w]; corr [batch, num, 196, h, w]; flow [batch, num, 4, h, w]
    or None (zeros); ii [num] or None.  Returns float64 (net' [batch, num, 128, h, w], delta, weight [batch, num, h, w, 2])
    and, when ii is given, (0.01 * eta [batch, M, h, w], upmask [batch, M, 576, h, w]) with one row per distinct source
    frame in sorted order (torch.unique(ii, sorted=True, return_inverse=True), scatter-mean = sum / count)."""
    r = _round16 if round16 else _keep
    p = _Params(sd, "", r)
    batch, num, _, ht, wd = net.shape
    flat = lambda t: t.reshape(batch * num, -1, ht, wd).double()                  # noqa: E731
    if flow is None:
        flow = torch.zeros((batch, num, 4, ht, wd), dtype=torch.float64, device=net.device)
    relu = torch.relu
    c = r(relu(p.conv(r(flat(corr)), "corr_encoder.0")))
    c = r(relu(p.conv(c, "corr_encoder.2")))
    f = r(relu(p.conv(r(flat(flow)), "flow_encoder.0")))
    f = r(relu(p.conv(f, "flow_encoder.2")))
    net = conv_gru(sd, flat(net), flat(inp), c, f, round16=round16, prefix="gru.")
    delta = p.conv(r(relu(p.conv(net, "delta.0"))), "delta.2")
    weight = torch.sigmoid(p.conv(r(relu(p.conv(net, "weight.0"))), "weight.2"))
    nhwc = lambda t: t.view(batch, num, 2, ht, wd).permute(0, 1, 3, 4, 2).contiguous()   # noqa: E731
    out = (net.view(batch, num, 128, ht, wd), nhwc(delta), nhwc(weight))
    if ii is None:
        return out
    frames, ix = torch.unique(ii.to(net.device), sorted=True, return_inverse=True)
    m = frames.numel()
    a1 = r(relu(p.conv(net, "agg.conv1"))).view(batch, num, 128, ht, wd)
    total = torch.zeros((batch, m, 128, ht, wd), dtype=torch.float64, device=net.device).index_add_(1, ix, a1)
    cnt = torch.bincount(ix, minlength=m).to(torch.float64)
    mean = r(total / cnt.view(1, m, 1, 1, 1)).view(batch * m, 128, ht, wd)
    a2 = r(relu(p.conv(mean, "agg.conv2")))
    eta = 0.01 * F.softplus(p.conv(a2, "agg.eta.0"))
    upmask = r(p.conv(a2, "agg.upmask.0"))
    return out + (eta.view(batch, m, ht, wd), upmask.view(batch, m, 576, ht, wd))
