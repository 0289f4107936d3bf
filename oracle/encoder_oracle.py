"""BasicEncoder (src/modules/extractor.py) restated with torch.nn.functional, and the pieces of a MotionFilter replay.

Three modes of `basic_encoder`:
  float64      every op in f64 (the yardstick);
  autocast     the same functional graph under torch.autocast("cuda") with f32 weights: every op gets the dtype and
               rounding point the reference's nn modules get when DroidNet runs them (MotionFilter's autocast);
  round16      float64 arithmetic, rounded to f16 exactly where goslam_basic_encoder (csrc/encoder.cu) stores f16:
    stem input   (x - mean) / std in f32, then f16; an f16 image is rounded after the subtract and after the divide
    weights      f16; biases exact
    conv output  accumulator + bias, then f16; norm 'none': ReLU of the f16 value, and conv2's relu(y + res) in f16
    instance     mean and biased variance (eps 1e-5) of the f16 conv output; the layer that reads it normalises on
                 load, applies the ReLU and rounds to f16; the residual tail relu(relu(n2(y)) + x') is rounded once
                 (x' = relu(n1(stem)) of layer1.0, n3(downsample) of a stride-2 block, unrounded)
    output       conv2 in f16; split applies tanh / relu to the f16 value and rounds again
  What is left between round16 and the kernels is the order of their fp32 accumulations and fp32 statistics.
Weights are a state_dict with the reference's key names (`conv1.weight`, `layer2.0.downsample.0.bias`, ...).
"""
import numpy as np
import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STDV = (0.229, 0.224, 0.225)


def _round16(x):
    return x.to(torch.float16).to(torch.float64)


def _keep(x):
    return x


def _instance16(x, stats=None):
    """instance norm (biased variance, eps 1e-5) of f16-valued x in float64.  stats: a list that collects the
    per-(image, channel) mean, rstd, min and max of x, [B, C] each"""
    if x.shape[2] * x.shape[3] == 1:
        raise ValueError("Expected more than 1 spatial element when training, got input size %s" % (x.shape,))
    mean = x.mean(dim=(2, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt((x - mean).pow(2).mean(dim=(2, 3), keepdim=True) + 1e-5)
    if stats is not None:
        stats.append((mean[..., 0, 0], rstd[..., 0, 0], x.amin(dim=(2, 3)), x.amax(dim=(2, 3))))
    return (x - mean) * rstd


class _Ops:
    """the graph's convolutions, normalisation and f16 rounding points: identities and F.instance_norm for the float64
    and autocast modes, so that those run the reference's op sequence unchanged"""

    def __init__(self, sd, inst, round16, trace=None):
        self.sd, self.inst, self.trace = sd, inst, trace
        self.r = _round16 if round16 else _keep
        stats = trace.setdefault("norm", []) if trace is not None else None
        self.n = (lambda x: _instance16(x, stats)) if round16 else (lambda x: F.instance_norm(x, eps=1e-5))

    def conv(self, x, name, stride, pad):
        return self.r(F.conv2d(x, self.r(self.sd[name + ".weight"]), self.sd[name + ".bias"], stride, pad))

    def norm(self, x):
        return self.n(x) if self.inst else x


def _block(o, p, x, x_in, stride):
    """x: the block's input as conv1 reads it; x_in: as the residual adds it"""
    r, relu = o.r, F.relu
    y = r(relu(o.norm(o.conv(x, p + "conv1", stride, 1))))
    y = relu(o.norm(o.conv(y, p + "conv2", 1, 1)))
    if stride > 1:
        x_in = o.norm(o.conv(x, p + "downsample.0", stride, 0))
    return r(relu(x_in + y))


def _graph(o, x):
    x_in = F.relu(o.norm(o.conv(x, "conv1", 2, 3)))
    x = o.r(x_in)
    for layer, stride in ((1, 1), (2, 2), (3, 2)):
        x = x_in = _block(o, "layer%d.0." % layer, x, x_in, stride)
        x = x_in = _block(o, "layer%d.1." % layer, x, x_in, 1)
    if o.trace is not None:
        o.trace["head"] = x
    return o.conv(x, "conv2", 1, 0)


def _stem_input16(x, mean, std):
    """the stem's operand: (x - mean) / std in f32 (after each op in f16 for an f16 image), rounded to f16"""
    if mean is not None:
        mu = torch.tensor(mean, dtype=torch.float32, device=x.device)[:, None, None]
        sd = torch.tensor(std, dtype=torch.float32, device=x.device)[:, None, None]
        if x.dtype == torch.float16:
            x = ((x.float() - mu).half().float() / sd).half()
        else:
            x = (x.float() - mu) / sd
    return _round16(x)


def basic_encoder(sd, norm_fn, x, mean=None, std=None, autocast=False, round16=False, trace=None):
    """x [B, 3, H, W] -> [B, out_dim, H/8, W/8].  mean / std: (x - mean) / std first, in f32 (autocast) or f64.
    float64 mode returns f64; autocast mode returns what the reference's autocast graph returns (f16); round16 returns
    f64 holding the f16 values goslam_basic_encoder writes, for an f32 or f16 x.  trace: a dict that receives, in
    round16 mode, "norm": each instance norm's statistics in graph order (see _instance16) and "head": the output
    conv's input."""
    if norm_fn not in ("instance", "none"):
        raise NotImplementedError(norm_fn)
    if autocast and round16:
        raise ValueError("autocast and round16 are exclusive")
    inst = norm_fn == "instance"
    dt = torch.float32 if autocast else torch.float64
    sd = {k: v.detach().to(x.device, dt) for k, v in sd.items()}
    if round16:
        x = _stem_input16(x, mean, std)
    else:
        x = x.to(dt)
        if mean is not None:
            x = (x - torch.tensor(mean, dtype=dt, device=x.device)[:, None, None]) / \
                torch.tensor(std, dtype=dt, device=x.device)[:, None, None]
    o = _Ops(sd, inst, round16, trace if round16 else None)
    with torch.no_grad():
        if not autocast:
            return _graph(o, x)
        with torch.autocast("cuda"):
            return _graph(o, x)


def context_split(out):
    """MotionFilter.__context_encoder's split of the 256-channel cnet output"""
    net, inp = out.split([128, 128], dim=1)
    return net.tanh(), inp.relu()


def errors(got, ref):
    """(max-abs, rms) of got - ref, both relative to ref's RMS"""
    d = (got.double() - ref.double())
    rms = ref.double().pow(2).mean().sqrt().item()
    return d.abs().max().item() / rms, d.pow(2).mean().sqrt().item() / rms


def contract_ok(got, autocast_out, ref64):
    """the kernel's error against f64 is at most 2x the autocast path's, plus one f16 ulp of the output's scale"""
    e_k = errors(got, ref64)
    e_a = errors(autocast_out, ref64)
    scale = ref64.double().abs().max().item()
    rms = ref64.double().pow(2).mean().sqrt().item()
    floor = float(np.spacing(np.float16(scale))) / rms
    return all(k <= 2.0 * a + floor for k, a in zip(e_k, e_a)), e_k, e_a


def seeded_params(module, seed):
    """fill every parameter in sorted-name order with U(-b, b), b = 1/sqrt(fan_in) (nn.Conv2d's default scale): the
    same values for the reference's module and ours, whatever their construction order"""
    g = torch.Generator().manual_seed(seed)
    params = dict(module.named_parameters())
    with torch.no_grad():
        for name in sorted(params):
            p = params[name]
            fan_in = p[0].numel() if p.dim() > 1 else max(1, p.numel())
            b = 1.0 / np.sqrt(fan_in)
            p.copy_(((torch.rand(p.shape, generator=g, dtype=torch.float64) * 2 - 1) * b).to(p.dtype))
    return module


SHIFTS = (0, 0, 1, 1, 9, 9, 10, 18, 18, 19, 27, 28)


def sequence(H=128, W=128, seed=5, shifts=SHIFTS):
    """a seeded synthetic RGB sequence [len(shifts), 3, H, W] (values k/255, f32): one smooth random field (a 40 x 40
    bicubic lattice, so that its features decorrelate over a few feature pixels) cropped at offset (s // 2, s) for
    each shift s: repeated frames, 1-pixel steps and 8-9 pixel jumps"""
    g = torch.Generator().manual_seed(seed)
    pad = max(shifts) + 8
    low = torch.rand(1, 3, 40, 40, generator=g, dtype=torch.float64)
    field = F.interpolate(low, size=(H + pad, W + pad), mode="bicubic", align_corners=True)[0].clamp(0, 1)
    imgs = [field[:, s // 2:s // 2 + H, s:s + W] for s in shifts]
    return (torch.round(torch.stack(imgs) * 255.0) / 255.0).float()


def motion_update_params(update, seed):
    """update-operator weights for the motion-filter replay: seeded_params, then a gate that responds to motion.
    Random weights alone give nearly the same mean flow on every frame, so:
      corr_encoder.0   every output = 1 + 0.2 * (mean of the level-0 window - its centre tap): the correlation's
                       zero-displacement peak above its level (static frame) drives it to 0 through the ReLU, a
                       frame moved by a few feature pixels leaves it near 1;
      gru              z = sigmoid(5) with no other input, and q reads only the correlation features (net, inp, flow
                       and the global-context terms zeroed), so net' ~ q;
      delta head       seeded, biases zeroed: the flow is ~0 where q ~ 0.
    The mean flow is then ~0.005-0.01 for repeated frames and 1-pixel steps and ~0.04 for 8-9 pixel jumps."""
    seeded_params(update, seed)
    with torch.no_grad():
        c = update.corr_encoder[0]
        c.weight.zero_()
        c.bias.fill_(1.0)
        c.weight[:, 0:49] = 0.2 / 49.0
        c.weight[:, 24] -= 0.2
        gru = update.gru
        gru.convz.weight.zero_()
        gru.convz.bias.fill_(5.0)
        gru.convq.weight[:, :256].zero_()
        gru.convq.weight[:, 384:].zero_()
        gru.convq.bias.zero_()
        for name in ("convz_glo", "convr_glo", "convq_glo"):
            getattr(gru, name).weight.zero_()
            getattr(gru, name).bias.zero_()
        update.delta[0].bias.zero_()
        update.delta[2].bias.zero_()
    return update


class RecordingVideo:
    """the part of DepthVideo MotionFilter uses: `counter.value` and `append`, recorded"""

    class _Counter:
        value = 0

    def __init__(self):
        self.counter = self._Counter()
        self.items = []

    def append(self, *item):
        self.items.append(item)
        self.counter.value += 1


def coords_grid(ht, wd, device):
    y, x = torch.meshgrid(torch.arange(ht, device=device).float(), torch.arange(wd, device=device).float(), indexing="ij")
    return torch.stack([x, y], dim=-1)


def track_step(fnet_sd, cnet_sd, update, corr_block, state, image, thresh, mean=MEAN, std=STDV):
    """MotionFilter.track's work for one frame, restated with the autocast oracle encoders (for timing and
    cross-checks).  state: dict with net / inp / fmap of the last keyframe, or empty.  Returns (accepted, delta mean)."""
    gmap = basic_encoder(fnet_sd, "instance", image, mean, std, autocast=True)
    ht, wd = gmap.shape[-2:]
    if not state:
        state["net"], state["inp"] = context_split(basic_encoder(cnet_sd, "none", image[:1], mean, std, autocast=True))
        state["fmap"] = gmap
        return True, None
    corr = corr_block(state["fmap"][None, [0]], gmap[None, [0]])(coords_grid(ht, wd, image.device)[None, None])
    _, delta, _ = update(state["net"][None], state["inp"][None], corr)
    dm = delta.norm(dim=-1).mean().item()
    if dm > thresh:
        state["net"], state["inp"] = context_split(basic_encoder(cnet_sd, "none", image[:1], mean, std, autocast=True))
        state["fmap"] = gmap
        return True, dm
    return False, dm
