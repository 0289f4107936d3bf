"""`ConvGRU` with the reference's constructor, parameter names and call signature (src/modules/gru.py:5-39),
so `UpdateModule.gru` state dicts load unchanged — forward runs on the wgmma implicit-GEMM kernel
(csrc/conv_tc.cu, goslam_conv_gru): three convolution passes with the gate arithmetic fused into their
epilogues instead of 7 cuDNN convolutions + 2 concatenations + ~12 elementwise kernels.

    gru = ConvGRU(128, 128 + 128 + 64)
    net = gru(net, inp, corr, flow)          # [B,128,h,w], [B,128,h,w], [B,128,h,w], [B,64,h,w] -> [B,128,h,w]

Inference only (torch.no_grad, as the SLAM threads run it); fp16 operands with fp32 accumulation, i.e. what the
reference computes inside its autocast region.  No CPU path."""
import ctypes

import torch
import torch.nn as nn

from .. import _lib


def to_nhwc(x):
    """[B, C, h, w] (any float dtype) -> [B, h, w, C] float16, one kernel"""
    b, c, h, w = x.shape
    src = x.contiguous() if x.dtype == torch.float16 else x.half().contiguous()
    dst = torch.empty((b, h, w, c), dtype=torch.float16, device=x.device)
    _lib.call("nchw_to_nhwc_f16", src, dst, b, c, h * w)
    return dst


def to_nchw(x):
    """[B, h, w, C] float16 -> [B, C, h, w] float16"""
    b, h, w, c = x.shape
    dst = torch.empty((b, c, h, w), dtype=torch.float16, device=x.device)
    _lib.call("nhwc_to_nchw_f16", x, dst, b, c, h * w)
    return dst


class ConvGRU(nn.Module):
    def __init__(self, h_planes=128, i_planes=128):
        super().__init__()
        if h_planes != 128 or i_planes != 320:
            raise ValueError("goslam_b200 ConvGRU is specialised to the update operator's 128 + (128+128+64) channels")
        self.do_checkpoint = False
        self.convz = nn.Conv2d(h_planes + i_planes, h_planes, 3, padding=1)
        self.convr = nn.Conv2d(h_planes + i_planes, h_planes, 3, padding=1)
        self.convq = nn.Conv2d(h_planes + i_planes, h_planes, 3, padding=1)
        self.w = nn.Conv2d(h_planes, h_planes, 1)
        self.convz_glo = nn.Conv2d(h_planes, h_planes, 1)
        self.convr_glo = nn.Conv2d(h_planes, h_planes, 1)
        self.convq_glo = nn.Conv2d(h_planes, h_planes, 1)
        self._packed = None

    def _pack(self):
        """kernel-side weight layout ([tap][cout][cin] fp16, include/goslam_b200.h), cached per parameter version"""
        params = [self.convz.weight, self.convr.weight, self.convq.weight, self.w.weight, self.convz_glo.weight,
                  self.convr_glo.weight, self.convq_glo.weight, self.convz.bias, self.convr.bias, self.convq.bias,
                  self.w.bias, self.convz_glo.bias, self.convr_glo.bias, self.convq_glo.bias]
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is None or self._packed[0] != key:
            def taps(wt):            # [co, ci, 3, 3] -> [9, co, ci]
                return wt.detach().permute(2, 3, 0, 1).reshape(9, wt.shape[0], wt.shape[1])
            t = dict(
                w_zr=torch.cat([taps(self.convz.weight), taps(self.convr.weight)], dim=1).half().contiguous(),
                w_q=taps(self.convq.weight).half().contiguous(),
                w_w=self.w.weight.detach().reshape(128, 128).half().contiguous(),
                b_zr=torch.cat([self.convz.bias, self.convr.bias]).detach().float().contiguous(),
                b_q=self.convq.bias.detach().float().contiguous(),
                b_w=self.w.bias.detach().float().contiguous(),
                w_glo=torch.cat([m.weight.detach().reshape(128, 128) for m in (self.convz_glo, self.convr_glo, self.convq_glo)]).float().contiguous(),
                b_glo=torch.cat([m.bias.detach() for m in (self.convz_glo, self.convr_glo, self.convq_glo)]).float().contiguous())
            st = _lib.GruWeights()
            for k, v in t.items():
                setattr(st, k, v.data_ptr())
            self._packed = (key, t, st)
        return self._packed[2]

    @torch.no_grad()
    def forward_nhwc(self, net, inp, corr, flow):
        """all tensors NHWC float16 ([B,h,w,128] x3, [B,h,w,64]); returns the new state [B,h,w,128] float16"""
        if not net.is_cuda:
            raise RuntimeError("ConvGRU: CUDA tensors required (no CPU fallback)")
        b, h, w, _ = net.shape
        out = torch.empty_like(net)
        st = self._pack()
        ws = _lib.workspace(_lib.load().goslam_conv_gru_workspace_bytes(b, h, w), net.device)
        _lib.call("conv_gru", ctypes.byref(st), net, inp, corr, flow, out, b, h, w, ws, ws.numel())
        return out

    @torch.no_grad()
    def forward(self, net, *inputs):
        """reference call: net [B,128,h,w], inputs = (inp [B,128,h,w], corr [B,128,h,w], flow [B,64,h,w])"""
        if len(inputs) != 3 or [t.shape[1] for t in inputs] != [128, 128, 64] or net.shape[1] != 128:
            raise RuntimeError("ConvGRU: expected (net[128], inp[128], corr[128], flow[64]) channel layout")
        out = self.forward_nhwc(to_nhwc(net), *[to_nhwc(t) for t in inputs])
        return to_nchw(out).to(net.dtype)


# ------------------------------------------------------------------------------------------------------
# Generic layer entry (goslam_conv2d_nhwc): the encoders, heads and GraphAgg of the update operator
# ------------------------------------------------------------------------------------------------------
ACT = {None: 0, "none": 0, "relu": 1, "sigmoid": 2, "softplus": 3}


def pack_conv(weights, biases, cin_pad=None, cout_pad=None):
    """torch conv parameters -> the kernel's layout.  `weights`: list of [co_i, ci, k, k] tensors stacked along cout
    (k = 1 or 3); returns (w f16 [k*k, cout_pad, cin_pad], b f32 [cout_pad]); padding rows / columns are zero."""
    w = torch.cat([x.detach() for x in weights], dim=0)
    b = torch.cat([x.detach() for x in biases], dim=0).float()
    co, ci, k, _ = w.shape
    cin_pad = cin_pad or ci
    cout_pad = cout_pad or ((co + 15) // 16 * 16)
    out = torch.zeros((k * k, cout_pad, cin_pad), dtype=torch.float16, device=w.device)
    out[:, :co, :ci] = w.permute(2, 3, 0, 1).reshape(k * k, co, ci).half()
    bias = torch.zeros(cout_pad, dtype=torch.float32, device=w.device)
    bias[:co] = b
    return out.contiguous(), bias


def conv2d_nhwc(inputs, weight, bias, cout, act=None, out=None, out_f32=False, out_offset=0, out_scale=1.0):
    """One 1x1 / 3x3 layer on the wgmma kernel.  inputs: list of (NHWC f16 tensor, channels used, first channel);
    weight / bias from `pack_conv`; out: optional NHWC destination (a wider tensor, written at channel out_offset)."""
    x0 = inputs[0][0]
    B, h, w, _ = x0.shape
    taps, cout_pad, cin_total = weight.shape
    if sum(c for _, c, _ in inputs) != cin_total:
        raise RuntimeError("conv2d_nhwc: packed weight expects %d input channels" % cin_total)
    if out is None:
        out = torch.empty((B, h, w, cout), dtype=torch.float32 if out_f32 else torch.float16, device=x0.device)
    d = _lib.ConvDesc()
    for i, (t, c, off) in enumerate(inputs):
        if t.dtype != torch.float16 or not t.is_contiguous():
            raise RuntimeError("conv2d_nhwc: inputs must be contiguous NHWC float16")
        d.inp[i], d.cin[i], d.cin_off[i], d.cin_stride[i] = t.data_ptr(), c, off, t.shape[-1]
    d.n_in = len(inputs)
    d.weight, d.bias = weight.data_ptr(), bias.data_ptr()
    d.taps, d.cout, d.cout_pad, d.act = taps, cout, cout_pad, ACT[act]
    d.out_scale = float(out_scale)
    d.out, d.out_f32, d.out_stride, d.out_offset = out.data_ptr(), int(out.dtype == torch.float32), out.shape[-1], out_offset
    _lib.call("conv2d_nhwc", ctypes.byref(d), B, h, w, device=x0.device)
    return out


def to_nhwc_padded(x, cpad):
    """[B, C, h, w] -> [B, h, w, cpad] float16 with zero channels C..cpad-1 (one kernel)"""
    b, c, h, w = x.shape
    src = x.contiguous() if x.dtype == torch.float16 else x.half().contiguous()
    dst = torch.empty((b, h, w, cpad), dtype=torch.float16, device=x.device)
    _lib.call("nchw_to_nhwc_f16_pad", src, dst, b, c, cpad, h * w)
    return dst
