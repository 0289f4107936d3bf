"""The two upsampling helpers of src/droid_net.py (:9-32) on the sm_90a kernel.

`cvx_upsample(data, mask)` and `upsample_disp(disp, mask)` keep the reference's signatures;
DepthVideo.upsample (src/depth_video.py:194-196) is `cvx_upsample(disps[ix].unsqueeze(-1), mask)`.
One launch (goslam_cvx_upsample) replaces permute + softmax + unfold + mul + sum + permute.
"""
import torch

from . import _lib


def cvx_upsample(data, mask):
    """data [b, ht, wd, dim] (dim <= 4), mask [b, 9*8*8, ht, wd] (f16 or f32) -> [b, 8ht, 8wd, dim] f32."""
    _lib.need_cuda("cvx_upsample", data)
    batch, ht, wd, dim = data.shape
    d = data.float().contiguous()
    m = mask.reshape(batch, 576, ht, wd).contiguous()
    if m.dtype not in (torch.float16, torch.float32):
        m = m.float()
    out = torch.empty((batch, 8 * ht, 8 * wd, dim), dtype=torch.float32, device=data.device)
    _lib.call("cvx_upsample", d, m, 1 if m.dtype == torch.float16 else 0, out, batch, ht, wd, dim)
    return out


def upsample_disp(disp, mask):
    batch, num, ht, wd = disp.shape
    disp = disp.reshape(batch * num, ht, wd, 1)
    mask = mask.reshape(batch * num, -1, ht, wd)
    return cvx_upsample(disp, mask).view(batch, num, 8 * ht, 8 * wd)


# ------------------------------------------------------------------------------------------------------
# The update operator (SURVEY §8f-4): UpdateModule / GraphAgg with the reference's parameter names
# (src/droid_net.py:33-140), so the `update.*` entries of pretrained/droid.pth load with load_state_dict.
# The whole forward is one library call (goslam_update_op, csrc/conv_tc.cu): every 1x1 / 3x3 layer and the
# ConvGRU on the wgmma implicit-GEMM kernel, the 7x7 motion encoder on a tensor-core im2col kernel, and GraphAgg's
# per-frame mean on a deterministic scatter-mean kernel, all in NHWC half precision.
# ------------------------------------------------------------------------------------------------------
import torch.nn as nn  # noqa: E402

from .modules.gru import ConvGRU  # noqa: E402


class _Identity(nn.Module):
    """GradientClip (src/modules/clipping.py) only acts in backward; inference sees the identity.  Kept as a
    module so that Sequential indices — and therefore state_dict keys — match the reference."""

    def forward(self, x):
        return x


def _nhwc_view(x):
    """[B,C,h,w] channels-last tensor -> its [B,h,w,C] contiguous view (a copy only if it was not channels-last)"""
    v = x.permute(0, 2, 3, 1)
    return v if v.is_contiguous() else v.contiguous()


class GraphAgg(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(128, 128, 3, padding=1)
        self.conv2 = nn.Conv2d(128, 128, 3, padding=1)
        self.relu = nn.ReLU(inplace=True)
        self.eta = nn.Sequential(nn.Conv2d(128, 1, 3, padding=1), _Identity(), nn.Softplus())
        self.upmask = nn.Sequential(nn.Conv2d(128, 8 * 8 * 9, 1))

    def forward(self, net, ii):
        """net [batch, num, 128, h, w], ii [num] -> 0.01 * eta [batch, M, h, w], upmask [batch, M, 576, h, w] with one
        row per distinct source frame, in sorted frame order (src/droid_net.py:51-67; scatter_mean = index_add / count)"""
        batch, num, ch, ht, wd = net.shape
        frames, ix = torch.unique(ii, sorted=True, return_inverse=True)
        x = self.relu(self.conv1(net.reshape(batch * num, ch, ht, wd))).view(batch, num, 128, ht, wd)
        m = frames.numel()
        agg = torch.zeros((batch, m, 128, ht, wd), dtype=x.dtype, device=x.device).index_add_(1, ix, x)
        cnt = torch.zeros(m, dtype=x.dtype, device=x.device).index_add_(0, ix, torch.ones_like(ix, dtype=x.dtype))
        x = (agg / cnt.view(1, m, 1, 1, 1)).view(-1, 128, ht, wd)
        x = self.relu(self.conv2(x))
        eta = self.eta(x).view(batch, -1, ht, wd)
        upmask = self.upmask(x).view(batch, -1, 8 * 8 * 9, ht, wd)
        return 0.01 * eta, upmask


class UpdateModule(nn.Module):
    """src/droid_net.py:70-140 with the reference's parameter names.  Every layer runs on a wgmma kernel in NHWC half
    precision:
        corr (196 ch, zero-padded to 256) -1x1-> 128 -3x3-> 128          goslam_conv2d_nhwc x2
        motion (4 ch) -7x7 (im2col + wgmma)-> 128 -3x3-> 64               flow7x7_tc_kernel + goslam_conv2d_nhwc
        ConvGRU(net, inp, corr, flow)                                     goslam_conv_gru (3 passes)
        delta.0 | weight.0 stacked to 256 outputs, then the two 2-channel heads (fp32 out)   x3
        GraphAgg: 3x3 -> per-source-frame mean -> 3x3 -> {eta 3x3 + softplus, upmask 1x1 -> 576}   x4
    """

    def __init__(self):
        super().__init__()
        cor_planes = 4 * (2 * 3 + 1) ** 2
        self.corr_encoder = nn.Sequential(nn.Conv2d(cor_planes, 128, 1), nn.ReLU(inplace=True),
                                          nn.Conv2d(128, 128, 3, padding=1), nn.ReLU(inplace=True))
        self.flow_encoder = nn.Sequential(nn.Conv2d(4, 128, 7, padding=3), nn.ReLU(inplace=True),
                                          nn.Conv2d(128, 64, 3, padding=1), nn.ReLU(inplace=True))
        self.weight = nn.Sequential(nn.Conv2d(128, 128, 3, padding=1), nn.ReLU(inplace=True),
                                    nn.Conv2d(128, 2, 3, padding=1), _Identity(), nn.Sigmoid())
        self.delta = nn.Sequential(nn.Conv2d(128, 128, 3, padding=1), nn.ReLU(inplace=True),
                                   nn.Conv2d(128, 2, 3, padding=1), _Identity())
        self.gru = ConvGRU(128, 128 + 128 + 64)
        self.agg = GraphAgg()
        self._packed = None

    def _pack(self):
        """kernel-side weights of every layer (include/goslam_b200.h: goslam_update_weights), cached per parameter version"""
        from .modules.gru import pack_conv
        params = list(self.parameters())
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is None or self._packed[0] != key:
            c, f, d, w, a = self.corr_encoder, self.flow_encoder, self.delta, self.weight, self.agg
            t = dict(
                corr0=pack_conv([c[0].weight], [c[0].bias], cin_pad=256), corr2=pack_conv([c[2].weight], [c[2].bias]),
                flow2=pack_conv([f[2].weight], [f[2].bias]),
                hid=pack_conv([d[0].weight, w[0].weight], [d[0].bias, w[0].bias]),
                delta=pack_conv([d[2].weight], [d[2].bias]), weight=pack_conv([w[2].weight], [w[2].bias]),
                agg1=pack_conv([a.conv1.weight], [a.conv1.bias]), agg2=pack_conv([a.conv2.weight], [a.conv2.bias]),
                eta=pack_conv([a.eta[0].weight], [a.eta[0].bias]), upmask=pack_conv([a.upmask[0].weight], [a.upmask[0].bias]))
            # 7x7 motion encoder (im2col + tensor cores): [co, ci, ky, kx] -> [co][k = (ky*7+kx)*4 + ci], K padded to 256
            w7 = torch.zeros((128, 256), dtype=torch.float16, device=f[0].weight.device)
            w7[:, :196] = f[0].weight.detach().permute(0, 2, 3, 1).reshape(128, 196).half()
            t["flow0"] = (w7.contiguous(), f[0].bias.detach().float().contiguous())
            # the two 2-channel heads as one block-diagonal layer over the 256 hidden channels
            hw_ = torch.zeros((9, 16, 256), dtype=torch.float16, device=w7.device)
            hw_[:, 0:2, 0:128] = t["delta"][0][:, 0:2]
            hw_[:, 2:4, 128:256] = t["weight"][0][:, 0:2]
            hb = torch.zeros(16, dtype=torch.float32, device=w7.device)
            hb[0:2], hb[2:4] = t["delta"][1][0:2], t["weight"][1][0:2]
            t["delta"] = (hw_.contiguous(), hb)
            st = _lib.UpdateWeights()
            st.gru = self.gru._pack()
            for name, (wt, bs) in t.items():
                setattr(st, name + "_w", wt.data_ptr())
                setattr(st, name + "_b", bs.data_ptr())
            self._packed = (key, t, st)
        return self._packed[2]

    def set_source_frames(self, frames, slot):
        """optional hint from FactorGraph: the distinct source frames (sorted) and each edge's slot among them — what
        GraphAgg's torch.unique(ii, return_inverse=True) would compute with a device->host sync"""
        self._frames_hint = (int(frames.numel()), slot.to(torch.int32).contiguous())

    @torch.no_grad()
    def forward(self, net, inp, corr, flow=None, ii=None, jj=None):
        """net, inp [batch, num, 128, h, w]; corr [batch, num, 196, h, w]; flow [batch, num, 4, h, w] ->
        net', delta [batch, num, h, w, 2], weight [batch, num, h, w, 2] (, eta [batch, M, h, w], upmask [batch, M, 576, h, w]
        when ii is given; M = distinct source frames, sorted) — src/droid_net.py:107-140.  One library call."""
        import ctypes
        batch, num, ch, ht, wd = net.shape
        _lib.need_cuda("UpdateModule", net)
        if batch != 1:
            raise RuntimeError("UpdateModule: batch 1 (as GO-SLAM calls it)")
        dev = net.device
        st = self._pack()
        N = num
        h16 = lambda t: (t if t.dtype == torch.float16 else t.half()).reshape(N, -1, ht, wd).contiguous()   # noqa: E731
        net_c, inp_c, corr_c = h16(net), h16(inp), h16(corr)
        flow_c = (torch.zeros(N, 4, ht, wd, device=dev) if flow is None else flow.reshape(N, 4, ht, wd).float().contiguous())
        M, slot = 0, None
        if ii is not None:
            hint = getattr(self, "_frames_hint", None)
            if hint is not None and hint[1].numel() == N:
                M, slot = hint
            else:
                frames, ix = torch.unique(ii.to(dev), sorted=True, return_inverse=True)
                M, slot = int(frames.numel()), ix.to(torch.int32).contiguous()
            self._frames_hint = None
        net_out = torch.empty((1, N, 128, ht, wd), dtype=torch.float16, device=dev)
        delta = torch.empty((1, N, ht, wd, 2), dtype=torch.float32, device=dev)
        weight = torch.empty((1, N, ht, wd, 2), dtype=torch.float32, device=dev)
        eta = torch.empty((1, M, ht, wd), dtype=torch.float32, device=dev) if slot is not None else None
        upmask = torch.empty((1, M, 576, ht, wd), dtype=torch.float16, device=dev) if slot is not None else None
        ws = _lib.workspace(_lib.load().goslam_update_op_workspace_bytes(N, M, ht, wd), dev)
        _lib.call("update_op", ctypes.byref(st), net_c, inp_c, corr_c, flow_c, slot, N, M, ht, wd, net_out, delta, weight,
                  eta, upmask, ws, ws.numel())
        net_out = net_out.to(net.dtype)
        if slot is None:
            return net_out, delta, weight
        return net_out, delta, weight, eta, upmask
