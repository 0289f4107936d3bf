"""Time DroidNet's feature / context encoders and one MotionFilter.track on the GPU.

  encoders  fnet ('instance', 128 out) and cnet ('none', 256 out) at 240x320, 384x512 and 320x640 with B = 1 and 16:
            goslam_b200's BasicEncoder against the reference's numerics on cuDNN (oracle.encoder_oracle's functional
            graph under autocast), CUDA events after warm-up, median of several windows.  Achieved FLOP/s counts
            2 * MACs of every convolution, from the shapes below.  Each sample is one event pair around --iters calls.
  track     one MotionFilter.track per frame at 384x512, accept and reject paths: goslam_b200.MotionFilter against the
            same steps restated in torch (autocast encoders, CorrBlock, net.update, .item()).
Prints the card name and power limit with the numbers, one JSON object per line.
Run:  python tools/time_encoder.py [--windows 7] [--iters 20] [--profile]
"""
import argparse
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools import measure  # noqa: E402
measure.require_cuda("time_encoder.py")

import torch  # noqa: E402

from oracle import encoder_oracle as eo  # noqa: E402

DEV = torch.device("cuda:0")
SIZES = [(240, 320), (384, 512), (320, 640)]
PEAK_F16 = 989e12     # dense FP16 tensor-core rate of the H100 SXM data sheet (700 W)


def encoder_flops(H, W, out_dim):
    """2 * MACs of BasicEncoder's convolutions for one image"""
    def conv(ho, wo, cin, cout, k):
        return 2 * ho * wo * cin * cout * k * k
    h, w = H // 2, W // 2
    f = conv(h, w, 3, 32, 7)
    cin = 32
    for dim, stride in ((32, 1), (64, 2), (128, 2)):
        h, w = h // stride, w // stride
        f += conv(h, w, cin, dim, 3) + conv(h, w, dim, dim, 3)
        if stride == 2:
            f += conv(h, w, cin, dim, 1)
        f += 2 * conv(h, w, dim, dim, 3)
        cin = dim
    return f + conv(h, w, 128, out_dim, 1)


def timed(fn, windows, iters):
    return measure.cuda_time(fn, windows, batch=iters)["median_ms"]


def profile():
    """per-kernel CUDA time of one encoder call (measure.kernel_times, 10 calls after warm-up), summed by kernel name"""
    from goslam_b200.modules.extractor import BasicEncoder
    torch.manual_seed(0)
    for norm, dim in (("instance", 128), ("none", 256)):
        enc = BasicEncoder(dim, norm).to(DEV)
        for B in (1, 16):
            x = torch.rand(1, B, 3, 384, 512, device=DEV)
            with torch.autocast("cuda"):
                for _ in range(3):
                    enc(x)
                us = measure.kernel_times(lambda: enc(x), steps=10)
            per = {}
            for name, t in us.items():
                m = re.search(r"(encoder_\w+)(<[^>]*>)?", name)
                k = name if m is None else ("stem" if m.group(2) == "<32, true>" else m.group(1) + (m.group(2) or ""))
                per[k] = per.get(k, 0.0) + t / 1000.0
            total = sum(per.values())
            measure.emit({"what": "profile", "norm": norm, "H": 384, "W": 512, "B": B,
                          "kernel_ms_total": round(total, 4),
                          "ms": {k: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--profile", action="store_true", help="per-kernel breakdown of fnet / cnet at 384x512 instead")
    args = ap.parse_args()
    if args.profile:
        return profile()
    from goslam_b200.droid_net import UpdateModule
    from goslam_b200.modules.corr import CorrBlock
    from goslam_b200.modules.extractor import BasicEncoder
    from goslam_b200.motion_filter import MotionFilter
    torch.manual_seed(0)
    encs = {"fnet": BasicEncoder(128, "instance").to(DEV), "cnet": BasicEncoder(256, "none").to(DEV)}
    for H, W in SIZES:
        for B in (1, 16):
            x = torch.rand(1, B, 3, H, W, device=DEV)
            for tag, enc in encs.items():
                sd = {k: v.float() for k, v in enc.state_dict().items()}
                norm = enc.norm_fn

                def ours():
                    with torch.autocast("cuda"):
                        enc(x)

                def ref():
                    eo.basic_encoder(sd, norm, x[0], autocast=True)
                t_ours = timed(ours, args.windows, args.iters)
                t_ref = timed(ref, args.windows, args.iters)
                fl = B * encoder_flops(H, W, enc.out_dim)
                measure.emit({"what": tag, "H": H, "W": W, "B": B, "ours_ms": round(t_ours, 4),
                              "autocast_cudnn_ms": round(t_ref, 4), "speedup": round(t_ref / t_ours, 3),
                              "ours_tflops": round(fl / t_ours / 1e9, 2),
                              "share_of_f16_peak": round(fl / t_ours / 1e9 / (PEAK_F16 / 1e12), 4)})

    # one MotionFilter.track per frame, 384 x 512
    class Net:
        pass
    net = Net()
    net.fnet, net.cnet = encs["fnet"], encs["cnet"]
    net.update = eo.seeded_params(UpdateModule(), 3).to(DEV)
    fsd = {k: v.float() for k, v in net.fnet.state_dict().items()}
    csd = {k: v.float() for k, v in net.cnet.state_dict().items()}
    img = torch.rand(1, 3, 384, 512, device=DEV)
    intr = torch.tensor([500.0, 500.0, 256.0, 192.0], device=DEV)
    for path, thresh in (("accept", -1.0), ("reject", 1e9)):
        mf = MotionFilter(net, eo.RecordingVideo(), thresh=thresh, device=DEV)
        mf.track(0.0, img, intrinsic=intr)
        state = {}
        eo.track_step(fsd, csd, net.update, CorrBlock, state, img, thresh)

        def ours():
            mf.video.items.clear()
            mf.track(1.0, img, intrinsic=intr)

        def ref():
            eo.track_step(fsd, csd, net.update, CorrBlock, state, img, thresh)
        t_ours = timed(ours, args.windows, max(1, args.iters // 2))
        t_ref = timed(ref, args.windows, max(1, args.iters // 2))
        measure.emit({"what": "track", "path": path, "H": 384, "W": 512, "ours_ms": round(t_ours, 4),
                      "torch_restatement_ms": round(t_ref, 4), "speedup": round(t_ref / t_ours, 3)})


if __name__ == "__main__":
    main()
