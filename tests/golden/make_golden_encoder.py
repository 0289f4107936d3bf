"""Generate tests/golden/encoder.npz by running THE REFERENCE'S OWN PYTHON on the CPU:

  BasicEncoder.forward (src/modules/extractor.py) in float64 for norm_fn 'instance' (out 128) and 'none' (out 256),
  weights from the reference's own seeded kaiming init, (b, n) in (1, 1), (1, 2), (2, 3) at 48 x 64.  Each image's
  output is independent of its batch, so the three inputs are prefixes of one 6-image set and one output per image is
  stored.

  MotionFilter.track (src/motion_filter.py) on a 12-frame seeded synthetic sequence (oracle.encoder_oracle.sequence),
  float32 (autocast is off on the CPU): DroidNet's fnet / cnet / update of the reference, update weights from
  oracle.encoder_oracle.motion_update_params, droid_backends / lietorch replaced as in make_golden.py, the video a
  recording stub.  `thresh` is the one that keeps every frame's mean flow farthest from it (relative to it) while both
  decisions occur; that margin is asserted to be at least 5 %.

  The key names and shapes of pretrained/droid.pth's fnet.* / cnet.* entries (not their values).
Run:  python tests/golden/make_golden_encoder.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_golden as mg  # noqa: E402
from oracle import encoder_oracle as eo  # noqa: E402

ENC_SEED = {"instance": 11, "none": 12}
UPDATE_SEED = 21
MF_SEED = 5
DEPTH_SEED = 8
MF_MARGIN = 0.05


def gen_encoder(out):
    ext = mg.ref_import("src.modules.extractor")
    g = torch.Generator().manual_seed(3)
    H, W = 48, 64
    u8 = (torch.rand(6, 3, H, W, generator=g) * 255).round().to(torch.uint8)
    x = u8.double() / 255.0
    out["enc_image_u8"] = u8.numpy()
    for norm, dim in (("instance", 128), ("none", 256)):
        torch.manual_seed(ENC_SEED[norm])
        enc = ext.BasicEncoder(out_dim=dim, norm_fn=norm).double().eval()
        sd = enc.state_dict()
        out["enc_%s_wsum" % norm] = np.array([sd[k].double().sum().item() for k in sorted(sd)])
        full = None
        for b, n in ((1, 1), (1, 2), (2, 3)):
            with torch.no_grad():
                y = enc(x[: b * n].reshape(b, n, 3, H, W)).reshape(b * n, dim, H // 8, W // 8)
            if full is not None:
                assert (y[: full.shape[0]] - full).abs().max().item() < 1e-10
            full = y
        assert torch.allclose(eo.basic_encoder(sd, norm, x), full, rtol=1e-10, atol=1e-12)
        out["enc_%s_out" % norm] = full.float().numpy()


def run_motion_filter(thresh, images, intr, depth):
    dn = mg.ref_import("src.droid_net")
    mf_mod = mg.ref_import("src.motion_filter")
    torch.manual_seed(ENC_SEED["instance"])
    fnet = mg.ref_import("src.modules.extractor").BasicEncoder(out_dim=128, norm_fn="instance")
    torch.manual_seed(ENC_SEED["none"])
    cnet = mg.ref_import("src.modules.extractor").BasicEncoder(out_dim=256, norm_fn="none")
    update = eo.motion_update_params(dn.UpdateModule(), UPDATE_SEED)

    class Net:
        pass
    net = Net()
    net.fnet, net.cnet, net.update = fnet, cnet, update
    video = eo.RecordingVideo()
    mf = mf_mod.MotionFilter(net, video, thresh=thresh, device="cpu")
    deltas, decisions = [], []
    real_norm = torch.Tensor.norm

    def spy(self, *a, **k):           # the one `delta.norm(dim=-1)` of track
        r = real_norm(self, *a, **k)
        deltas.append(r.mean().item())
        return r
    for t in range(images.shape[0]):
        before = video.counter.value
        torch.Tensor.norm = spy
        try:
            mf.track(float(t), images[t:t + 1].clone(), depth=depth[t].clone(), intrinsic=intr.clone())
        finally:
            torch.Tensor.norm = real_norm
        decisions.append(int(video.counter.value > before))
        if t == 0:
            deltas.append(float("nan"))
        assert len(deltas) == t + 1
    return decisions, deltas, video, mf.count


def gen_motion_filter(out):
    images = eo.sequence(seed=MF_SEED)
    n, _, H, W = images.shape
    intr = torch.tensor([100.0, 101.0, 63.5, 64.0])
    g = torch.Generator().manual_seed(DEPTH_SEED)
    depth = (1.0 + 2.0 * torch.rand(n, H, W, generator=g)).float()
    _, probe, _, _ = run_motion_filter(1e9, images, intr, depth)       # every frame compared with frame 0
    best = None
    for thresh in np.linspace(min(probe[1:]), max(probe[1:]), 200):
        dec, dl, video, count = run_motion_filter(float(thresh), images, intr, depth)
        margin = float(np.min(np.abs(np.array(dl[1:]) - thresh)) / thresh)
        if 0 < sum(dec[1:]) < n - 1 and (best is None or margin > best[0]):
            best = (margin, float(thresh), dec, dl, video, count)
    margin, thresh, dec, dl, video, count = best
    assert margin >= MF_MARGIN, margin
    print("motion filter: thresh %.5f margin %.4f decisions %s deltas %s" % (thresh, margin, dec, np.round(dl, 4)))
    out["mf_thresh"] = np.float64(thresh)
    out["mf_shifts"] = np.array(eo.SHIFTS)
    out["mf_margin"] = np.float64(margin)
    out["mf_image_u8_sum"] = np.int64((images.double() * 255).round().sum().item())
    out["mf_decisions"] = np.array(dec)
    out["mf_delta_mean"] = np.array(dl)
    out["mf_count"] = np.int64(count)
    out["mf_intrinsic"] = intr.numpy()
    out["mf_timestamps"] = np.array([it[0] for it in video.items])
    out["mf_video_intrinsics"] = np.stack([it[5].numpy() for it in video.items])


def gen_droid_keys(out):
    sd = torch.load(os.path.join(mg.REF, "pretrained", "droid.pth"), map_location="cpu", weights_only=False)
    keys = sorted(k.replace("module.", "", 1) for k in sd if k.replace("module.", "", 1).split(".")[0] in ("fnet", "cnet"))
    shapes = {k.replace("module.", "", 1): tuple(v.shape) for k, v in sd.items()}
    out["droid_keys"] = np.array(keys)
    out["droid_shapes"] = np.array([";".join(map(str, shapes[k])) for k in keys])


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        raise SystemExit("needs the reference tree")
    mg.install_stubs()
    out = {"enc_seed_instance": np.int64(ENC_SEED["instance"]), "enc_seed_none": np.int64(ENC_SEED["none"])}
    gen_droid_keys(out)
    gen_encoder(out)
    gen_motion_filter(out)
    np.savez_compressed(os.path.join(HERE, "encoder.npz"), **out)
    print("wrote encoder.npz", os.path.getsize(os.path.join(HERE, "encoder.npz")))
