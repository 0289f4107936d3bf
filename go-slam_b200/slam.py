"""Drop-in for the end of src/slam.py: `SLAM.terminate` with the trajectory error computed by the library, so a run
finishes and reports its APE without evo.

    import src.slam
    import goslam_b200.slam
    src.slam.SLAM.terminate = goslam_b200.slam.terminate

`ape(ref_poses, est_positions)` is evo's main_ape.ape(traj_ref, traj_est, pose_relation=translation_part, align=True,
correct_scale=True) on CUDA tensors: one library call (goslam_ape_sim3, DESIGN §3.19) and one read of its result.  The
rules are restated in oracle/ape_oracle.py.

Differences from evo: everything is f64 (evo keeps parts of an f32 estimate's arithmetic in f32); failures raise
ValueError (evo raises GeometryException / LinAlgError); timestamps, which do not enter the translation APE, are not
taken; a non-finite estimate in a kept row raises instead of propagating NaN; fewer than three kept rows are degenerate
whatever the rounding of their covariance.
"""
import os

import numpy as np
import torch

from . import _lib
from .lietorch import SE3

TITLE = "APE w.r.t. translation part (m)\n(with Sim(3) Umeyama alignment)"
STATS = ("rmse", "mean", "median", "std", "min", "max", "sse")     # the library's order (include/goslam_b200.h)
MESSAGES = {1: "APE: no reference pose has finite entries",
            2: "APE: an estimated position of a kept row is not finite",
            3: "Degenerate covariance rank, Umeyama alignment is not possible"}
OUT, SIM3, KEPT, STAT0, SINGULAR = 28, 2, 1, 18, 25


class _Arrays(dict):
    """evo's np_arrays: 'alignment_transformation_sim3' at once; 'error_array' is copied from the device when first
    read, so a caller that only needs the text and the alignment moves nothing else across PCIe"""

    def __init__(self, sim3, errors):
        super().__init__(alignment_transformation_sim3=sim3)
        self._errors = errors

    def __missing__(self, key):
        if key != "error_array":
            raise KeyError(key)
        self["error_array"] = value = self._errors.cpu().numpy()
        return value


class ApeResult:
    """the parts of evo's Result that callers of main_ape.ape read: stats, np_arrays, info['title'], pretty_str().
    `errors` is the kept rows' error array on the device, `singular_values` the covariance's d."""

    def __init__(self, stats, sim3, errors, singular_values):
        self.info = {"title": TITLE}
        self.stats = stats
        self.errors = errors
        self.singular_values = singular_values
        self.np_arrays = _Arrays(sim3, errors)

    def pretty_str(self, title=True, stats=True):
        text = ""
        if title:
            text += "{}\n\n".format(self.info["title"])
        if stats:
            for name, val in sorted(self.stats.items()):
                text += "{:>10}\t{:.6f}\n".format(name, val)
        return text


@torch.no_grad()
def ape(ref_poses, est_positions):
    """APE w.r.t. the translation part after a Sim(3) Umeyama alignment of est_positions [n,3] onto the translations
    of ref_poses [n,4,4] (c2w).  Both CUDA tensors of any float dtype, widened to f64 on the device; reference rows
    whose entries sum to NaN or Inf are skipped.  Raises ValueError when no row is kept, a kept estimate is not finite
    or the alignment is degenerate.  One host synchronisation."""
    ref, est = torch.as_tensor(ref_poses), torch.as_tensor(est_positions)
    if not (ref.is_cuda and est.is_cuda):
        raise RuntimeError("ape: CUDA tensors required (no CPU fallback)")
    if ref.device != est.device:
        raise ValueError("ape: poses and positions on different devices")
    if not (ref.is_floating_point() and est.is_floating_point()):
        raise ValueError("ape: float tensors required, got %s and %s" % (ref.dtype, est.dtype))
    n = ref.shape[0] if ref.dim() == 3 else -1
    if tuple(ref.shape[1:]) != (4, 4) or tuple(est.shape) != (n, 3):
        raise ValueError("ape: ref_poses must be [n,4,4] and est_positions [n,3], got %s and %s"
                         % (tuple(ref.shape), tuple(est.shape)))
    dev = ref.device
    ref = ref.to(torch.float64).contiguous()
    est = est.to(torch.float64).contiguous()
    nbytes = _lib.load().goslam_ape_workspace_bytes(n)
    if nbytes == 0:
        raise ValueError("ape: %d poses is more than the library takes" % n)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out = torch.empty(OUT, dtype=torch.float64, device=dev)
    errors = torch.empty(max(n, 1), dtype=torch.float64, device=dev)
    _lib.call("ape_sim3", est, ref, n, ws, nbytes, out, errors)
    host = out.cpu().numpy()
    status = int(host[0])
    if status != 0:
        raise ValueError(MESSAGES.get(status, "APE: status %d" % status))
    stats = {k: float(v) for k, v in zip(STATS, host[STAT0:STAT0 + 7])}
    return ApeResult(stats, host[SIM3:SIM3 + 16].reshape(4, 4).copy(), errors[:int(host[KEPT])],
                     host[SINGULAR:SINGULAR + 3].copy())


def terminate(self, rank, stream=None):
    """ fill poses for non-keyframe images and evaluate (src/slam.py:289-370, with the APE on the device) """

    while (self.optimizing_finished < 1):
        if self.num_running_thread == 1 and self.tracking_finished > 0:
            break

    os.makedirs(f'{self.output}/checkpoints/', exist_ok=True)
    torch.save({
        'mapping_net': self.mapping_net.state_dict(),
        'tracking_net': self.net.state_dict(),
        'keyframe_timestamps': self.video.timestamp,
    }, f'{self.output}/checkpoints/go.ckpt')

    do_evaluation = True
    if do_evaluation:
        print("#" * 20 + f" Results for {stream.input_folder} ...")

        camera_trajectory = self.traj_filler(stream)  # w2cs
        w2w = SE3(self.video.pose_compensate[0].clone().unsqueeze(dim=0)).to(camera_trajectory.device)
        camera_trajectory = w2w * camera_trajectory.inv()
        traj_est = camera_trajectory.data                                  # stays on the device
        estimate_c2w_list = camera_trajectory.matrix().data.cpu()
        np.save(
            f'{self.output}/checkpoints/est_poses.npy',
            estimate_c2w_list.numpy(),  # c2ws
        )

        if stream.poses is None:  # for eth3d submission
            if stream.image_timestamps is not None:
                submission_txt = f'{self.output}/submission.txt'
                with open(submission_txt, 'w') as fp:
                    for tm, pos in zip(stream.image_timestamps, traj_est.cpu().numpy().tolist()):
                        line = f'{tm:.9f}'
                        for ps in pos:  # timestamp tx ty tz qx qy qz qw
                            line += f' {ps:.14f}'
                        fp.write(line + '\n')
                print('Poses are save to {}!'.format(submission_txt))

            print("Terminate: no GT poses found!")
            trans_init = None
            gt_c2w_list = None
        else:
            n = len(stream.poses)
            if n > traj_est.shape[0]:
                raise ValueError("terminate: %d reference poses but %d estimated poses" % (n, traj_est.shape[0]))
            traj_ref = []
            for i in range(n):
                val = stream.poses[i].sum()
                if np.isnan(val) or np.isinf(val):
                    print(f'Nan or Inf found in gt poses, skipping {i}th pose!')
                    continue
                traj_ref.append(stream.poses[i])
            gt_c2w_list = torch.from_numpy(np.stack(traj_ref, axis=0)) if traj_ref else None

            # the poses go up once as f64; row i pairs with traj_est[i], the device skips the same rows
            ref = torch.from_numpy(np.stack([np.asarray(p, np.float64) for p in stream.poses], axis=0))
            result = ape(ref.to(traj_est.device), traj_est[:n, :3])

            out_path = f'{self.output}/metrics_traj.txt'
            with open(out_path, 'a') as fp:
                fp.write(result.pretty_str())
            trans_init = result.np_arrays['alignment_transformation_sim3']

        if self.meshing_finished > 0 and (not self.only_tracking):
            self.mesher(the_end=True, estimate_c2w_list=estimate_c2w_list, gt_c2w_list=gt_c2w_list, trans_init=trans_init)

    print("Terminate: Done!")
