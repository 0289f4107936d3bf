"""`droid_backends` — the reference's native module name and its nine functions
(src/lib/droid.cpp:237-250), bound to libgoslam_b200.so through the C-ABI.

Same names, argument order, dtypes, in-place semantics and error behaviour as the pybind
module the reference builds from src/lib/*.cu:
  * every wrapper only checks contiguity (`TORCH_CHECK(x.is_contiguous())`, droid.cpp:84-85)
    and raises RuntimeError — plus a CUDA-device check, because there is no CPU path here;
  * `ba` mutates `poses` / `disps` in place through the caller's storage
    (src/lib/droid_kernels.cu:1389-1391,1420-1428) and returns [dx, dz];
  * the backward entry points exist and raise (inference is torch.no_grad, src/slam.py:45).

Install under the reference's import name with `goslam_b200.install()`.
"""
import torch

from . import _lib
from ._lib import contig as _contig


def _need_cuda(*ts):
    _lib.need_cuda("goslam_b200.droid_backends", *ts)


def _dtype_code(t):
    if t.dtype == torch.float16:
        return 1
    if t.dtype == torch.float32:
        return 0
    raise RuntimeError("correlation volume must be float16 or float32 (got %s)" % t.dtype)


# ----------------------------------------------------------------------------- correlation
def corr_index_forward(volume, coords, radius):
    """src/lib/droid.cpp:170-178 — volume [N,h1,w1,h2,w2], coords [N,2,h1,w1] -> [corr]."""
    _contig(volume=volume, coords=coords)
    _need_cuda(volume, coords)
    N, h1, w1, h2, w2 = volume.shape
    rd = 2 * radius + 1
    corr = torch.empty((N, rd, rd, h1, w1), dtype=volume.dtype, device=volume.device)
    _lib.call("corr_index_forward", volume, _dtype_code(volume), coords.float(), corr, N, h1, w1, h2, w2, int(radius))
    return [corr]


def corr_index_backward(volume, coords, corr_grad, radius):
    _contig(volume=volume, coords=coords, corr_grad=corr_grad)
    raise RuntimeError("corr_index_backward: training-only entry point, not part of the "
                       "inference hot path (GOSLAM_EUNSUPPORTED)")


def altcorr_forward(fmap1, fmap2, coords, radius):
    """src/lib/droid.cpp:193-203 — fmap1 [B,H,W,C], fmap2 [B,H2,W2,C], coords [B,S,H,W,2]."""
    _contig(fmap1=fmap1, fmap2=fmap2, coords=coords)
    _need_cuda(fmap1, fmap2, coords)
    if fmap1.dtype != torch.float32 or fmap2.dtype != torch.float32:
        raise RuntimeError("altcorr_forward expects float32 feature maps (as the reference calls it, "
                           "src/modules/corr.py:125)")
    B, H, W, C = fmap1.shape
    _, H2, W2, _ = fmap2.shape
    S = coords.shape[1]
    rd = 2 * radius + 1
    corr = torch.empty((B, S, rd * rd, H, W), dtype=torch.float32, device=fmap1.device)
    _lib.call("altcorr_forward", fmap1, fmap2, coords, corr, B, S, H, W, H2, W2, C, int(radius))
    return [corr]


def altcorr_backward(fmap1, fmap2, coords, corr_grad, radius):
    _contig(fmap1=fmap1, fmap2=fmap2, coords=coords, corr_grad=corr_grad)
    raise RuntimeError("altcorr_backward: training-only entry point, not part of the inference "
                       "hot path (GOSLAM_EUNSUPPORTED)")


# ----------------------------------------------------------------------------- geometry
def frame_distance(poses, disps, intrinsics, ii, jj, beta):
    """src/lib/droid.cpp:120-126 -> Tensor[K]."""
    _contig(poses=poses, disps=disps, intrinsics=intrinsics, ii=ii, jj=jj)
    _need_cuda(poses, disps, intrinsics, ii, jj)
    K = ii.shape[0]
    ht, wd = disps.shape[1], disps.shape[2]
    dist = torch.empty((K,), dtype=torch.float32, device=poses.device)
    _lib.call("frame_distance", poses, disps, intrinsics, ii, jj, dist, K, ht, wd, float(beta))
    return dist


def frame_distance_bidirectional(poses, disps, intrinsics, ii, jj, beta):
    """Not in the reference module: DepthVideo.distance(bidirectional=True) (src/depth_video.py:233-245)
    = 0.5 * (frame_distance(ii, jj) + frame_distance(jj, ii)) in one launch, bit-identical to that form."""
    _contig(poses=poses, disps=disps, intrinsics=intrinsics, ii=ii, jj=jj)
    _need_cuda(poses, disps, intrinsics, ii, jj)
    K = ii.shape[0]
    ht, wd = disps.shape[1], disps.shape[2]
    dist = torch.empty((K,), dtype=torch.float32, device=poses.device)
    _lib.call("frame_distance_bidir", poses, disps, intrinsics, ii, jj, dist, K, ht, wd, float(beta))
    return dist


def frame_distance_grid(poses, disps, intrinsics, r0, r1, c0, c1, k, beta):
    """Not in the reference module: the distance matrix Backend.ba builds (src/backend.py:31-44) over frames
    [r0, r1) x [c0, c1) -> Tensor[r1-r0, c1-c0].  Entry (i, j) equals frame_distance_bidirectional of the pair bit for
    bit where j - i <= k and is +inf elsewhere; no index tensors, and the poses are snapshot on the stream first."""
    _contig(poses=poses, disps=disps, intrinsics=intrinsics)
    _need_cuda(poses, disps, intrinsics)
    r0, r1, c0, c1 = int(r0), int(r1), int(c0), int(c1)
    if max(r1, c1) > min(poses.shape[0], disps.shape[0]):
        raise RuntimeError("frame_distance_grid: frame range [%d, %d) x [%d, %d) exceeds the video (%d frames)"
                           % (r0, r1, c0, c1, min(poses.shape[0], disps.shape[0])))
    ht, wd = disps.shape[1], disps.shape[2]
    dist = torch.empty((max(r1 - r0, 0), max(c1 - c0, 0)), dtype=torch.float32, device=poses.device)
    nbytes = _lib.load().goslam_frame_distance_grid_workspace_bytes(r0, r1, c0, c1)
    ws = _lib.workspace(nbytes, poses.device) if nbytes else None
    _lib.call("frame_distance_grid", poses, disps, intrinsics, r0, r1, c0, c1, int(k), ht, wd, float(beta), dist, ws,
              0 if ws is None else ws.numel())
    return dist


def projmap(poses, disps, intrinsics, ii, jj):
    """src/lib/droid.cpp:139-144 -> [coords(N,h,w,3), valid(N,h,w,1)]."""
    _contig(poses=poses, disps=disps, intrinsics=intrinsics, ii=ii, jj=jj)
    _need_cuda(poses, disps, intrinsics, ii, jj)
    K = ii.shape[0]
    ht, wd = disps.shape[1], disps.shape[2]
    coords = torch.empty((K, ht, wd, 3), dtype=torch.float32, device=poses.device)
    valid = torch.empty((K, ht, wd, 1), dtype=torch.float32, device=poses.device)
    _lib.call("projmap", poses, disps, intrinsics, ii, jj, coords, valid, K, ht, wd)
    return [coords, valid]


def iproj(poses, disps, intrinsics):
    """src/lib/droid.cpp:157-160 -> points [n,h,w,3]."""
    _contig(poses=poses, disps=disps, intrinsics=intrinsics)
    _need_cuda(poses, disps, intrinsics)
    num, ht, wd = disps.shape
    points = torch.empty((num, ht, wd, 3), dtype=torch.float32, device=disps.device)
    _lib.call("iproj", poses, disps, intrinsics, points, num, ht, wd)
    return points


def depth_filter(poses, disps, intrinsics, ix, thresh):
    """src/lib/droid.cpp:220-225 -> counter [n,h,w]."""
    _contig(poses=poses, disps=disps, intrinsics=intrinsics, ix=ix, thresh=thresh)
    _need_cuda(poses, disps, intrinsics, ix, thresh)
    K = ix.shape[0]
    num, ht, wd = disps.shape
    counter = torch.empty((K, ht, wd), dtype=torch.float32, device=disps.device)
    _lib.call("depth_filter", poses, disps, intrinsics, ix, thresh, counter, K, num, ht, wd)
    return counter


def reproject(poses, disps, intrinsics_all, ii, jj, want_valid=True):
    """Fused DepthVideo.reproject (src/depth_video.py:207-217): coords [1,N,h,w,2], valid [1,N,h,w,1].
    Not a droid_backends symbol upstream (the reference composes it from lietorch + torch ops)."""
    _contig(poses=poses, disps=disps, intrinsics_all=intrinsics_all, ii=ii, jj=jj)
    _need_cuda(poses, disps, intrinsics_all, ii, jj)
    K = ii.shape[0]
    ht, wd = disps.shape[1], disps.shape[2]
    coords = torch.empty((1, K, ht, wd, 2), dtype=torch.float32, device=poses.device)
    valid = torch.empty((1, K, ht, wd, 1), dtype=torch.float32, device=poses.device) if want_valid else None
    _lib.call("reproject", poses, disps, intrinsics_all, ii, jj, coords, valid, K, ht, wd)
    return coords, valid


def reproject_motion(poses, disps, intrinsics_all, ii, jj, target):
    """DepthVideo.reproject + FactorGraph's motion features in one launch (src/factor_graph.py:202-206):
    returns coords1 [1,N,h,w,2] and motion [1,N,4,h,w] = clamp(cat([coords1 - coords0, target - coords1]), +-64)."""
    _contig(poses=poses, disps=disps, intrinsics_all=intrinsics_all, ii=ii, jj=jj, target=target)
    _need_cuda(poses, disps, intrinsics_all, ii, jj, target)
    K = ii.shape[0]
    ht, wd = disps.shape[1], disps.shape[2]
    if target.dtype != torch.float32 or target.numel() != K * ht * wd * 2:
        raise RuntimeError("reproject_motion: target must be float32 [1, N, ht, wd, 2]")
    coords = torch.empty((1, K, ht, wd, 2), dtype=torch.float32, device=poses.device)
    motion = torch.empty((1, K, 4, ht, wd), dtype=torch.float32, device=poses.device)
    _lib.call("reproject_motion", poses, disps, intrinsics_all, ii, jj, target, coords, None, motion, K, ht, wd)
    return coords, motion


# ----------------------------------------------------------------------------- bundle adjustment
def ba(poses, disps, intrinsics, disps_sens, targets, weights, eta, ii, jj,
       t0, t1, iterations, lm, ep, motion_only, return_status=False, eta_by_frame=False):
    """src/lib/droid.cpp:88-117.  In place on poses [num,7] / disps [num,ht,wd].

    Returns [dx (t1-t0, 6), dz].  dz is laid out [num, ht*wd] indexed by FRAME id (rows of
    frames that carry no depth variable are zero) instead of the reference's packed
    [len(unique frames), ht*wd]: producing the packed shape needs the size of a device-side
    unique(), i.e. a host sync per call, and every caller in the reference discards the
    return value (src/depth_video.py:266).  dz is None when motion_only (reference: undefined
    tensor).

    eta: [M, ht, wd] with M = |unique([t0,t1) U ii)| rows in sorted frame order (what FactorGraph passes,
    src/factor_graph.py:236-238), or one row.  A different row count leaves the state untouched and
    reports status 2 (the reference raises a broadcast error there).  eta_by_frame=True (not in the
    reference): eta is [num, ht, wd] indexed by frame id."""
    _contig(targets=targets, weights=weights, poses=poses, disps=disps, intrinsics=intrinsics,
            disps_sens=disps_sens, ii=ii, jj=jj)
    _need_cuda(poses, disps, intrinsics, disps_sens, targets, weights, ii, jj)
    if ii.dtype != torch.int64 or jj.dtype != torch.int64:
        raise RuntimeError("ii / jj must be int64")
    dev = poses.device
    N = int(ii.shape[0])
    num, ht, wd = disps.shape
    t0, t1 = int(t0), int(t1)
    P = max(t1 - t0, 0)
    eta_c = None
    eta_rows = 0
    if not motion_only:
        eta_c = eta.contiguous().view(-1, ht * wd).float()
        eta_rows = int(eta_c.shape[0])
        if eta_by_frame:
            if eta_rows != num:
                raise RuntimeError("ba: eta_by_frame needs one row per frame (%d), got %d" % (num, eta_rows))
            eta_rows = -num
    dx = torch.zeros((P, 6), dtype=torch.float32, device=dev)
    dz = None if motion_only else torch.empty((num, ht * wd), dtype=torch.float32, device=dev)
    status = torch.zeros((max(int(iterations), 1),), dtype=torch.int32, device=dev)
    nbytes = _lib.load().goslam_ba_workspace_bytes(N, num, ht, wd, t0, t1)
    if nbytes == 0:
        raise RuntimeError("ba: invalid shapes (N=%d num=%d t0=%d t1=%d)" % (N, num, t0, t1))
    ws = _lib.workspace(nbytes, dev)
    _lib.call("ba", poses, disps, intrinsics, disps_sens, targets, weights, eta_c, eta_rows, ii, jj, N, num, ht, wd,
              t0, t1, int(iterations), float(lm), float(ep), int(bool(motion_only)), dx, dz, status, ws, ws.numel())
    if return_status:
        return [dx, dz, status]
    return [dx, dz]
