"""One factor graph sharded over the GPUs of a box (SURVEY.md §8e) — host-side logic.

Edges are partitioned BY SOURCE KEYFRAME `ii` (all outgoing edges of a frame live on one rank),
which keeps every per-pixel depth quantity (C, w, Q, the Schur products of a depth frame) local.
Per Gauss-Newton iteration the only exchange is ONE all-reduce(sum) of the reduced camera system
[(6P)^2 + 6P] float64 (0.57 MB at P = 63, latency bound on NVLink/NVSwitch); every rank then solves
the identical system redundantly, retracts all poses, back-substitutes the depth of the frames it
owns, and the updated disparity rows are re-replicated.

The kernels are reached through a small backend object so the same driver runs
  * on GPUs   : CudaBackend  -> goslam_ba_phase1 / goslam_ba_phase2 over NCCL,
  * in tests  : any object with the same two methods over gloo (tests/test_sharded_ba_gloo.py).
"""
import ctypes

import torch
import torch.distributed as dist


def shard_frames_by_edges(ii, num_frames, world):
    """Contiguous frame ranges [lo, hi) per rank, balanced by outgoing-edge count.
    Deterministic and identical on every rank (pure function of ii)."""
    counts = torch.bincount(ii.cpu().long(), minlength=num_frames).tolist()
    total = sum(counts)
    bounds, acc, lo = [], 0, 0
    for r in range(world):
        target = total * (r + 1) / world
        hi = lo
        while hi < num_frames and (acc + counts[hi] <= target or hi == lo and r < world - 1 and acc < target):
            acc += counts[hi]
            hi += 1
        if r == world - 1:
            hi = num_frames
        bounds.append((lo, hi))
        lo = hi
    return bounds


def local_edges(ii, lo, hi):
    return ((ii >= lo) & (ii < hi)).nonzero(as_tuple=False).reshape(-1)


class CudaBackend:
    """goslam_ba_phase1 / goslam_ba_phase2 on the current CUDA device.

    The backend OWNS its BA workspace: phase 2 reads what phase 1 left there (E, Q, w, the graph
    tables), so it must not be the shared grow-only scratch other calls may reallocate in between."""

    def __init__(self, poses, disps, intrinsics, disps_sens, t0, t1):
        from . import _lib
        self._lib = _lib
        self.poses, self.disps, self.intr, self.sens = poses, disps, intrinsics, disps_sens
        self.t0, self.t1 = int(t0), int(t1)
        self.num, self.ht, self.wd = disps.shape
        self._ws = None
        self.N = 0

    def _workspace(self, N):
        n = self._lib.load().goslam_ba_workspace_bytes(N, self.num, self.ht, self.wd, self.t0, self.t1)
        if n == 0:
            raise RuntimeError("sharded BA: invalid shapes (N=%d num=%d t0=%d t1=%d)" % (N, self.num, self.t0, self.t1))
        if self._ws is None or self._ws.numel() < n:
            self._ws = torch.empty(int(n), dtype=torch.uint8, device=self.poses.device)
        return self._ws

    def phase1(self, targets, weights, eta_by_frame, ii, jj, motion_only):
        self.N = int(ii.shape[0])
        ws = self._workspace(self.N)
        n_sys = self._lib.load().goslam_ba_system_doubles(self.t0, self.t1)
        system = torch.empty(n_sys, dtype=torch.float64, device=self.poses.device)
        # eta is FRAME-indexed here ([num, ht, wd]; eta_rows == num selects that form in the kernel),
        # so every rank reads the rows of its own frames whatever its local slot order is
        eta = eta_by_frame.reshape(self.num, -1)
        if not eta.is_contiguous() or eta.dtype != torch.float32:
            eta = eta.float().contiguous()
        self._lib.call("ba_phase1", self.poses, self.disps, self.intr, self.sens, targets, weights, eta, -int(eta.shape[0]),
                       ii, jj, self.N, self.num, self.ht, self.wd, self.t0, self.t1, int(bool(motion_only)), system, ws,
                       ws.numel())
        return system

    def phase2(self, system, lm, ep, motion_only, owner_lo, owner_hi, return_status=False):
        ws = self._workspace(self.N)
        dev = self.poses.device
        dx = torch.empty((self.t1 - self.t0, 6), dtype=torch.float32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev) if return_status else None
        self._lib.call("ba_phase2", self.poses, self.disps, system, self.N, self.num, self.ht, self.wd, self.t0, self.t1,
                       float(lm), float(ep), int(bool(motion_only)), int(owner_lo), int(owner_hi), dx, None, status, ws,
                       ws.numel())
        return (dx, status) if return_status else dx


class _PeerBuffer:
    """a device allocation the other ranks can map (goslam_peer_alloc), viewed as a torch tensor through the CUDA array
    interface (zero copy); freed when the object dies"""

    def __init__(self, lib_mod, shape, dtype, device):
        self._lib = lib_mod
        self.shape, self.dtype = tuple(int(x) for x in shape), dtype
        nbytes = max(1, int(torch.empty((), dtype=dtype).element_size() * int(torch.Size(self.shape).numel())))
        ptr, handle = ctypes.c_void_p(), (ctypes.c_ubyte * 64)()
        lib_mod.call("peer_alloc", nbytes, ctypes.byref(ptr), handle, device=device)
        self.ptr, self.handle, self.nbytes = int(ptr.value), bytes(handle), nbytes
        typestr = {torch.float32: "<f4", torch.float64: "<f8", torch.int32: "<i4", torch.uint8: "|u1"}[dtype]
        self.__cuda_array_interface__ = {"shape": self.shape, "typestr": typestr, "data": (self.ptr, False), "version": 2}
        self.tensor = torch.as_tensor(self, device=device)

    def __del__(self):
        try:
            self._lib.call("peer_free", self.ptr)
        except Exception:
            pass


class PeerLink:
    """Peer-memory plumbing of one sharded graph (one node, NVLink / NVSwitch), set up ONCE (collective call):
    every rank allocates its partial-system buffer, its replica of disps and its flag words in IPC-shareable memory,
    the 64-byte handles travel through one all_gather_object, and every rank maps the others' (goslam_ipc_open).
    After that an iteration needs no collective and no host synchronisation (include/goslam_b200.h, goslam_ba_peers)."""

    def __init__(self, disps_like, n_system, group=None):
        from . import _lib
        self._lib = _lib
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if self.world > 8:
            raise ValueError("peer-memory BA: at most 8 ranks (one NVSwitch node)")
        dev = disps_like.device
        self.system = _PeerBuffer(_lib, (int(n_system),), torch.float64, dev)
        self.disps = _PeerBuffer(_lib, disps_like.shape, torch.float32, dev)
        self.flags = _PeerBuffer(_lib, (2 * self.world,), torch.int32, dev)
        self.timeout = torch.zeros(1, dtype=torch.int32, device=dev)
        self.disps.tensor.copy_(disps_like)
        mine = {k: getattr(self, k).handle for k in ("system", "disps", "flags")}
        handles = [None] * self.world
        dist.all_gather_object(handles, mine, group=group)
        self._mapped = []
        self.ptrs = {k: [0] * self.world for k in mine}
        for r in range(self.world):
            for k in mine:
                if r == self.rank:
                    self.ptrs[k][r] = getattr(self, k).ptr
                else:
                    q = ctypes.c_void_p()
                    _lib.call("ipc_open", handles[r][k], ctypes.byref(q), device=dev)
                    self.ptrs[k][r] = int(q.value)
                    self._mapped.append(int(q.value))
        self.epoch = 0
        torch.cuda.synchronize(dev)
        dist.barrier(group=group)                 # every rank's buffers are zeroed and mapped before the first signal

    def struct(self):
        p = self._lib.BaPeers()
        p.world, p.rank = self.world, self.rank
        for r in range(self.world):
            p.system[r] = self.ptrs["system"][r]
            p.disps[r] = self.ptrs["disps"][r]
            p.flags[r] = self.ptrs["flags"][r]
        p.epoch = self.epoch
        p.timeout = self.timeout.data_ptr()
        return p

    def wait_idle(self):
        """stream-ordered: every rank has finished the last iteration (call before touching `disps.tensor` by hand)"""
        if self.epoch > 0 and self.world > 1:
            self._lib.call("ba_peers_wait", ctypes.byref(self.struct()), device=self.timeout.device)

    def close(self):
        torch.cuda.synchronize(self.timeout.device)
        dist.barrier(group=self.group)            # nobody still reads my buffers
        for q in self._mapped:
            self._lib.call("ipc_close", q)
        self._mapped = []


class PeerBackend(CudaBackend):
    """goslam_ba_phase1_peers / goslam_ba_phase2_peers: the exchange steps of the split form are done by the kernels over
    peer memory.  `link.disps.tensor` IS the replica of disps this backend reads and updates."""

    def __init__(self, poses, link, intrinsics, disps_sens, t0, t1):
        super().__init__(poses, link.disps.tensor, intrinsics, disps_sens, t0, t1)
        self.link = link

    def iteration(self, targets, weights, eta_by_frame, ii, jj, lm, ep, motion_only, owner_lo, owner_hi):
        self.N = int(ii.shape[0])
        ws = self._workspace(self.N)
        eta = eta_by_frame.reshape(self.num, -1)
        if not eta.is_contiguous() or eta.dtype != torch.float32:
            eta = eta.float().contiguous()
        self.link.epoch += 1
        peers = self.link.struct()
        dev = self.poses.device
        dx = torch.empty((self.t1 - self.t0, 6), dtype=torch.float32, device=dev)
        self._lib.call("ba_phase1_peers", self.poses, self.intr, self.sens, targets, weights, eta, -int(eta.shape[0]), ii,
                       jj, self.N, self.num, self.ht, self.wd, self.t0, self.t1, int(bool(motion_only)),
                       ctypes.byref(peers), ws, ws.numel())
        self._lib.call("ba_phase2_peers", self.poses, self.N, self.num, self.ht, self.wd, self.t0, self.t1, float(lm),
                       float(ep), int(bool(motion_only)), int(owner_lo), int(owner_hi), ctypes.byref(peers), dx, None, None,
                       ws, ws.numel())
        return dx


class RowExchange:
    """Re-replication of the disparity rows each rank owns after the back-substitution: ONE
    all-gather of [max_rows, hw] per rank (frame ranges are balanced by edge count, so they are padded
    to the widest range) followed by one indexed copy — not one broadcast per rank."""

    def __init__(self, disps, bounds, rank):
        self.bounds, self.rank = bounds, rank
        world = len(bounds)
        self.hw = disps[0].numel()
        self.max_rows = max(1, max(hi - lo for lo, hi in bounds))
        self.send = disps.new_zeros((self.max_rows, self.hw))
        self.recv = disps.new_zeros((world, self.max_rows, self.hw))
        frames, src = [], []
        for r, (lo, hi) in enumerate(bounds):
            if r == rank:
                continue
            frames += list(range(lo, hi))
            src += [r * self.max_rows + k for k in range(hi - lo)]
        self.frames = torch.tensor(frames, dtype=torch.long, device=disps.device)
        self.src = torch.tensor(src, dtype=torch.long, device=disps.device)

    def __call__(self, disps, group=None):
        lo, hi = self.bounds[self.rank]
        flat = disps.view(disps.shape[0], self.hw)
        if hi > lo:
            self.send[:hi - lo].copy_(flat[lo:hi])
        dist.all_gather(list(self.recv.unbind(0)), self.send, group=group)
        if self.frames.numel():
            flat.index_copy_(0, self.frames, self.recv.view(-1, self.hw).index_select(0, self.src))


def sharded_ba(backend, disps, targets, weights, eta_by_frame, ii, jj, iterations, lm, ep,
               motion_only=False, group=None):
    """Run `iterations` Gauss-Newton steps of ONE graph whose edges are sharded by source frame.

    `targets` / `weights` / `ii` / `jj` are the FULL (replicated) edge list; each rank picks its
    shard.  `disps` is the replicated [num, ht, wd] tensor the backend mutates; `eta_by_frame` is
    [num, ht, wd] (frame-indexed damping).  Per iteration: one all-reduce of the reduced camera
    system, one all-gather of the owned disparity rows.  Returns the last dx."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    num = disps.shape[0]
    bounds = shard_frames_by_edges(ii, num, world)
    lo, hi = bounds[rank]
    sel = local_edges(ii, lo, hi)
    tl, wl = targets[sel].contiguous(), weights[sel].contiguous()
    il, jl = ii[sel].contiguous(), jj[sel].contiguous()
    exchange = None if motion_only or world == 1 else RowExchange(disps, bounds, rank)
    dx = None
    for _ in range(iterations):
        system = backend.phase1(tl, wl, eta_by_frame, il, jl, motion_only)
        dist.all_reduce(system, op=dist.ReduceOp.SUM, group=group)        # exchange 1: reduced system
        dx = backend.phase2(system, lm, ep, motion_only, lo, hi)
        if exchange is not None:
            exchange(disps, group)                                        # exchange 2: owned rows
    return dx


class ShardedGraph:
    """ONE factor graph (global BA, config 4) sharded over the ranks of a process group — the multi-GPU form
    of FactorGraph.update_lowmem's per-step work without the update operator (SURVEY §8e):

        reproject + motion features of the LOCAL edges        (no exchange)
        windowed 4-level correlation of the LOCAL edges        (no exchange; feature pyramid replicated)
        dense BA: local linearisation + local reduced system -> all-reduce [(6P)^2 + 6P] f64 -> redundant
        solve + pose retraction -> depth back-substitution of the OWNED frames -> all-gather of those rows

    Edges are assigned by source frame (`shard_frames_by_edges`), state (poses, disps, intrinsics, sensor
    depth, feature maps) is replicated; every rank ends each update with identical poses and disps."""

    def __init__(self, poses, disps, intrinsics_all, disps_sens, fmaps, ii, jj, t0, t1, group=None, exchange="nccl"):
        """exchange = "nccl": all-reduce + all-gather per iteration (any backend torch.distributed has);
        exchange = "peer": the BA kernels exchange over peer memory themselves (one node; PeerLink) — then `self.disps` is
        the peer-mapped replica (a copy of the `disps` passed in), not the caller's tensor."""
        from .modules.corr import AltCorrBlock
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.link = None
        if exchange == "peer" and self.world > 1:
            from . import _lib
            n_sys = _lib.load().goslam_ba_system_doubles(int(t0), int(t1))
            self.link = PeerLink(disps, n_sys, group)
            disps = self.link.disps.tensor
        self.poses, self.disps, self.intr_all = poses, disps, intrinsics_all
        num = disps.shape[0]
        self.bounds = shard_frames_by_edges(ii, num, self.world)
        self.lo, self.hi = self.bounds[self.rank]
        self.sel = local_edges(ii, self.lo, self.hi)
        self.ii, self.jj = ii[self.sel].contiguous(), jj[self.sel].contiguous()
        if self.link is not None:
            self.backend = PeerBackend(poses, self.link, intrinsics_all[0].contiguous(), disps_sens, t0, t1)
        else:
            self.backend = CudaBackend(poses, disps, intrinsics_all[0].contiguous(), disps_sens, t0, t1)
        f, rig, ch, ht, wd = fmaps.shape
        self.rig = rig
        self.corr_op = AltCorrBlock(fmaps.view(1, f * rig, ch, ht, wd))
        self.f1 = (rig * self.ii).contiguous()
        self.f2 = (rig * self.jj + (self.ii == self.jj).long()).contiguous()
        self.exchange = RowExchange(disps, self.bounds, self.rank) if self.world > 1 and self.link is None else None

    def local(self, per_edge):
        """this rank's slice of a replicated per-edge tensor [N, ...]"""
        return per_edge[self.sel].contiguous()

    def features(self, target_local):
        """coords1, motion features and correlation features of the local edges (what the update operator eats)"""
        from . import droid_backends
        coords, motion = droid_backends.reproject_motion(self.poses, self.disps, self.intr_all, self.ii, self.jj,
                                                         target_local)
        return coords, motion, self.corr_op(coords, self.f1, self.f2)

    def bundle_adjust(self, target_planar_local, weight_planar_local, eta_by_frame, iters, lm, ep, motion_only=False):
        dx = None
        if self.link is not None:
            for _ in range(iters):
                dx = self.backend.iteration(target_planar_local, weight_planar_local, eta_by_frame, self.ii, self.jj, lm, ep,
                                            motion_only, self.lo, self.hi)
            return dx
        for _ in range(iters):
            system = self.backend.phase1(target_planar_local, weight_planar_local, eta_by_frame, self.ii, self.jj,
                                         motion_only)
            if self.world > 1:
                dist.all_reduce(system, op=dist.ReduceOp.SUM, group=self.group)
            dx = self.backend.phase2(system, lm, ep, motion_only, self.lo, self.hi)
            if self.exchange is not None and not motion_only:
                self.exchange(self.disps, self.group)
        return dx


def sharded_pairs(fn, ii, jj, group=None):
    """Embarrassingly parallel per-pair work (DepthVideo.distance over K frame pairs, SURVEY §8e row 3):
    the pair list is split evenly and contiguously over the ranks, each rank evaluates `fn(ii_part,
    jj_part) -> [k]` on its slice, and ONE all-gather of K floats rebuilds the replicated result.
    `fn` is droid_backends.frame_distance bound to the replicated poses / disps on GPUs (any callable
    with that contract in the gloo tests)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    K = int(ii.shape[0])
    per = (K + world - 1) // world
    lo, hi = min(K, rank * per), min(K, (rank + 1) * per)
    part = fn(ii[lo:hi].contiguous(), jj[lo:hi].contiguous()) if hi > lo else ii.new_zeros(0, dtype=torch.float32)
    padded = torch.zeros(per, dtype=torch.float32, device=part.device)
    padded[:hi - lo] = part.float()
    gathered = [torch.empty_like(padded) for _ in range(world)]
    dist.all_gather(gathered, padded, group=group)
    return torch.cat(gathered)[:K]


def sharded_distance(poses, disps, intrinsics, ii, jj, beta=0.3, bidirectional=True, group=None):
    """DepthVideo.distance (src/depth_video.py:219-255) with the pair list sharded over the ranks."""
    from . import droid_backends

    def one_way(a, b):
        return droid_backends.frame_distance(poses, disps, intrinsics, a, b, beta)

    if not bidirectional:
        return sharded_pairs(one_way, ii, jj, group)
    return sharded_pairs(lambda a, b: droid_backends.frame_distance_bidirectional(poses, disps, intrinsics, a, b, beta),
                         ii, jj, group)


# ---------------------------------------------------------------------------------------------------------------
# Data-parallel mapping step (SURVEY 8f-3: "multi-GPU adds an all-reduce of grid grads").  Rays are independent: every rank
# renders and back-propagates its slice of the ray batch; the losses are written in SUM form over the GLOBAL counts so that the
# SUM of the ranks' gradients is exactly the gradient of the reference's single-process loss on the whole batch
# (src/mapping.py:97-128), whatever the split and however many rays of a slice have no sensor depth.
# ---------------------------------------------------------------------------------------------------------------
def _world_rank(group=None):
    """(world, rank); a process that never initialised torch.distributed is one rank"""
    if not dist.is_available() or not dist.is_initialized():
        return 1, 0
    return dist.get_world_size(group), dist.get_rank(group)


def ray_slice(n_rays, group=None):
    """contiguous, balanced slice [lo, hi) of a ray batch for this rank"""
    world, rank = _world_rank(group)
    per, rem = divmod(int(n_rays), world)
    lo = rank * per + min(rank, rem)
    return lo, lo + per + (1 if rank < rem else 0)


def mapping_loss_local(net, out, rays_color, rays_depth, n_rays_global, w_color, w_sdf, w_eikonal, uncertainty_based=True,
                       group=None):
    """this rank's share of Mapper.optimize_map's total loss (src/mapping.py:97-128) on its ray slice: color / depth / sdf
    terms are sums over the slice's valid rays divided by the GLOBAL number of valid rays (one tiny all-reduce of the
    count), the eikonal term is the slice's gradient_error weighted by its share of the samples.  Summed over the ranks
    this IS the reference's loss on the whole batch; so are the gradients after `allreduce_gradients`."""
    depth = rays_depth.reshape(-1, 1)
    valid = (depth > 0).reshape(-1)
    n_valid = valid.sum().to(torch.float32).reshape(1)
    if _world_rank(group)[0] > 1:
        dist.all_reduce(n_valid, op=dist.ReduceOp.SUM, group=group)
    n_valid = n_valid.clamp_min(1.0)
    unc = 1.0 / torch.sqrt(out["depth_variance"][valid].detach() + 1e-10)
    if not uncertainty_based:
        unc = torch.ones_like(unc)
    total = torch.abs(out["color"][valid] - rays_color[valid]).sum() / (3.0 * n_valid) * w_color
    total = total + (torch.abs(out["depth"][valid] - depth[valid]) * unc).sum() / n_valid
    if w_sdf > 0 and bool(valid.any()):
        n_local = valid.sum().to(torch.float32)
        sdf_loss, sparse_loss = net.compute_sdf_error(sdf=out["sdf"][valid], z_vals=out["z_vals"][valid], gt_depth=depth[valid])
        total = total + (sdf_loss + sparse_loss) * (n_local / n_valid) * w_sdf          # its means are over the local valid rays
    if w_eikonal > 0:
        total = total + w_eikonal * out["gradient_error"].mean() * (float(rays_depth.numel()) / float(n_rays_global))
    return total.reshape(())


def broadcast_parameters(params, src=0, group=None):
    """every replica starts from rank `src`'s parameters (also the ones no loss term touches: weight decay moves them)"""
    if _world_rank(group)[0] == 1:
        return
    with torch.no_grad():
        for p in params:
            dist.broadcast(p.data, src=src, group=group)


def allreduce_gradients(params, group=None):
    """SUM the .grad of `params` over the ranks: the small tensors travel as one flat buffer, every tensor above 1 M elements
    (the 12.6 M-entry hash grid) on its own.  Parameters without a gradient on some rank count as zero."""
    if _world_rank(group)[0] == 1:
        return
    params = [p for p in params]
    small = [p for p in params if p.numel() <= (1 << 20)]
    for p in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)
    if small:
        flat = torch.cat([p.grad.reshape(-1) for p in small])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        o = 0
        for p in small:
            p.grad.copy_(flat[o:o + p.numel()].view_as(p.grad))
            o += p.numel()
    for p in params:
        if p.numel() > (1 << 20):
            dist.all_reduce(p.grad, op=dist.ReduceOp.SUM, group=group)
