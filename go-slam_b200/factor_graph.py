"""`FactorGraph` — the frontend / backend / trajectory-filler factor graph with the reference's constructor,
attributes and method signatures (src/factor_graph.py:9-450), built on the sm_90a kernels.

Same state machine (edges `ii/jj/age`, stored inactive edges, bad edges, per-edge `net/inp/target/weight`,
per-frame `damping`), different mechanics:
  * the correlation pyramid of the `volume` implementation lives in a slot pool (CorrPool): add_factors
    builds the new edges' volumes straight from the video's feature maps with the wgmma kernel and
    appends slot ids; rm_factors hands slots back.  The reference copies the whole pyramid on both
    (torch.cat / boolean mask, src/modules/corr.py:55-65);
  * edge de-duplication, t0/t1 defaults, the inactive-edge window, unique source frames and the 13-frame
    chunking of update_lowmem are decided on HOST mirrors of the edge lists that are maintained with
    every edit — no per-edge `.item()` round trips (src/factor_graph.py:44-54 does two per stored edge);
  * reproject + motion features are one launch (goslam_reproject_motion), the 4-level lookup one launch,
    all BA iterations one cooperative launch (or the cluster-Cholesky driver for global BA), the damping
    vector is handed to BA frame-indexed, so no `unique`/gather on the device;
  * edge selection of add_proximity_factors runs in one kernel (graph.proximity_edges).
`update_op` is injected exactly as in the reference (DroidNet.update); it is the one stage that stays
PyTorch (SURVEY §8f-4).
"""
import numpy as np
import torch

from . import droid_backends, graph as graph_ops
from .modules.corr import AltCorrBlock, CorrBlock, CorrPool, fmaps_to_kmajor


class FactorGraph:
    def __init__(self, video, update_op, device="cuda:0", corr_impl="volume", max_factors=-1.0, upsample=False):
        self.video, self.update_op, self.device = video, update_op, device
        self.max_factors, self.corr_impl, self.upsample = max_factors, corr_impl, upsample
        self.ht, self.wd = video.ht // 8, video.wd // 8
        ht, wd = self.ht, self.wd
        y, x = torch.meshgrid(torch.arange(ht, device=device).float(), torch.arange(wd, device=device).float(),
                              indexing="ij")
        self.coords0 = torch.stack([x, y], dim=-1)                               # [ht, wd, 2]

        def no_edges():
            return torch.zeros(0, dtype=torch.long, device=device)

        def no_flow():
            return torch.zeros([1, 0, ht, wd, 2], device=device, dtype=torch.float)
        self.ii, self.jj, self.age = no_edges(), no_edges(), no_edges()
        self.corr, self.net, self.inp = None, None, None
        self.damping = 1e-6 * torch.ones_like(video.disps)
        self.target, self.weight = no_flow(), no_flow()
        self.ii_inac, self.jj_inac, self.ii_bad, self.jj_bad = no_edges(), no_edges(), no_edges(), no_edges()
        self.target_inac, self.weight_inac = no_flow(), no_flow()
        # host mirrors of the edge lists (kept in step by every method that edits them)
        self._h = {k: np.zeros(0, np.int64) for k in ("ii", "jj", "ii_inac", "jj_inac")}
        self._pool = None
        self._kmajor = None
        self._eta = None
        self._uniq = None                     # cached (unique source frames on host, on device)

    # ------------------------------------------------------------------------------------ helpers
    def _as_edges(self, x):
        if not isinstance(x, torch.Tensor):
            x = torch.tensor(x, dtype=torch.long, device=self.device)
        return x.to(device=self.device, dtype=torch.long).reshape(-1)

    def _set_edges(self, ii, jj, age):
        self.ii, self.jj, self.age = ii, jj, age
        self._uniq = None

    def _unique_sources(self):
        """sorted unique source frames of the active edges: (host array, device tensor)"""
        if self._uniq is None:
            u = np.unique(self._h["ii"])
            self._uniq = (u, torch.from_numpy(u).to(self.device))
        return self._uniq

    def _pool_for(self, n_new):
        """slot pool for the correlation pyramids: FactorGraph.max_factors slots when the graph is bounded
        (+ the batch that may overshoot before eviction), doubling otherwise"""
        need = self._h["ii"].size + n_new
        if self._pool is None:
            cap = int(self.max_factors) + 8 if self.max_factors > 0 else 32
            self._pool = CorrPool(max(cap, need), self.ht, self.wd, device=self.device)
        if self._pool.free_slots < n_new:
            self._pool.grow(max(2 * self._pool.capacity, self._pool.capacity - self._pool.free_slots + n_new))
        return self._pool

    def _kmajor_rows(self, frames):
        """K-major, /4-scaled copies of the feature maps of frames [lo, hi) that the new edges touch, in a
        video-sized cache (re-laid every call: a few MB, and always current with video.fmaps)"""
        fm = self.video.fmaps
        rig = fm.shape[1]
        if self._kmajor is None:
            self._kmajor = torch.empty((fm.shape[0] * rig, self.ht * self.wd, 128), dtype=torch.float16, device=self.device)
        lo, hi = int(frames.min()), int(frames.max()) + 1
        fmaps_to_kmajor(fm[lo:hi], out=self._kmajor[lo * rig:hi * rig])
        return self._kmajor, rig

    def _filter_repeated_edges(self, ii, jj):
        """drop candidates the graph already holds, active or inactive (src/factor_graph.py:44-54)"""
        return graph_ops.filter_repeated_edges(ii, jj, self.ii, self.jj, self.ii_inac, self.jj_inac)

    def print_edges(self):
        order = np.argsort(self._h["ii"], kind="stable")
        w = torch.mean(self.weight, dim=[0, 2, 3, 4]).cpu().numpy()[order]
        msg = "INFO: Edges of Graph: \n Start  End    Weight\n"
        for i, j, c in zip(self._h["ii"][order], self._h["jj"][order], w):
            msg += f" {i:05d}, {j:05d}, {c:.4f}\n"
        print(msg)

    def filter_edges(self):
        """remove edges the update operator gives (almost) no weight (src/factor_graph.py:70-77)"""
        conf = torch.mean(self.weight, dim=[0, 2, 3, 4])
        mask = (torch.abs(self.ii - self.jj) > 2) & (conf < 1e-3)
        self.ii_bad = torch.cat([self.ii_bad, self.ii[mask]])
        self.jj_bad = torch.cat([self.jj_bad, self.jj[mask]])
        self.rm_factors(mask, store=False)

    def clear_edges(self):
        self.rm_factors(self.ii >= 0)
        self.net = None
        self.inp = None

    @torch.no_grad()
    def adopt_edges(self, other):
        """take copies of another graph's active edges and their state: ii / jj / age / net / target / weight, each
        only where `other` has it (what Backend.loop_ba does with setattr + deepcopy, src/backend.py:151-156).  The
        host mirrors come from `other`'s own when it is a goslam_b200.FactorGraph, otherwise from one device->host
        copy of its edge lists; `other` is left untouched."""
        ii, jj, age = (getattr(other, k) for k in ("ii", "jj", "age"))
        self._set_edges(self.ii if ii is None else ii.clone(), self.jj if jj is None else jj.clone(),
                        self.age if age is None else age.clone())
        for k in ("net", "target", "weight"):
            val = getattr(other, k)
            if val is not None:
                setattr(self, k, val.clone())
        if isinstance(other, FactorGraph):
            self._h["ii"], self._h["jj"] = other._h["ii"].copy(), other._h["jj"].copy()
        else:
            h = torch.stack([self.ii.long(), self.jj.long()]).cpu().numpy()
            self._h["ii"], self._h["jj"] = h[0].copy(), h[1].copy()

    # ------------------------------------------------------------------------------------ edits
    @torch.no_grad()
    def add_factors(self, ii, jj, remove=False):
        """add edges (src/factor_graph.py:85-131)"""
        ii, jj = self._as_edges(ii), self._as_edges(jj)
        ii, jj = self._filter_repeated_edges(ii, jj)
        n_new = int(ii.shape[0])                                   # the one sync of this call (boolean compaction)
        if n_new == 0:
            return
        # limit on the number of factors: evict by age (positions taken from the age order, as the reference does)
        if self.max_factors > 0 and self._h["ii"].size + n_new > self.max_factors and self.corr is not None and remove:
            order = torch.argsort(self.age, descending=False, stable=True).cpu()
            self.rm_factors(order >= self.max_factors - n_new, store=True)
        ii_h, jj_h = ii.cpu().numpy(), jj.cpu().numpy()
        net = self.video.nets[ii].to(self.device).unsqueeze(0)
        if self.corr_impl == "volume":
            km, rig = self._kmajor_rows(np.concatenate([ii_h, jj_h]))
            corr = CorrBlock.from_video(km, ii, jj, self.ht, self.wd, rig=rig, pool=self._pool_for(n_new))
            self.corr = corr if self.corr is None else self.corr.cat(corr)
            inp = self.video.inps[ii].to(self.device).unsqueeze(0)
            self.inp = inp if self.inp is None else torch.cat([self.inp, inp], dim=1)
        target, _ = self.video.reproject(ii, jj)                   # initial flow target: the current reprojection
        self._h["ii"] = np.concatenate([self._h["ii"], ii_h])
        self._h["jj"] = np.concatenate([self._h["jj"], jj_h])
        self._set_edges(torch.cat([self.ii, ii]), torch.cat([self.jj, jj]), torch.cat([self.age, torch.zeros_like(ii)]))
        self.net = net if self.net is None else torch.cat([self.net, net], dim=1)
        self.target = torch.cat([self.target, target], dim=1)
        self.weight = torch.cat([self.weight, torch.zeros_like(target)], dim=1)

    @torch.no_grad()
    def rm_factors(self, mask, store=False):
        """drop the masked edges, optionally keeping their estimates as inactive factors (:134-160)"""
        mask = mask.to(torch.bool)
        mask_h = mask.cpu().numpy()
        mask = mask.to(self.ii.device)
        if store:
            self.ii_inac = torch.cat([self.ii_inac, self.ii[mask]])
            self.jj_inac = torch.cat([self.jj_inac, self.jj[mask]])
            self.target_inac = torch.cat([self.target_inac, self.target[:, mask]], dim=1)
            self.weight_inac = torch.cat([self.weight_inac, self.weight[:, mask]], dim=1)
            self._h["ii_inac"] = np.concatenate([self._h["ii_inac"], self._h["ii"][mask_h]])
            self._h["jj_inac"] = np.concatenate([self._h["jj_inac"], self._h["jj"][mask_h]])
        keep = ~mask
        self._h["ii"], self._h["jj"] = self._h["ii"][~mask_h], self._h["jj"][~mask_h]
        self._set_edges(self.ii[keep], self.jj[keep], self.age[keep])
        if self.corr_impl == "volume" and self.corr is not None:
            self.corr = self.corr[torch.from_numpy(~mask_h)]       # slot table edit, O(edges)
        if self.net is not None:
            self.net = self.net[:, keep]
        if self.inp is not None:
            self.inp = self.inp[:, keep]
        self.target = self.target[:, keep]
        self.weight = self.weight[:, keep]

    _SHIFTED = ("timestamp", "images", "dirty", "red", "poses", "poses_gt", "disps", "disps_sens", "disps_up",
                "depths_gt", "intrinsics", "poses_filtered", "disps_filtered", "mask_filtered", "update_priority",
                "nets", "inps", "fmaps")

    @torch.no_grad()
    def rm_keyframe(self, ix):
        """drop keyframe ix: its slot takes the next frame's data, edge indices above it shift down, its
        edges go (src/factor_graph.py:162-196)"""
        v = self.video
        with v.get_lock():
            for name in self._SHIFTED:
                buf = getattr(v, name)
                buf[ix] = buf[ix + 1]
        h = self._h
        m = (h["ii_inac"] == ix) | (h["jj_inac"] == ix)
        self.ii_inac[self.ii_inac >= ix] -= 1
        self.jj_inac[self.jj_inac >= ix] -= 1
        h["ii_inac"] = h["ii_inac"] - (h["ii_inac"] >= ix)
        h["jj_inac"] = h["jj_inac"] - (h["jj_inac"] >= ix)
        if m.any():
            keep = torch.from_numpy(~m).to(self.device)
            self.ii_inac, self.jj_inac = self.ii_inac[keep], self.jj_inac[keep]
            self.target_inac, self.weight_inac = self.target_inac[:, keep], self.weight_inac[:, keep]
            h["ii_inac"], h["jj_inac"] = h["ii_inac"][~m], h["jj_inac"][~m]
        m = (h["ii"] == ix) | (h["jj"] == ix)
        self.ii[self.ii >= ix] -= 1
        self.jj[self.jj >= ix] -= 1
        h["ii"] = h["ii"] - (h["ii"] >= ix)
        h["jj"] = h["jj"] - (h["jj"] >= ix)
        self._uniq = None
        self.rm_factors(torch.from_numpy(m).to(self.device), store=False)

    # ------------------------------------------------------------------------------------ updates
    def _window(self, t0, t1):
        """default optimisation window (first keyframe fixed), from the host mirrors"""
        if t0 is None:
            t0 = max(1, int(self._h["ii"].min()) + 1)
        t0 = max(1, t0)
        if t1 is None:
            t1 = max(int(self._h["ii"].max()), int(self._h["jj"].max())) + 1
        return t0, t1

    def _frame_eta(self, EPS):
        """0.2 * damping + EPS for every frame (src/factor_graph.py:236-238 gathers the rows BA uses; BA takes the
        frame-indexed form directly, so no unique()/gather is needed)"""
        if self._eta is None:
            self._eta = torch.empty_like(self.damping)
        torch.mul(self.damping, 0.2, out=self._eta)
        return self._eta.add_(EPS)

    @staticmethod
    def _planar(x, ht, wd):
        return x.view(-1, ht, wd, 2).permute(0, 3, 1, 2).contiguous()

    def _bundle_adjust(self, target, weight, ii, jj, t0, t1, iters, lm, ep, motion_only, ba_type, EPS):
        tgt, wgt = self._planar(target, self.ht, self.wd), self._planar(weight, self.ht, self.wd)
        kw = dict(t0=t0, t1=t1, iters=iters, lm=lm, ep=ep, motion_only=motion_only, ba_type=ba_type)
        if getattr(self.video, "takes_frame_eta", False):
            self.video.ba(tgt, wgt, self._frame_eta(EPS), ii, jj, eta_by_frame=True, **kw)
        else:
            # a video with the reference's ba() signature: pack the rows BA reads, in sorted frame order
            # (src/factor_graph.py:236-238), from the host mirror of the edge list
            src = ii.cpu().numpy() if ii is not self.ii else self._h["ii"]
            rows = np.unique(np.concatenate([np.arange(t0, t1), src]))
            eta = 0.2 * self.damping[torch.from_numpy(rows).to(self.device)].contiguous() + EPS
            self.video.ba(tgt, wgt, eta, ii, jj, **kw)

    def _hint_sources(self, ii_host):
        """tell an update operator that can use it (goslam_b200.UpdateModule) which source-frame slot each edge has —
        GraphAgg's unique(ii, return_inverse) — from the host mirror instead of a device-side unique + sync"""
        hint = getattr(self.update_op, "set_source_frames", None)
        if hint is not None:
            frames, slot = np.unique(ii_host, return_inverse=True)
            hint(torch.from_numpy(frames), torch.from_numpy(slot.astype(np.int32)).to(self.device))

    def _features(self, ii, jj, target):
        """coords1 [1,N,h,w,2] and the clamped motion features [1,N,4,h,w] in one launch"""
        v = self.video
        return droid_backends.reproject_motion(v.poses, v.disps, v.intrinsics, ii, jj, target.contiguous())

    @torch.no_grad()
    def update(self, t0=None, t1=None, iters=2, use_inactive=False, EPS=1e-7, motion_only=False):
        """one update-operator step + dense BA on the graph (src/factor_graph.py:198-252)"""
        coords1, motion = self._features(self.ii, self.jj, self.target)
        corr = self.corr(coords1)
        self._hint_sources(self._h["ii"])
        with torch.autocast("cuda", enabled=True):
            self.net, delta, weight, damping, upmask = self.update_op(self.net, self.inp, corr, motion, self.ii, self.jj)
        t0, t1 = self._window(t0, t1)
        self.target = coords1 + delta.float()
        self.weight = weight.float()
        _, uniq = self._unique_sources()
        self.damping[uniq] = damping
        ii, jj, target, weight = self.ii, self.jj, self.target, self.weight
        if use_inactive:
            m = (self._h["ii_inac"] >= t0 - 3) & (self._h["jj_inac"] >= t0 - 3)
            if m.any():
                sel = torch.from_numpy(np.nonzero(m)[0]).to(self.device)
                ii = torch.cat([self.ii_inac[sel], ii])
                jj = torch.cat([self.jj_inac[sel], jj])
                target = torch.cat([self.target_inac[:, sel], target], dim=1)
                weight = torch.cat([self.weight_inac[:, sel], weight], dim=1)
        self._bundle_adjust(target, weight, ii, jj, t0, t1, iters, 1e-4, 0.1, motion_only, None, EPS)
        if self.upsample:
            self.video.upsample(uniq, upmask)
        self.age += 1

    @torch.no_grad()
    def update_fast(self, t0=None, t1=None, iters=2, use_inactive=False, EPS=1e-7, steps=8, max_t=None,
                    ba_type="loop", motion_only=False):
        """`steps` update + BA rounds on the volume implementation (src/factor_graph.py:323-366)"""
        t0, t1 = self._window(t0, t1)
        _, uniq = self._unique_sources()
        for _ in range(steps):
            coords1, motion = self._features(self.ii, self.jj, self.target)
            corr = self.corr(coords1)
            self._hint_sources(self._h["ii"])
            with torch.autocast("cuda", enabled=True):
                self.net, delta, weight, damping, upmask = self.update_op(self.net, self.inp, corr, motion, self.ii, self.jj)
            self.target = coords1 + delta.float()
            self.weight = weight.float()
            self.damping[uniq] = damping
            self._bundle_adjust(self.target, self.weight, self.ii, self.jj, t0, t1, iters, 1e-4, 1e-1, motion_only,
                                ba_type, EPS)
            if self.upsample:
                self.video.upsample(uniq, upmask)

    @torch.no_grad()
    def update_lowmem(self, t0=None, t1=None, iters=2, use_inactive=False, EPS=1e-7, steps=8, max_t=None,
                      ba_type="dense", motion_only=False):
        """global-BA form without correlation volumes: on-the-fly windowed correlation, the update operator run
        over chunks of 13 source frames (src/factor_graph.py:254-321)"""
        v = self.video
        cur_t = v.counter.value
        t = max_t if max_t is not None else cur_t
        fm = v.fmaps[:cur_t + 2]
        num, rig, ch, ht, wd = fm.shape
        corr_op = AltCorrBlock(fm.view(1, num * rig, ch, ht, wd))
        t0, t1 = self._window(t0, t1)
        ii_h, jj_h = self._h["ii"], self._h["jj"]
        chunks = []                                                     # (edge positions, source frames, unique sources)
        for i in range(int(ii_h.min()), int(ii_h.max()) + 1, 13):
            pos = np.nonzero((ii_h >= i) & (ii_h < i + 13))[0]
            if pos.size:
                same = (ii_h[pos] == jj_h[pos]).astype(np.int64)        # stereo pair: the right image's map
                chunks.append(dict(pos=torch.from_numpy(pos).to(self.device), pos_h=pos, contiguous=bool(pos[-1] - pos[0] + 1 == pos.size),
                                   lo=int(pos[0]), hi=int(pos[-1]) + 1,
                                   f1=torch.from_numpy(rig * ii_h[pos]).to(self.device),
                                   f2=torch.from_numpy(rig * jj_h[pos] + same).to(self.device),
                                   uniq=torch.from_numpy(np.unique(ii_h[pos])).to(self.device)))
        lm, ep = (1e-4, 1e-1) if ba_type == "loop" else (1e-5, 1e-2)
        for _ in range(steps):
            coords1, motion = self._features(self.ii, self.jj, self.target)
            for c in chunks:
                sl = slice(c["lo"], c["hi"]) if c["contiguous"] else c["pos"]
                iis, jjs = self.ii[sl], self.jj[sl]
                corr1 = corr_op(coords1[:, sl], c["f1"], c["f2"])
                self._hint_sources(ii_h[c["pos_h"]])
                with torch.autocast("cuda", enabled=True):
                    net, delta, weight, damping, upmask = self.update_op(self.net[:, sl], v.inps[None, iis], corr1,
                                                                         motion[:, sl], iis, jjs)
                    if self.upsample:
                        v.upsample(c["uniq"], upmask)
                self.net[:, sl] = net
                self.target[:, sl] = coords1[:, sl] + delta.float()
                self.weight[:, sl] = weight.float()
                self.damping[c["uniq"]] = damping
            self._bundle_adjust(self.target, self.weight, self.ii, self.jj, t0, t1, iters, lm, ep, motion_only, ba_type, EPS)
            v.dirty[:t] = True

    # ------------------------------------------------------------------------------------ edge proposals
    def add_neighborhood_factors(self, t0, t1, r=3):
        """edges between frames at most r apart (src/factor_graph.py:368-382)"""
        ii, jj = torch.meshgrid(torch.arange(t0, t1), torch.arange(t0, t1), indexing="ij")
        ii, jj = ii.reshape(-1), jj.reshape(-1)
        d = (ii - jj).abs()
        keep = (d > (1 if self.video.stereo else 0)) & (d <= r)
        self.add_factors(ii[keep].to(self.device), jj[keep].to(self.device))

    def add_proximity_factors(self, t0=0, t1=0, rad=2, nms=2, beta=0.25, thresh=16.0, remove=False, max_t=None):
        """edges by frame distance: local window + greedy non-maximum-suppressed candidates
        (src/factor_graph.py:384-450; the selection itself is goslam_proximity_edges)"""
        t = max_t if max_t is not None else self.video.counter.value
        ii, jj = torch.meshgrid(torch.arange(t0, t), torch.arange(t1, t), indexing="ij")
        d = self.video.distance(ii.reshape(-1), jj.reshape(-1), beta=beta)
        old_i = torch.cat([self.ii, self.ii_bad, self.ii_inac])
        old_j = torch.cat([self.jj, self.jj_bad, self.jj_inac])
        ei, ej = graph_ops.proximity_edges(d, t0, t1, t, rad, nms, thresh, self.max_factors, self.video.stereo,
                                           old_i, old_j)
        self.add_factors(ei, ej, remove)
