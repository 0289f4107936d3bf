"""`Frontend` — the tracking process's keyframe update with the reference's constructor, attributes and call schedule
(src/frontend.py:9-150), on goslam_b200.FactorGraph (correlation volumes in the slot pool) and goslam_b200.Backend for
loop closure.

Per new keyframe: drop edges older than `max_age` into the inactive set, add proximity edges, four update + BA
rounds, then the keyframe test on the distance between the two previous keyframes.  A redundant keyframe is removed;
otherwise either loop-closure BA runs over the last `loop_window` keyframes (with the local graph's edges copied in,
FactorGraph.adopt_edges) or two more update rounds do.  The keyframe test's distance is the one decision sync per
frame; the start of the dirty range comes from the graph's host edge mirror instead of a device reduction.
"""
from time import gmtime, strftime

import torch

from .backend import Backend
from .factor_graph import FactorGraph


class Frontend:
    def __init__(self, net, video, args, cfg):
        self.video = video
        self.update_op = net.update
        tr = cfg["tracking"]
        fe = tr["frontend"]
        self.warmup = tr["warmup"]
        self.upsample = tr["upsample"]
        self.beta = tr["beta"]
        self.verbose = cfg["verbose"]
        self.frontend_max_factors = fe["max_factors"]
        self.frontend_nms = fe["nms"]
        self.keyframe_thresh = fe["keyframe_thresh"]
        self.frontend_window = fe["window"]
        self.frontend_thresh = fe["thresh"]
        self.frontend_radius = fe["radius"]
        self.enable_loop = fe["enable_loop"]
        self.loop_closing = Backend(net, video, args, cfg)
        self.last_loop_t = -1
        self.graph = FactorGraph(video, net.update, device=args.device, corr_impl="volume",
                                 max_factors=self.frontend_max_factors, upsample=self.upsample)
        self.t0 = 0                    # local optimisation window
        self.t1 = 0
        self.is_initialized = False
        self.count = 0
        self.max_age = 25
        self.iters1 = 4
        self.iters2 = 2

    def _update(self):
        """edges for the newest keyframe, update rounds, keyframe test, loop closure"""
        g, v = self.graph, self.video
        self.count += 1
        self.t1 += 1
        if g.corr is not None:
            g.rm_factors(g.age > self.max_age, store=True)
        # candidate edges from [t1 - 5, counter) to [t1 - window, counter)
        g.add_proximity_factors(self.t1 - 5, max(self.t1 - self.frontend_window, 0), rad=self.frontend_radius,
                                nms=self.frontend_nms, thresh=self.frontend_thresh, beta=self.beta, remove=True)
        k = self.t1 - 1
        v.disps[k] = torch.where(v.disps_sens[k] > 0, v.disps_sens[k], v.disps[k])
        for _ in range(self.iters1):
            g.update(t0=None, t1=None, use_inactive=True)

        d = v.distance([self.t1 - 3], [self.t1 - 2], beta=self.beta, bidirectional=True)
        if d.item() < self.keyframe_thresh:
            g.rm_keyframe(self.t1 - 2)
            with v.get_lock():
                v.counter.value -= 1
                self.t1 -= 1
        else:
            cur_t = v.counter.value
            if self.enable_loop and cur_t > self.frontend_window:
                n_kf, _ = self.loop_closing.loop_ba(t_start=0, t_end=cur_t, steps=self.iters2, motion_only=False,
                                                    local_graph=g)
                if self.verbose:
                    print("%s - Loop BA: [0, %d]; %d KFs, last loop at %d" % (
                        strftime("%Y-%m-%d %H:%M:%S", gmtime()), cur_t, n_kf, self.last_loop_t))
                self.last_loop_t = cur_t
            else:
                for _ in range(self.iters2):
                    g.update(t0=None, t1=None, use_inactive=True)

        # initial pose and depth of the next keyframe
        v.poses[self.t1] = v.poses[self.t1 - 1]
        v.disps[self.t1] = v.disps[self.t1 - 1].mean()
        v.dirty[int(g._h["ii"].min()):self.t1] = True

    def _initialize(self):
        """bootstrap on the first `warmup` keyframes"""
        g, v = self.graph, self.video
        self.t0 = 0
        self.t1 = v.counter.value
        g.add_neighborhood_factors(self.t0, self.t1, r=3)
        for _ in range(8):
            g.update(t0=1, t1=None, use_inactive=True)
        # the reference passes no beta here, so the graph's default applies
        g.add_proximity_factors(t0=0, t1=0, rad=2, nms=2, thresh=self.frontend_thresh, remove=False)
        for _ in range(8):
            g.update(t0=1, t1=None, use_inactive=True)
        v.poses[self.t1] = v.poses[self.t1 - 1].clone()
        v.disps[self.t1] = v.disps[self.t1 - 4:self.t1].mean()
        self.is_initialized = True
        self.last_pose = v.poses[self.t1 - 1].clone()
        self.last_disp = v.disps[self.t1 - 1].clone()
        self.last_time = v.timestamp[self.t1 - 1].clone()
        with v.get_lock():
            v.ready.value = 1
            v.dirty[:self.t1] = True
        g.rm_factors(g.ii < self.warmup - 4, store=True)

    def __call__(self):
        if not self.is_initialized and self.video.counter.value == self.warmup:
            self._initialize()
        elif self.is_initialized and self.t1 < self.video.counter.value:
            self._update()
