"""`Backend` — global and loop-closure bundle adjustment with the reference's constructor, config keys, attributes and
methods (src/backend.py:7-163): `dense_ba` (the optimizing process's full BA) and `loop_ba` (run by the frontend on
every new keyframe once enough exist).

Edge selection is two launches and one host sync instead of a host-side index grid, two distance launches and a
Python loop with a device sync per candidate:
  * `droid_backends.frame_distance_grid` computes the distances straight from the frame ranges, only inside the band
    the selection can read (j - i <= -radius dense, <= 2 - radius in loop mode; DESIGN.md §3.18), from a snapshot of
    the poses taken on the stream;
  * `graph.backend_edges` runs the masking, local window, sort and greedy suppression in one kernel; reading its edge
    count is the one sync.
The optimisation itself is goslam_b200.FactorGraph.update_lowmem, as in the reference.
"""
import torch

from . import droid_backends
from . import graph as graph_ops
from .factor_graph import FactorGraph


class Backend:
    def __init__(self, net, video, args, cfg):
        self.video = video
        self.device = args.device
        self.update_op = net.update
        tr = cfg["tracking"]
        be = tr["backend"]
        self.upsample = tr["upsample"]
        self.beta = tr["beta"]
        self.backend_thresh = be["thresh"]
        self.backend_radius = be["radius"]
        self.backend_nms = be["nms"]
        self.backend_loop_window = be["loop_window"]
        self.backend_loop_thresh = be["loop_thresh"]
        self.backend_loop_radius = be["loop_radius"]
        self.backend_loop_nms = be["loop_nms"]

    def select_edges(self, t_start, t_end, nms, radius, thresh, max_factors, t_start_loop=None, loop=False):
        """the (ii, jj) Backend.ba hands to add_factors (src/backend.py:27-99), or None where it returns 0"""
        if t_start_loop is None or not loop:
            t_start_loop = t_start
        assert t_start_loop >= t_start, f"short: {t_start_loop}, long: {t_start}."
        v = self.video
        band = 2 - radius if loop else -radius
        d = droid_backends.frame_distance_grid(v.poses, v.disps, v.intrinsics[0], t_start_loop, t_end, t_start, t_end,
                                               band, self.beta)
        return graph_ops.backend_edges(d, t_start, t_end, radius, nms, thresh, max_factors, v.stereo,
                                       t_start_loop=t_start_loop, loop=loop)

    @torch.no_grad()
    def ba(self, t_start, t_end, steps, graph, nms, radius, thresh, max_factors, t_start_loop=None, loop=False,
           motion_only=False):
        """select edges, add them to `graph`, run `steps` low-memory update + BA rounds, clear the graph"""
        if t_start_loop is None or not loop:
            t_start_loop = t_start
        edges = self.select_edges(t_start, t_end, nms, radius, thresh, max_factors, t_start_loop, loop)
        if edges is None:
            return 0
        graph.add_factors(*edges, remove=True)
        edge_num = len(graph.ii)
        # t0 = t_start_loop + 1: the first frame of the window stays fixed
        graph.update_lowmem(t0=t_start_loop + 1, t1=t_end, iters=2, use_inactive=False, steps=steps, max_t=t_end,
                            ba_type="dense", motion_only=motion_only)
        graph.clear_edges()
        self.video.dirty[t_start:t_end] = True
        return edge_num

    @torch.no_grad()
    def dense_ba(self, t_start, t_end, steps=6, motion_only=False):
        radius = self.backend_radius
        n = t_end - t_start
        max_factors = (int(self.video.stereo) + (radius + 2) * 2) * n
        graph = FactorGraph(self.video, self.update_op, device=self.device, corr_impl="alt", max_factors=max_factors,
                            upsample=self.upsample)
        n_edges = self.ba(t_start, t_end, steps, graph, self.backend_nms, radius, self.backend_thresh, max_factors,
                          motion_only=motion_only)
        return n, n_edges

    @torch.no_grad()
    def loop_ba(self, t_start, t_end, steps=6, motion_only=False, local_graph=None):
        window = self.backend_loop_window
        max_factors = 8 * window
        t_start_loop = max(0, t_end - window)
        graph = FactorGraph(self.video, self.update_op, device=self.device, corr_impl="alt", max_factors=max_factors,
                            upsample=self.upsample)
        if local_graph is not None:
            graph.adopt_edges(local_graph)
        left_factors = max_factors - len(graph.ii)
        n_edges = self.ba(t_start, t_end, steps, graph, self.backend_loop_nms, self.backend_loop_radius,
                          self.backend_loop_thresh, left_factors, t_start_loop=t_start_loop, loop=True,
                          motion_only=motion_only)
        return t_end - t_start_loop, n_edges
