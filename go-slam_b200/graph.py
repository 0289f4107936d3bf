"""Factor-graph edge selection on the device (SURVEY §8f-2).

`proximity_edges` is the body of FactorGraph.add_proximity_factors (src/factor_graph.py:384-450) after
`d = self.video.distance(ii, jj, beta)`: one kernel launch instead of Python loops with a
device->host sync per candidate.  It returns the `(ii, jj)` the reference hands to `add_factors`.

    # src/factor_graph.py:397-449 become
    d = self.video.distance(ii, jj, beta=beta)
    ii1 = torch.cat([self.ii, self.ii_bad, self.ii_inac]); jj1 = torch.cat([self.jj, self.jj_bad, self.jj_inac])
    ii, jj = goslam_b200.graph.proximity_edges(d, t0, t1, t, rad, nms, thresh, self.max_factors,
                                               self.video.stereo, ii1, jj1)
    self.add_factors(ii, jj, remove)
"""
import math

import torch

from . import _lib


def local_edge_count(t0, t, rad, stereo, jfloor=0):
    return sum((1 if stereo else 0) + 2 * (i - min(i, max(i - rad, jfloor))) for i in range(t0, t))


def backend_edges(dist, t_start, t_end, radius, nms, thresh, max_factors, stereo, t_start_loop=None, loop=False):
    """Backend.ba's edge selection (src/backend.py:25-99; dense global BA, and loop-closure BA with
    loop=True): returns the (ii, jj) it hands to graph.add_factors — or None where the reference returns
    early (fewer than 3 edges, :96-97).  dist = video.distance over (t_start_loop..t_end) x (t_start..t_end)."""
    if t_start_loop is None or not loop:
        t_start_loop = t_start
    empty = torch.zeros(0, dtype=torch.long, device=dist.device)
    ii, jj = proximity_edges(dist, t_start_loop, t_start, t_end, radius, nms, thresh, max_factors,
                             stereo and not loop, empty, empty, dmax=thresh, jfloor=t_start_loop, loop=loop)
    return None if ii.numel() < 3 else (ii, jj)


def proximity_edges(dist, t0, t1, t, rad, nms, thresh, max_factors, stereo, ii_old, jj_old, dmax=100.0, jfloor=0,
                    loop=False):
    _lib.need_cuda("proximity_edges", dist)
    dev = dist.device
    d = dist.reshape(-1).float().contiguous()
    if d.numel() != (t - t0) * (t - t1):
        raise RuntimeError("proximity_edges: distance vector does not match the (t0..t) x (t1..t) grid")
    io = ii_old.to(dev).long().contiguous()
    jo = jj_old.to(dev).long().contiguous()
    mf = int(math.floor(float(max_factors)))
    cap = local_edge_count(t0, t, rad, stereo, jfloor) + max(0, mf + 2) + 10
    es_i = torch.empty(cap, dtype=torch.int64, device=dev)
    es_j = torch.empty(cap, dtype=torch.int64, device=dev)
    num = torch.zeros(1, dtype=torch.int32, device=dev)
    nbytes = _lib.load().goslam_proximity_workspace_bytes(int(t0), int(t1), int(t))
    if nbytes == 0:
        raise RuntimeError("proximity_edges: empty window (t0=%d t1=%d t=%d)" % (t0, t1, t))
    ws = _lib.workspace(nbytes, dev)
    _lib.call("proximity_edges", d, int(t0), int(t1), int(t), int(rad), int(nms), float(thresh), float(dmax), int(jfloor),
              int(bool(loop)), mf, int(bool(stereo)), io, jo, int(io.numel()), es_i, es_j, cap, num, ws, ws.numel())
    n = int(num.item())            # the one host sync (the reference builds its edge tensor on the host here)
    return es_i[:n], es_j[:n]


def filter_repeated_edges(ii, jj, ii_active, jj_active, ii_inactive, jj_inactive):
    """FactorGraph.__filter_repeated_edges (src/factor_graph.py:44-54): drop the candidate edges the
    graph already holds (active or inactive), keeping the order of the rest.  The reference builds a
    Python set with two .item() syncs per stored edge and tests every candidate against it; here it is
    a key comparison on the device (key = i * 2^32 + j), the only sync being the boolean compaction."""
    dev = ii.device
    key = (ii.long() << 32) | jj.long()
    old = torch.cat([(ii_active.to(dev).long() << 32) | jj_active.to(dev).long(),
                     (ii_inactive.to(dev).long() << 32) | jj_inactive.to(dev).long()])
    keep = ~torch.isin(key, old)
    return ii[keep], jj[keep]
