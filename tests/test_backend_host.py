"""The band rule of Backend.ba's distance grid (DESIGN.md §3.18), checked on the CPU restatement of its edge selection
(oracle/graph_oracle.backend_edges, pinned to the reference by tests/golden/backend_edges.npz).

Backend.ba only ever reads distance (i, j) with j - i <= k, k = -radius for dense BA and k = 2 - radius for loop
closure, so goslam_frame_distance_grid computes just that band and writes +inf elsewhere.  Here: for random grids
(dense and loop mode, stereo on and off, radius 1-3, nms 1-12, t_start > 0) the edges from the full grid equal the
edges from the same grid with everything outside the band set to +inf, although many discarded entries lie below the
threshold.  The loop band is also tight: one diagonal fewer changes some selections (the dense band is not: its
local-window edges and their suppression boxes overwrite the diagonals next to it, but they are cheap to compute)."""
import numpy as np
import pytest

from oracle import graph_oracle


def band_k(radius, loop):
    return 2 - radius if loop else -radius


def banded(dist, r0, r1, c0, c1, k):
    d = dist.reshape(r1 - r0, c1 - c0).copy()
    i = np.arange(r0, r1)[:, None]
    j = np.arange(c0, c1)[None, :]
    d[(j - i) > k] = np.inf
    return d.reshape(-1)


def make_case(seed, loop):
    rng = np.random.default_rng(seed)
    t_start = int(rng.integers(0, 6))
    t_end = t_start + int(rng.integers(8, 40))
    radius = int(rng.integers(1, 4))
    nms = int(rng.integers(1, 13))
    stereo = bool(rng.integers(0, 2))
    thresh = float(rng.uniform(12.0, 26.0))
    tsl = None
    if loop:
        tsl = int(rng.integers(t_start, t_end - 2))
    r0 = tsl if loop else t_start
    ilen, jlen = t_end - r0, t_end - t_start
    dist = rng.random(ilen * jlen) * 40
    if loop:                            # smooth field: 3x3 neighbourhoods agree often enough to pass the vote
        ph = rng.uniform(0, 3, size=2)
        dist = (dist.reshape(ilen, jlen) * 0.25 + 30.0 * np.abs(np.sin(np.arange(ilen)[:, None] * 0.4 + ph[0]
                                                                        + np.arange(jlen)[None] * 0.3 + ph[1]))).reshape(-1)
    maxf = int(rng.integers(10, 8 * jlen + 20))
    return dict(dist=dist.astype(np.float32), t_start=t_start, t_end=t_end, radius=radius, nms=nms, stereo=stereo,
                thresh=np.float32(thresh), maxf=maxf, tsl=tsl, r0=r0)


def select(c, dist):
    return graph_oracle.backend_edges(dist, c["t_start"], c["t_end"], c["radius"], c["nms"], c["thresh"], c["maxf"],
                                      c["stereo"], t_start_loop=c["tsl"], loop=c["tsl"] is not None)


def same(a, b):
    return (a is None and b is None) or (a is not None and b is not None and np.array_equal(a, b))


@pytest.mark.parametrize("loop", [False, True], ids=["dense", "loop"])
def test_band_keeps_every_selection(loop):
    hidden_below = 0
    for seed in range(300):
        c = make_case(1000 * int(loop) + seed, loop)
        k = band_k(c["radius"], loop)
        full = select(c, c["dist"])
        cut = banded(c["dist"], c["r0"], c["t_end"], c["t_start"], c["t_end"], k)
        hidden_below += int(np.sum((cut == np.inf) & (c["dist"] <= c["thresh"])))
        got = select(c, cut)
        assert same(full, got), (seed, c["t_start"], c["t_end"], c["radius"], c["nms"], c["stereo"], c["tsl"])
    assert hidden_below > 1000          # the band hides many entries the selection would have taken as candidates


def test_loop_vote_is_exercised_and_band_is_tight():
    """the loop cases accept 3x3 votes, and dropping the diagonal j - i = 2 - radius changes some of them"""
    voted, tighter_differs = 0, 0
    for seed in range(300):
        c = make_case(1000 + seed, True)
        full = select(c, c["dist"])
        if full is None:
            continue
        n_local = sum(2 * (i - max(i - c["radius"], c["tsl"])) for i in range(c["tsl"], c["t_end"]))
        voted += int(len(full) > n_local)
        tight = banded(c["dist"], c["r0"], c["t_end"], c["t_start"], c["t_end"], band_k(c["radius"], True) - 1)
        tighter_differs += int(not same(full, select(c, tight)))
    assert voted > 100
    assert tighter_differs > 0

