"""Reverse-edge pairing of the correlation build: when one build call holds both (i, j) and (j, i) once each, the
later edge (the reader) stores levels 1-3 only and the lookup reads its level 0 as the transpose of its partner's
(CorrPool.alias).  Every result must equal the same edges built unpaired, one build call per edge, bit for bit:
all four levels of gather_pyramid() and the lookup, also for out-of-image and non-finite coordinates, and through
every pool operation (masking one side of a pair off and reusing its slot, cat within and across pools, grow)."""
import pytest
import torch

import corr_envelope

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def window_edges(nkf=8, radius=3):
    """the |i - j| <= radius window as FactorGraph.add_factors gets it: every forward edge, then every reverse"""
    fwd = [(i, j) for i in range(nkf) for j in range(nkf) if 0 < j - i <= radius]
    ii = torch.tensor([i for i, _ in fwd] + [j for _, j in fwd])
    jj = torch.tensor([j for _, j in fwd] + [i for i, _ in fwd])
    return ii, jj


def km_of(F, h, w, g, rig=1, scale=1.0):
    from goslam_b200.modules.corr import fmaps_to_kmajor
    return fmaps_to_kmajor((torch.randn(F, rig, 128, h, w, generator=g) * scale).half().to(dev()))


def build(km, ii, jj, h, w, pool=None, rig=1):
    from goslam_b200.modules import CorrBlock
    return CorrBlock.from_video(km, ii.to(dev()), jj.to(dev()), h, w, rig=rig, pool=pool)


def unpaired(km, ii, jj, h, w, rig=1):
    """the same edges, one build call per edge (a call of one edge is never paired)"""
    return [build(km, ii[e:e + 1], jj[e:e + 1], h, w, rig=rig) for e in range(len(ii))]


def coords_for(N, h, w, g):
    """[1, N, h, w, 2]: random windows around and past the image, non-finite and huge values on the first pixels"""
    c = corr_envelope.nonfinite_coords(N, h, w, h, w, g)
    return c.permute(0, 2, 3, 1)[None].contiguous().to(dev())


def n_readers(blk):
    return int((blk.pool.alias[blk.slots.long(), 0] & 1).sum())


def assert_same(blk, singles, coords, edges=None):
    edges = range(len(singles)) if edges is None else edges
    pyr = blk.gather_pyramid()
    out = blk(coords)
    for k, e in enumerate(edges):
        ref = singles[e]
        for lvl, (a, b) in enumerate(zip(pyr, ref.gather_pyramid())):
            assert torch.equal(a[k:k + 1].view(torch.int16), b.view(torch.int16)), "edge %d level %d" % (e, lvl)
        want = ref(coords[:, k:k + 1].contiguous())
        assert torch.equal(out[:, k:k + 1].view(torch.int16), want.view(torch.int16)), "lookup, edge %d" % e


@pytest.mark.parametrize("hw", [(40, 80), (60, 80)])
def test_window_pairs_match_unpaired_builds(hw):
    h, w = hw
    g = torch.Generator().manual_seed(500 + h)
    km = km_of(8, h, w, g)
    ii, jj = window_edges()
    blk = build(km, ii, jj, h, w)
    assert n_readers(blk) == len(ii) // 2
    singles = unpaired(km, ii, jj, h, w)
    assert_same(blk, singles, coords_for(len(ii), h, w, g))


def test_duplicates_and_self_edges_are_never_aliased():
    h, w = 24, 40
    g = torch.Generator().manual_seed(7)
    km = km_of(4, h, w, g)
    # (0,1) twice with (1,0) once, a self-edge (2,2), and one clean pair (2,3)/(3,2)
    ii, jj = torch.tensor([0, 1, 0, 2, 2, 3]), torch.tensor([1, 0, 1, 2, 3, 2])
    blk = build(km, ii, jj, h, w)
    al = blk.pool.alias[blk.slots.long(), 0].cpu()
    assert (al & 1).tolist() == [0, 0, 0, 0, 0, 1]
    assert int(al[5]) >> 1 == blk._slots_host[4]
    assert_same(blk, unpaired(km, ii, jj, h, w), coords_for(len(ii), h, w, g))


def test_stereo_rig_pairs_and_left_right_edges():
    """rig 2: the left-right self-edges read the second camera and stay unpaired; left-left reverse edges pair"""
    h, w = 40, 60
    g = torch.Generator().manual_seed(8)
    km = km_of(4, h, w, g, rig=2)
    ii = torch.tensor([0, 1, 2, 3, 0, 1, 2, 1, 2, 3])
    jj = torch.tensor([0, 1, 2, 3, 1, 2, 3, 0, 1, 2])
    blk = build(km, ii, jj, h, w, rig=2)
    assert (blk.pool.alias[blk.slots.long(), 0] & 1).tolist() == [0] * 7 + [1] * 3
    assert_same(blk, unpaired(km, ii, jj, h, w, rig=2), coords_for(len(ii), h, w, g))


def test_masking_one_side_then_reusing_the_slots():
    """keep one side of each pair (the reader for some pairs, the partner for others), then build new edges into the
    released slots: the survivors' pyramids and lookups are unchanged"""
    from goslam_b200.modules.corr import CorrPool
    h, w = 40, 80
    g = torch.Generator().manual_seed(9)
    km = km_of(8, h, w, g)
    ii, jj = window_edges()
    N = len(ii)
    pool = CorrPool(N, h, w, device=dev())
    blk = build(km, ii, jj, h, w, pool=pool)
    singles = unpaired(km, ii, jj, h, w)
    half = N // 2
    keep = torch.zeros(N, dtype=torch.bool)
    keep[torch.arange(0, half, 2)] = True                 # partners of pairs 0, 2, 4, ...
    keep[half + torch.arange(1, half, 2)] = True          # readers of pairs 1, 3, 5, ...
    blk = blk[keep]
    edges = keep.nonzero().reshape(-1).tolist()
    assert n_readers(blk) == 0 and pool.free_slots == N - len(edges)
    new = build(km, jj[:pool.free_slots], ii[:pool.free_slots], h, w, pool=pool)   # overwrites every freed slot
    assert pool.free_slots == 0
    assert_same(blk, singles, coords_for(len(edges), h, w, g), edges)
    new_ref = unpaired(km, jj[:len(new._slots_host)], ii[:len(new._slots_host)], h, w)
    assert_same(new, new_ref, coords_for(len(new_ref), h, w, g))


def test_cat_within_and_across_pools_and_grow():
    from goslam_b200.modules.corr import CorrPool
    h, w = 24, 40
    g = torch.Generator().manual_seed(10)
    km = km_of(5, h, w, g)
    ii, jj = window_edges(5, 2)
    ii2, jj2 = torch.tensor([4, 0, 4]), torch.tensor([0, 4, 3])
    singles = unpaired(km, torch.cat([ii, ii2]), torch.cat([jj, jj2]), h, w)
    coords = coords_for(len(ii) + len(ii2), h, w, g)
    # within a pool: the slot tables join, the aliases stay live
    pool = CorrPool(len(ii) + len(ii2), h, w, device=dev())
    a = build(km, ii, jj, h, w, pool=pool)
    b = build(km, ii2, jj2, h, w, pool=pool)
    a.cat(b)
    assert n_readers(a) == len(ii) // 2 + 1
    assert_same(a, singles, coords)
    # grow with live aliases
    pool.grow(pool.capacity + 5)
    assert n_readers(a) == len(ii) // 2 + 1
    assert_same(a, singles, coords)
    # across pools: the raw slot copy gets every level 0 materialized
    c = build(km, ii, jj, h, w)
    d = build(km, ii2, jj2, h, w)
    c.cat(d)
    assert c.pool is not d.pool and n_readers(c) == 0
    assert_same(c, singles, coords)
    assert_same(d, singles[len(ii):], coords[:, len(ii):].contiguous())
