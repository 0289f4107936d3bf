"""The half-precision correlation build (corr_build_tc.cu, tiled layout) and the pooled lookup (corr_lookup.cu)
across their whole envelope, against float64 and the oracle, plus the CUDA-core fallback just outside it.

Numerics contract of the build (corr_build_tc.cu): level 0 is one rounding of an fp32 sum of the products of the
half-scaled maps; each coarser level is half((((a + b) + c) + d) * 0.25) of the rounded finer level, a..d in
row-major window order (avg_pool2d).  So level 0 is checked against the exact float64 product within one rounding
plus the fp32 accumulation bound, and levels 1-3 bit for bit against that pooling of the device's own finer level.
The lookup is a fixed sequence of correctly rounded half operations: bit for bit against the oracle."""
import math

import numpy as np
import pytest
import torch

import corr_envelope
import ref_golden
from corr_envelope import nonfinite_coords
from oracle import corr_oracle

pytestmark = pytest.mark.gpu

SHAPES = corr_envelope.SHAPES
NAN = float("nan")


def dev():
    return torch.device("cuda:0")


def _pooled_block(fmaps, ii, jj, h, w, num_levels=4, noncontig=False):
    """CorrBlock.from_video into a fresh pool whose levels hold NaN first; the block does not start at slot 0,
    and with `noncontig` its slot table has a hole"""
    from goslam_b200.modules import CorrBlock
    from goslam_b200.modules.corr import CorrPool, fmaps_to_kmajor
    N = len(ii)
    pool = CorrPool(N + 4, h, w, num_levels, device=dev())
    for lvl in pool.levels:
        lvl.fill_(NAN)
    if noncontig:
        held = pool.alloc(3)
        pool.release([held[1]])
    else:
        pool.alloc(1)
    blk = CorrBlock.from_video(fmaps_to_kmajor(fmaps.to(dev())), ii.to(dev()), jj.to(dev()), h, w,
                               num_levels=num_levels, pool=pool)
    assert blk.pool is pool and min(blk._slots_host) > 0
    s = blk._slots_host
    assert noncontig == (s != list(range(s[0], s[0] + N)))
    return blk


def _check_level0(got, fa, fb, tag):
    """got [N, h, w, h, w] (device, f16 or f32); fa, fb [N, 128, h, w] the edges' feature maps (device, same dtype).
    Per element |got - exact| <= 1/2 ulp(exact) + 128 * 2^-24 * sum |a b|, exact = the float64 product of the maps
    scaled by 1/4 in their own precision.  Half: inf where exact lies clearly past the half range, finite where it
    lies clearly inside.  Returns the worst error as a fraction of its bound."""
    N, D, h, w = fa.shape
    half = got.dtype == torch.float16
    e_min, mant = (-14, 10) if half else (-126, 23)
    worst = 0.0
    for n in range(N):
        a = (fa[n] / 4).double().reshape(D, h * w)
        b = (fb[n] / 4).double().reshape(D, h * w)
        exact = a.t() @ b
        acc = 128 * 2.0 ** -24 * (a.abs().t() @ b.abs())
        g = got[n].reshape(h * w, h * w).double()
        assert not torch.isnan(g).any(), tag                           # every entry written
        ax = exact.abs()
        ulp = torch.exp2(torch.floor(torch.log2(ax.clamp_min(2.0 ** e_min))) - mant)
        bound = 0.5 * ulp + acc
        inside = torch.ones_like(ax, dtype=torch.bool)
        if half:
            inside = ax + acc < 65520.0
            over = ax - acc > 65520.0
            assert torch.equal(g[over], torch.copysign(torch.full_like(g[over], math.inf), exact[over])), tag
            assert torch.isfinite(g[inside]).all(), tag
        err = (g - exact).abs()[inside] / bound[inside]
        if err.numel():
            worst = max(worst, err.max().item())
    assert worst <= 1.0, (tag, worst)
    return worst


def _pool_f32(x):
    """avg_pool2d(2, 2) of numpy [..., H, W] as the build does it: fp32 sum in row-major window order, x 0.25, one
    rounding to x's dtype"""
    H, W = x.shape[-2] // 2 * 2, x.shape[-1] // 2 * 2
    f = x[..., :H, :W].astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        s = ((f[..., 0::2, 0::2] + f[..., 0::2, 1::2]) + f[..., 1::2, 0::2]) + f[..., 1::2, 1::2]
        return (s * np.float32(0.25)).astype(x.dtype)


def _same_bits(got, want, tag):
    """bit for bit, any NaN equal to any NaN"""
    assert got.dtype == want.dtype and got.shape == want.shape, tag
    ng, nw = np.isnan(got), np.isnan(want)
    assert np.array_equal(ng, nw), (tag, int((ng != nw).sum()))
    u = np.uint16 if got.dtype == np.float16 else np.uint32
    bad = got.view(u)[~ng] != want.view(u)[~nw]
    assert not bad.any(), (tag, int(bad.sum()))


def _check_pooling(levels, tag):
    finer = levels[0].cpu().numpy()
    for i in range(1, len(levels)):
        got = levels[i].cpu().numpy()
        _same_bits(got, _pool_f32(finer), "%s level %d" % (tag, i))
        finer = got


def _random_fmaps(F, h, w, scale, g, dtype=torch.float16):
    return (torch.randn(F, 1, 128, h, w, generator=g) * scale).to(dtype)


# --------------------------------------------------------------------------------------------- build
@pytest.mark.parametrize("hw", SHAPES)
def test_build_exact_inputs_bit_for_bit(hw):
    """integer features (multiples of 4, so fmap / 4 is exact) on 7 channels with |values| <= 2: |level 0| <= 28, and
    every entry of every level is exactly representable in half.  All four levels equal the oracle bit for bit,
    so a misplaced or wrongly pooled element fails exactly."""
    h, w = hw
    g = torch.Generator().manual_seed(h * 1000 + w)
    fmaps = torch.zeros(3, 1, 128, h, w)
    ch = [3, 29, 64, 77, 100, 115, 127]                   # both 64-channel boxes of the K loop
    fmaps[:, :, ch] = 4.0 * torch.randint(-2, 3, (3, 1, len(ch), h, w), generator=g).float()
    fmaps = fmaps.half()
    ii, jj = torch.tensor([0, 2]), torch.tensor([1, 0])
    blk = _pooled_block(fmaps, ii, jj, h, w, noncontig=(h % 2 == 1))
    want = corr_oracle.corr_build(fmaps[ii, 0], fmaps[jj, 0], 4)
    for i, (x, y) in enumerate(zip(blk.gather_pyramid(), want)):
        x = x.cpu()
        assert x.shape == y.shape and not torch.isnan(x).any(), (hw, i)
        assert torch.equal(x, y), (hw, i, int((x != y).sum()))
    assert want[0].abs().max() <= 31


SCALES = {"unit": 1.0, "past2048": 32.0, "overflow": 256.0}


def _cancel_fmaps(h, w, g):
    """frames 0, 2: sources, (+-1, 1) on channels 0, 1; frames 1, 3: targets, +-8192 (+-2048 after / 4) on channel 0
    in even rows with the sign alternating along x, 2^-12 k (2^-14 k, k in {1, 3}) on channel 1 in odd rows.
    Every 2x2 window of level 0 then holds +-2048, -+2048 on top and two tiny values below: fp32 loses the tiny
    values unless the two big ones cancel first, as they do in row-major window order."""
    f = torch.zeros(4, 1, 128, h, w)
    sign = torch.where(torch.rand(2, h, w, generator=g) < 0.5, -1.0, 1.0)
    f[0::2, 0, 0], f[0::2, 0, 1] = 4.0 * sign, 4.0
    y, x = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    even = (y % 2 == 0).float()
    f[1::2, 0, 0] = 8192.0 * even * (1 - 2 * (x % 2)).float()
    f[1::2, 0, 1] = 2.0 ** -12 * (1 - even) * (1 + 2 * ((x + y // 2) % 2)).float()
    return f.half()


@pytest.mark.parametrize("kind", list(SCALES) + ["cancel"])
@pytest.mark.parametrize("hw", SHAPES)
def test_build_random_inputs_vs_float64(hw, kind):
    """random features at unit scale, at a scale where level 0 passes 2048 and at one where some of it overflows
    half, and a pattern whose pooling depends on the summation order; level 0 against float64, levels 1-3 bit for
    bit against the pooling of the device's own finer level"""
    h, w = hw
    g = torch.Generator().manual_seed(7 * h + w + len(kind))
    if kind == "cancel":
        fmaps, ii, jj = _cancel_fmaps(h, w, g), torch.tensor([0, 2]), torch.tensor([1, 3])
    else:
        fmaps, ii, jj = _random_fmaps(3, h, w, SCALES[kind], g), torch.tensor([0, 2]), torch.tensor([1, 0])
    blk = _pooled_block(fmaps, ii, jj, h, w, noncontig=(kind == "unit"))
    pyr = blk.gather_pyramid()
    fd = fmaps.to(dev())
    worst = _check_level0(pyr[0], fd[ii.to(dev()), 0], fd[jj.to(dev()), 0], (hw, kind))
    print("level0 %-8s %-10s worst |err| / bound = %.3f" % (kind, hw, worst))
    if kind == "past2048":
        assert pyr[0].abs().max().item() > 2048
    if kind == "overflow":
        assert torch.isinf(pyr[0]).any() and torch.isfinite(pyr[0]).any()
    _check_pooling(pyr, (hw, kind))


# --------------------------------------------------------------------------------------------- lookup
FRACS = (0.0, 0.25, 0.5, None)


def _sweep_coords(h, w, num_levels, g):
    """[M, 2] level-0 coordinates: for each level l, window origins floor(c / 2^l) - 3 over [-8, w_l + 1] x
    [-8, h_l + 1] with fractions 0, 1/4, 1/2 and a random one, i.e. every tile column, ragged tile, band boundary
    and level-2 row parity, with windows hanging over every border"""
    out = []
    for l in range(num_levels):
        x1, y1 = torch.meshgrid(torch.arange(-8, (w >> l) + 2).float(), torch.arange(-8, (h >> l) + 2).float(),
                                indexing="xy")
        x1, y1 = x1.reshape(-1), y1.reshape(-1)
        for f in FRACS:
            fx = torch.rand(x1.shape, generator=g) if f is None else torch.full_like(x1, f)
            fy = torch.rand(x1.shape, generator=g) if f is None else torch.full_like(x1, f)
            out.append(torch.stack([(x1 + 3 + fx) * 2 ** l, (y1 + 3 + fy) * 2 ** l], -1))
    return torch.cat(out)


def _sweep_calls(coords, N, h, w):
    """the sweep as coordinate fields [1, N, h, w, 2], one per lookup call (the last padded by repetition)"""
    per = N * h * w
    calls = []
    for k in range(0, coords.shape[0], per):
        c = coords[k:k + per]
        if c.shape[0] < per:
            c = torch.cat([c, c[:1].expand(per - c.shape[0], 2)])
        calls.append(c.reshape(1, N, h, w, 2).contiguous())
    return calls


def _edges_for(M, h, w):
    return max(2, min(-(-M // (h * w)), 8192 // (h * w)))


def _lookup_vs_oracle(blk, calls, tag, exact=True):
    pyr = [p.cpu().numpy() for p in blk.gather_pyramid()]
    for k, c in enumerate(calls):
        got = blk(c.to(dev()))[0].cpu().numpy()
        want = corr_oracle.corr_pyramid_lookup(pyr, c[0].numpy(), 3)
        if exact:
            np.testing.assert_array_equal(got.astype(np.float32), want.astype(np.float32), err_msg="%s call %d" % (tag, k))
        else:
            # chained FMAs in the reference's order; the oracle emulates FMA in float64: <= 1 ulp
            np.testing.assert_allclose(got, want, rtol=2e-7, atol=1e-7, err_msg="%s call %d" % (tag, k))


@pytest.mark.parametrize("hw,num_levels", [(s, 4) for s in SHAPES] + [((9, 13), 2), ((9, 13), 3), ((37, 127), 2),
                                                                      ((37, 127), 3)])
def test_lookup_sweep_vs_oracle(hw, num_levels):
    """CorrBlock(fmap1, fmap2) takes the tensor-core build and the tiled lookup for every envelope shape; the lookup
    equals the oracle on the de-tiled pyramid bit for bit, for window origins across every level"""
    from goslam_b200.modules import CorrBlock
    h, w = hw
    g = torch.Generator().manual_seed(31 * h + w + num_levels)
    coords = _sweep_coords(h, w, num_levels, g)
    N = _edges_for(coords.shape[0], h, w)
    f1 = torch.randn(1, N, 128, h, w, generator=g).half()
    f2 = torch.randn(1, N, 128, h, w, generator=g).half()
    blk = CorrBlock(f1.to(dev()), f2.to(dev()), num_levels=num_levels)
    assert blk.pool is not None
    _lookup_vs_oracle(blk, _sweep_calls(coords, N, h, w), (hw, num_levels))


@pytest.mark.parametrize("hw", SHAPES)
def test_lookup_never_reads_padding(hw):
    """overwriting every padding element of every level (the complement of CorrPool.level_rowmajor's positions)
    with NaN, 65504 or inf leaves the lookup bit-identical.  What the build leaves there: level 0's padding is 0
    (products with the zero-filled target rows and columns), the coarser levels' padding is pooled from it and
    from the last row or column of the finer level, so it is not zero where that row or column is odd."""
    h, w = hw
    g = torch.Generator().manual_seed(11 * h + w)
    fmaps = _random_fmaps(3, h, w, 1.0, g)
    blk = _pooled_block(fmaps, torch.tensor([0, 2]), torch.tensor([1, 0]), h, w)
    pool, slots = blk.pool, blk.slots.long()
    pads = [corr_envelope.padding_mask(h, w, i, device=dev()) for i in range(4)]
    held = [pool.levels[i][slots][:, :, pads[i]].float() for i in range(4)]
    assert (held[0] == 0).all()
    # the level-1 column (w >> 1), pooled from level-0 column w - 1, exists when w is odd and (w >> 1) is not a
    # multiple of 4 (the tile width); likewise for rows
    if (w % 2 and (w >> 1) % 4) or (h % 2 and (h >> 1) % 4):
        assert ((held[1] != 0) & ~torch.isnan(held[1])).any()
    calls = _sweep_calls(_sweep_coords(h, w, 4, g), 2, h, w)
    base = [blk(c.to(dev())) for c in calls]
    for poison in (NAN, 65504.0, math.inf):
        for i in range(4):
            lvl = pool.levels[i]
            lvl[:, :, pads[i]] = poison
        for c, b in zip(calls, base):
            assert torch.equal(blk(c.to(dev())).view(torch.int16), b.view(torch.int16)), (hw, poison)


def test_far_slots_past_4_gib():
    """a 96-slot 60x80 pool (~6.1 GB): edges in slots 93-95, whose level-0 planes cross and start past 2^32 bytes,
    build and look up exactly as in a 3-slot pool"""
    from goslam_b200.modules import CorrBlock
    from goslam_b200.modules.corr import CorrPool, fmaps_to_kmajor
    h, w = 60, 80
    g = torch.Generator().manual_seed(96)
    km = fmaps_to_kmajor(_random_fmaps(4, h, w, 1.0, g).to(dev()))
    ii, jj = torch.tensor([0, 1, 3], device=dev()), torch.tensor([1, 2, 0], device=dev())
    big = CorrPool(96, h, w, device=dev())
    big.alloc(93)
    far = CorrBlock.from_video(km, ii, jj, h, w, pool=big)
    assert far._slots_host == [93, 94, 95]
    assert 93 * h * w * big.plane_elems[0] * 2 < 2 ** 32 < 94 * h * w * big.plane_elems[0] * 2
    near = CorrBlock.from_video(km, ii, jj, h, w, pool=CorrPool(3, h, w, device=dev()))
    for x, y in zip(far.gather_pyramid(), near.gather_pyramid()):
        assert torch.equal(x, y)
    base = torch.stack(torch.meshgrid(torch.arange(w).float(), torch.arange(h).float(), indexing="xy"), -1)
    coords = (base[None, None] + 4 * torch.randn(1, 3, h, w, 2, generator=g)).to(dev())
    assert torch.equal(far(coords).view(torch.int16), near(coords).view(torch.int16))
    del far, near, big
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------- fallback
@pytest.mark.parametrize("dtype,hw", [(torch.float16, (20, 129)), (torch.float16, (24, 160)),
                                      (torch.float32, (9, 13)), (torch.float32, (23, 66))])
def test_fallback_build_and_lookup(dtype, hw):
    """just outside the envelope (half with w > 128, or float32): the CUDA-core build and the row-major lookup,
    under the same level-0 bound and pooling check; the half lookup bit for bit, the float one within 1 ulp"""
    from goslam_b200.modules import CorrBlock
    h, w = hw
    g = torch.Generator().manual_seed(h + w)
    f = _random_fmaps(4, h, w, 1.0, g, dtype)
    f1, f2 = f[0:2, 0][None], f[2:4, 0][None]
    blk = CorrBlock(f1.to(dev()), f2.to(dev()))
    assert blk.pool is None
    pyr = blk.gather_pyramid()
    assert all(p.dtype == dtype for p in pyr)
    worst = _check_level0(pyr[0], f1[0].to(dev()), f2[0].to(dev()), (hw, dtype))
    print("level0 fallback %s %s worst |err| / bound = %.3f" % (str(dtype)[6:], hw, worst))
    _check_pooling(pyr, (hw, dtype))
    coords = _sweep_coords(h, w, 4, g)
    _lookup_vs_oracle(blk, _sweep_calls(coords, 2, h, w), (hw, dtype), exact=dtype == torch.float16)


# --------------------------------------------------------------------------------------------- non-finite
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("shape", [(2, 9, 11, 7, 10), (1, 6, 8, 12, 16), (2, 5, 7, 3, 5), (1, 8, 8, 1, 1)])
def test_corr_index_forward_nonfinite_coordinates(dtype, shape):
    """NaN, +-inf, +-3e9 and +-1e30 in x and/or y: taps outside the level add nothing, as in the reference"""
    from goslam_b200 import droid_backends
    g = torch.Generator().manual_seed(sum(shape) + dtype.itemsize)
    vol = torch.randn(*shape, generator=g).to(dtype)
    coords = nonfinite_coords(*shape, g)
    out, = droid_backends.corr_index_forward(vol.to(dev()), coords.to(dev()), 3)
    got = out.cpu().numpy()
    want = corr_oracle.corr_index_forward(vol.numpy(), coords.numpy(), 3)
    N, h1, w1, h2, w2 = shape
    if h2 >= 5 and w2 >= 5:
        assert np.isnan(got[0].reshape(49, -1)[:, 0]).sum() == 25          # x = y = NaN
    assert (got[0].reshape(49, -1)[:, 1] == 0).all()                       # x = NaN, y = +inf
    if dtype == torch.float16:
        np.testing.assert_array_equal(got.astype(np.float32), want.astype(np.float32))
    else:
        assert np.array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_allclose(got, want, rtol=2e-7, atol=1e-7)


@pytest.mark.parametrize("hw", [(9, 13), (22, 50), (37, 127)])
def test_pooled_lookup_nonfinite_coordinates(hw):
    from goslam_b200.modules import CorrBlock
    h, w = hw
    g = torch.Generator().manual_seed(h * w)
    f1 = torch.randn(1, 2, 128, h, w, generator=g).half()
    f2 = torch.randn(1, 2, 128, h, w, generator=g).half()
    blk = CorrBlock(f1.to(dev()), f2.to(dev()))
    assert blk.pool is not None
    c = nonfinite_coords(2, h, w, h, w, g)                                 # [N, 2, h, w]
    coords = c.permute(0, 2, 3, 1)[None].contiguous()
    out = blk(coords.to(dev()))[0].cpu().numpy()
    want = corr_oracle.corr_pyramid_lookup([p.cpu().numpy() for p in blk.gather_pyramid()], coords[0].numpy(), 3)
    assert np.isnan(out[0, :49, 0, 0]).sum() == 25 and (out[0, :, 0, 1] == 0).all()
    np.testing.assert_array_equal(out.astype(np.float32), want.astype(np.float32))


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_nonfinite_coordinates_vs_reference_kernel(dtype):
    """the reference's own corr_index_forward on non-finite and huge coordinates (stored in ref_kernels.npz)"""
    from goslam_b200 import droid_backends
    g = torch.Generator().manual_seed(404)
    shape = (1, 4, 4, 7, 9)
    vol = torch.randn(*shape, generator=g).to(dtype).to(dev())
    coords = nonfinite_coords(*shape, g).to(dev())
    ours, = droid_backends.corr_index_forward(vol, coords, 3)
    c = ref_golden.compare("corr_index_nonfinite/%s" % str(dtype)[6:], {"out": ours},
                           lambda ref: {"out": ref.corr_index_forward(vol, coords, 3)[0]})
    a, b, _ = c["out"]
    assert torch.isnan(b).any() and (b == 0).any()
    np.testing.assert_array_equal(a.float().numpy(), b.float().numpy())
