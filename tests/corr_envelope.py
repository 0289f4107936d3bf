"""Shapes and layout facts shared by the correlation envelope tests (test_corr_layout_host.py on the CPU,
test_gpu_corr_envelope.py on the device)."""
import math

import torch

# (h, w) of level 0, all inside the tensor-core build's envelope (half, D = 128, w <= 128).  Together they cover
# every x-tile count n_xb = ceil(w / 16) from 1 to 8 (n_xb = 8 is the 218 KB shared-memory configuration), every
# h % 8 (the rows of the last 8-row band), every w % 4 (ragged 4x4 tiles), w < 16 (the 8x16 target patch wider
# than the image), and h*w < 128, h*w % 128 == 0, h*w % 16 != 0 and h*w % 8 != 0 (ragged 128-pixel source tiles,
# the lookup's scalar store path).  test_corr_layout_host.py asserts that coverage.
SHAPES = [(8, 8), (9, 13), (11, 17), (15, 31), (17, 45), (22, 50), (23, 66), (26, 81), (12, 96), (29, 97),
          (33, 112), (44, 100), (19, 113), (37, 127), (40, 128), (48, 128)]


def plane_positions(ht, wd, level, num_levels=4, device="cpu"):
    """[ht >> level, wd >> level] int64: the element of a source pixel's tiled plane that holds each entry of the
    level, read off CorrPool.level_rowmajor applied to a plane of indices."""
    from goslam_b200.modules.corr import CorrPool
    pool = CorrPool(0, ht, wd, num_levels, device=device)
    plane = pool.plane_elems[level]
    pool.levels[level] = torch.arange(plane, dtype=torch.int32, device=device).expand(1, ht * wd, plane)
    return pool.level_rowmajor(level)[0, 0, 0].long()


def padding_mask(ht, wd, level, num_levels=4, device="cpu"):
    """bool [plane_elems]: the elements of a tiled plane that hold no entry of the level."""
    from goslam_b200.modules.corr import CorrPool
    plane = CorrPool(0, ht, wd, num_levels, device=device).plane_elems[level]
    mask = torch.ones(plane, dtype=torch.bool, device=device)
    mask[plane_positions(ht, wd, level, num_levels, device).reshape(-1)] = False
    return mask


BAD = [math.nan, math.inf, -math.inf, 3e9, -3e9, 1e30, -1e30]


def nonfinite_coords(N, h1, w1, h2, w2, g):
    """[N, 2, h1, w1] f32: random coordinates around the level, the first pixels overwritten with every pairing of
    NaN, +-inf, +-3e9 and +-1e30 with each other and with finite partners (inside and hanging over a border)"""
    c = torch.stack([torch.rand(N, h1, w1, generator=g) * (w2 + 6) - 3,
                     torch.rand(N, h1, w1, generator=g) * (h2 + 6) - 3], 1)
    pairs = [(a, b) for a in BAD for b in BAD + [1.25, -2.5]] + [(b, a) for a in BAD for b in (2.75, w2 + 0.5)]
    flat = c.permute(0, 2, 3, 1).reshape(-1, 2)
    k = min(len(pairs), flat.shape[0])
    flat[:k] = torch.tensor(pairs[:k], dtype=torch.float32)
    return flat.reshape(N, h1, w1, 2).permute(0, 3, 1, 2).contiguous()
