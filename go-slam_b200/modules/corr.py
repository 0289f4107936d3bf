"""CorrBlock / AltCorrBlock with the reference's constructor and call signatures
(src/modules/corr.py:25-65,97-145), backed by the sm_90a kernels.

CorrBlock(fmap1, fmap2)      -> half inputs with D == 128, w <= 128: the wgmma all-pairs build with the
                                4-level pyramid in its epilogue, into a private CorrPool (goslam_corr_pool_build);
                                anything else (float32, other shapes): the CUDA-core build, row-major
                                (goslam_corr_build).  Reference: torch.matmul + 3x avg_pool2d.
CorrBlock.__call__(coords)   -> ONE fused 4-level radius-3 lookup (goslam_corr_pool_lookup /
                                goslam_corr_pyramid_lookup; reference: 4 x corr_index_forward + torch.cat)
AltCorrBlock(fmaps)(coords, ii, jj) -> windowed correlation, all levels in one launch (goslam_altcorr_pyramid)

A pooled pyramid is in the tiled layout, private to the build and lookup kernels; `corr_pyramid` /
`gather_pyramid()` give the reference's [N, h, w, h>>i, w>>i] levels as a de-tiled copy.
"""
import torch
import torch.nn.functional as F

from .. import _lib
from .._lib import ptr_array as _ptr_array


class CorrPool:
    """Slot pool for the correlation pyramids of a factor graph (SURVEY §8 a3).

    The reference concatenates / boolean-masks the whole pyramid on every add_factors /
    rm_factors (src/modules/corr.py:55-65 via src/factor_graph.py:114,149) — a copy of up to
    N*hw*1.33*hw*2 bytes each time.  Here the graph owns `capacity` slots per level, allocated
    once (FactorGraph.max_factors is the natural capacity); a CorrBlock built `from_video(...,
    pool=pool)` holds only a table of slot ids, so cat() joins two tables and __getitem__ filters
    one.  The build and lookup kernels follow the table on the device
    (goslam_corr_pool_build_paired / goslam_corr_pool_lookup_aliased).

    Reverse edges share level 0: corr(j,i)[q][p] == corr(i,j)[p][q] bit for bit, so when one build call holds
    both (i, j) and (j, i) once each, the later one (the reader) writes levels 1-3 only and reads level 0 as
    the transpose of its partner's.  `alias[s]` (int32, device) = 2 * (slot holding slot s's level 0) + (1 if
    transposed), in word 0 of a 16-byte row; the build writes it for every slot it fills.  Pairs never cross a build call, so they never
    cross a block; a block that keeps a reader but lets its partner go materializes the reader's level 0 first
    (`unalias`).  Every reader still owns its level-0 region, so slot bookkeeping is unchanged."""

    TILED = 1                                                    # == GOSLAM_LAYOUT_TILED

    def __init__(self, capacity, ht, wd, num_levels=4, device="cuda", layout="tiled"):
        """levels 0/1 as 4x4-element tiles (one 32-byte sector each), levels 2/3 as padded band pieces,
        private to the build and lookup kernels — nothing else in GO-SLAM reads the pyramid
        (include/goslam_b200.h, GOSLAM_LAYOUT_TILED).  "tiled" is the only layout."""
        if layout != "tiled":
            raise ValueError("CorrPool: layout must be \"tiled\", got %r" % (layout,))
        self.capacity, self.ht, self.wd, self.num_levels = int(capacity), ht, wd, num_levels
        self.plane_elems = [self._plane_elems(i) for i in range(num_levels)]
        self.levels = [torch.empty((self.capacity, ht * wd, self.plane_elems[i]), dtype=torch.float16, device=device)
                       for i in range(num_levels)]
        self._free = list(range(self.capacity - 1, -1, -1))     # stack; slot 0 is handed out first
        self._iota = torch.arange(self.capacity, dtype=torch.int32, device=device)
        # [capacity, 4]: word 0 of a row is the entry, the 16-byte rows let the build write them with bulk copies
        self.alias = torch.zeros((self.capacity, 4), dtype=torch.int32, device=device)
        self.alias[:, 0] = self._iota * 2                        # every slot holds its own level 0
        self.paired = False                                      # set once a paired build has run

    def slot_table(self, slots):
        """device int32 table for a list of slot ids (a view of a resident iota when the ids are a
        consecutive run — the common case — so that no host->device copy is needed)."""
        n = len(slots)
        if n and slots[-1] - slots[0] == n - 1 and all(slots[i + 1] == slots[i] + 1 for i in range(n - 1)):
            return self._iota[slots[0]:slots[0] + n]
        return torch.tensor(slots, dtype=torch.int32, device=self._iota.device)

    def _plane_elems(self, i):                                   # == goslam_corr_level_plane_elems
        hl, wl = self.ht >> i, self.wd >> i
        if i < 2:
            return ((hl + 3) // 4) * ((wl + 3) // 4) * 16
        n_yb, n_xb = (self.ht + 7) // 8, (self.wd + 15) // 16
        return n_yb * ((n_xb * 8 + 15) // 16 * 16) if i == 2 else n_yb * 16

    def level_rowmajor(self, i, slots=None):
        """level i as [n, ht, wd, ht>>i, wd>>i] (a gathered, de-tiled copy; tests / debugging); an aliased level 0
        is read through `alias`, as the lookup reads it."""
        if i == 0 and self.paired:
            slots = self._iota.long() if slots is None else torch.as_tensor(slots, device=self.alias.device).long()
            al = self.alias[slots, 0].long()
            own = self._detile(0, self.levels[0][al >> 1])
            return torch.where((al & 1).bool().view(-1, 1, 1, 1, 1), own.permute(0, 3, 4, 1, 2), own).contiguous()
        return self._detile(i, self.levels[i] if slots is None else self.levels[i][slots])

    def _detile(self, i, lvl):
        hl, wl = self.ht >> i, self.wd >> i
        n = lvl.shape[0]
        if i < 2:
            h4, w4 = (hl + 3) // 4, (wl + 3) // 4
            lvl = lvl.view(n, self.ht, self.wd, h4, w4, 4, 4).permute(0, 1, 2, 3, 5, 4, 6)
            return lvl.reshape(n, self.ht, self.wd, 4 * h4, 4 * w4)[..., :hl, :wl].contiguous()
        n_yb, n_xb = (self.ht + 7) // 8, (self.wd + 15) // 16
        if i == 2:              # per band: 2 rows of n_xb*4 columns, padded to a multiple of 16 elements
            lvl = lvl.view(n, self.ht, self.wd, n_yb, -1)[..., :2 * n_xb * 4]
            return lvl.reshape(n, self.ht, self.wd, 2 * n_yb, n_xb * 4)[..., :hl, :wl].contiguous()
        return lvl.view(n, self.ht, self.wd, n_yb, 16)[..., :hl, :wl].contiguous()

    @property
    def free_slots(self):
        return len(self._free)

    def alloc(self, n):
        if n > len(self._free):
            raise RuntimeError("CorrPool exhausted: %d slots requested, %d free of %d"
                               % (n, len(self._free), self.capacity))
        out = self._free[len(self._free) - n:][::-1]
        del self._free[len(self._free) - n:]
        return out

    def release(self, slots):
        self._free.extend(reversed(list(slots)))

    def grow(self, capacity):
        """enlarge the pool (graphs created with max_factors = -1 have no bound, e.g. PoseTrajectoryFiller's,
        src/trajectory_filler.py:63): new buffers, one copy of the old slots, slot ids stay valid."""
        capacity = int(capacity)
        if capacity <= self.capacity:
            return
        dev = self.levels[0].device
        for i, old in enumerate(self.levels):
            new = torch.empty((capacity,) + tuple(old.shape[1:]), dtype=old.dtype, device=dev)
            new[:self.capacity].copy_(old)
            self.levels[i] = new
        self._free = list(range(capacity - 1, self.capacity - 1, -1)) + self._free
        self._iota = torch.arange(capacity, dtype=torch.int32, device=dev)
        alias = torch.zeros((capacity, 4), dtype=torch.int32, device=dev)
        alias[:self.capacity].copy_(self.alias)                  # live aliases carry over
        alias[self.capacity:, 0] = self._iota[self.capacity:] * 2
        self.alias = alias
        self.capacity = capacity

    def unalias(self, slots, keep=lambda holder: False):
        """give each of `slots` whose level 0 is another slot's transpose its own copy, unless `keep(holder)`
        (one device kernel; reads the slots' alias entries on the host)."""
        if not self.paired or not slots:
            return
        al = self.alias[self.slot_table(list(slots)).long(), 0].tolist()
        todo = [(s, a >> 1) for s, a in zip(slots, al) if a & 1 and not keep(a >> 1)]
        if todo:
            dev = self.alias.device
            ss = torch.tensor([s for s, _ in todo], dtype=torch.int32, device=dev)
            hs = torch.tensor([t for _, t in todo], dtype=torch.int32, device=dev)
            _lib.call("corr_pool_unalias", self.levels[0], self.alias, ss, hs, len(todo), self.ht, self.wd)


class CorrBlock:
    """A half-precision block inside the tensor-core envelope lives in a CorrPool (`pool`, `slots`,
    `_slots_host`): the factor graph's, or a private one.  Any other block holds the reference's
    row-major list of levels (`_levels`) from the CUDA-core build."""
    pool = None

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        self.num_levels = num_levels
        self.radius = radius
        if not fmap1.is_cuda:
            raise RuntimeError("CorrBlock: CUDA tensors required (no CPU fallback)")
        batch, num, dim, ht, wd = fmap1.shape
        N = batch * num
        self.ht, self.wd = ht, wd
        dev = fmap1.device
        if fmap1.dtype == torch.float16 and dim == 128 and wd <= 128:
            # both maps K-major in one [2N, hw, 128] buffer; edge e pairs frame e with frame N + e
            km = torch.empty((2 * N, ht * wd, 128), dtype=torch.float16, device=dev)
            fmaps_to_kmajor(fmap1.reshape(N, dim, ht, wd), out=km[:N])
            fmaps_to_kmajor(fmap2.reshape(N, dim, ht, wd).half(), out=km[N:])
            ii = torch.arange(N, device=dev)
            self._build_pooled(km, ii, ii + N, 1, None)
            return
        dtype = torch.float16 if fmap1.dtype == torch.float16 else torch.float32
        f1 = fmap1.reshape(N, dim, ht, wd).to(dtype).contiguous()
        f2 = fmap2.reshape(N, dim, ht, wd).to(dtype).contiguous()
        self._levels = [torch.empty((N, ht, wd, ht >> i, wd >> i), dtype=dtype, device=dev)
                        for i in range(num_levels)]
        _lib.call("corr_build", f1, f2, 1 if dtype == torch.float16 else 0, _ptr_array(self._levels), num_levels,
                  N, dim, ht, wd)

    @classmethod
    def from_video(cls, fmaps_kmajor, ii, jj, ht, wd, rig=1, num_levels=4, radius=3, pool=None):
        """FactorGraph.add_factors' volume for edges (ii, jj) straight from video-level K-major
        feature maps [buffer*rig, ht*wd, 128] (see `fmaps_to_kmajor`): no gathered copies.
        The volumes are written into free slots of `pool`, or of a private CorrPool without one."""
        self = cls.__new__(cls)
        self.num_levels, self.radius, self.ht, self.wd = num_levels, radius, ht, wd
        self._build_pooled(fmaps_kmajor, ii, jj, rig, pool)
        return self

    def _build_pooled(self, fmaps_kmajor, ii, jj, rig, pool):
        dev = fmaps_kmajor.device
        N = int(ii.shape[0])
        if pool is None:
            pool = CorrPool(N, self.ht, self.wd, self.num_levels, device=dev)
        elif (pool.ht, pool.wd, pool.num_levels) != (self.ht, self.wd, self.num_levels):
            raise RuntimeError("CorrBlock.from_video: pool shape mismatch")
        self.pool = pool
        self._slots_host = pool.alloc(N)
        self.slots = pool.slot_table(self._slots_host)
        _lib.call("corr_pool_build_paired", fmaps_kmajor, int(fmaps_kmajor.shape[0]), int(rig), ii, jj, self.slots,
                  pool.alias, _ptr_array(pool.levels), self.num_levels, N, 128, self.ht, self.wd)
        pool.paired = pool.paired or N > 1

    def __call__(self, coords):
        batch, num, ht, wd, _ = coords.shape
        N = batch * num
        if self.pool is not None:
            return self._call_pooled(coords, batch, num, ht, wd)
        vol0 = self._levels[0]
        rd = 2 * self.radius + 1
        coords = coords.reshape(N, ht, wd, 2).contiguous().float()
        out = torch.empty((batch, num, self.num_levels * rd * rd, ht, wd), dtype=vol0.dtype,
                          device=vol0.device)
        pyr = [p.contiguous() for p in self._levels]
        _lib.call("corr_pyramid_lookup", _ptr_array(pyr), 1 if vol0.dtype == torch.float16 else 0, self.num_levels,
                  coords, out, N, ht, wd, vol0.shape[3], vol0.shape[4], int(self.radius))
        return out

    def _call_pooled(self, coords, batch, num, ht, wd):
        N = batch * num
        if N != len(self._slots_host):
            raise RuntimeError("CorrBlock: %d coordinate maps for %d edges" % (N, len(self._slots_host)))
        pool = self.pool
        rd = 2 * self.radius + 1
        coords = coords.reshape(N, ht, wd, 2).contiguous().float()
        out = torch.empty((batch, num, self.num_levels * rd * rd, ht, wd), dtype=torch.float16,
                          device=pool.levels[0].device)
        _lib.call("corr_pool_lookup_aliased", _ptr_array(pool.levels), 1, self.num_levels, self.slots, pool.alias,
                  pool.capacity, pool.TILED, coords, out, N, ht, wd, pool.ht, pool.wd, int(self.radius))
        return out

    def cat(self, other):
        if self.pool is None:
            for i in range(self.num_levels):
                self._levels[i] = torch.cat([self._levels[i], other.corr_pyramid[i]], dim=0)
            return self
        if other.pool is self.pool:
            # O(edges): join the slot tables; `other` gives up its slots
            self._slots_host = self._slots_host + other._slots_host
            self.slots = torch.cat([self.slots, other.slots])
            other._slots_host, other.slots = [], other.slots[:0]
            return self
        if other.pool is None:
            raise RuntimeError("CorrBlock.cat: a pooled block cannot take the edges of a row-major one")
        # blocks in different pools (e.g. two CorrBlock(f1, f2)): both copied into a new private pool, the
        # copy the reference's torch.cat makes; the raw slot copy needs every level 0 materialized first
        self.pool.unalias(self._slots_host)
        other.pool.unalias(other._slots_host)
        n = len(self._slots_host) + len(other._slots_host)
        pool = CorrPool(n, self.ht, self.wd, self.num_levels, device=self.pool.levels[0].device)
        for i, lvl in enumerate(pool.levels):
            torch.cat([self.pool.levels[i][self.slots.long()], other.pool.levels[i][other.slots.long()]], out=lvl)
        self.free()
        self.pool, self._slots_host = pool, pool.alloc(n)
        self.slots = pool.slot_table(self._slots_host)
        return self

    def __getitem__(self, index):
        if self.pool is None:
            for i in range(self.num_levels):
                self._levels[i] = self._levels[i][index]
            return self
        # O(edges): keep the selected slot ids, hand the others back to the pool.  Any index
        # form torch accepts on dim 0 works (FactorGraph passes boolean masks).
        ids = torch.arange(len(self._slots_host))[index.cpu() if torch.is_tensor(index) else index]
        keep = [int(i) for i in ids.reshape(-1).tolist()]
        kept = set(keep)
        if len(kept) != len(keep):
            raise RuntimeError("CorrBlock[index]: a pooled block cannot hold one slot twice")
        gone = [s for i, s in enumerate(self._slots_host) if i not in kept]
        if gone:
            # a kept reader whose partner goes takes a copy of its level 0 before the partner's slot is reused
            kept_slots = set(self._slots_host[i] for i in keep)
            self.pool.unalias([self._slots_host[i] for i in keep], keep=lambda holder: holder in kept_slots)
        self.pool.release(gone)
        self._slots_host = [self._slots_host[i] for i in keep]
        self.slots = self.pool.slot_table(self._slots_host)
        return self

    def free(self):
        """return every slot to the pool (FactorGraph drops `self.corr` when it clears edges)."""
        if self.pool is not None and self._slots_host:
            self.pool.release(self._slots_host)
            self._slots_host, self.slots = [], self.slots[:0]

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def gather_pyramid(self):
        """[N,h,w,h>>i,w>>i] per level: a de-tiled copy for a pooled block (tests / the smoke entry), the
        block's own levels otherwise."""
        if self.pool is None:
            return self._levels
        idx = self.slots.long()
        return [self.pool.level_rowmajor(i, idx) for i in range(self.num_levels)]

    corr_pyramid = property(gather_pyramid)

    @staticmethod
    def corr(fmap1, fmap2):
        """all-pairs correlation, level 0 only ([batch, num, h, w, h, w])."""
        blk = CorrBlock(fmap1, fmap2, num_levels=1)
        batch, num, _, ht, wd = fmap1.shape
        return blk.corr_pyramid[0].view(batch, num, ht, wd, ht, wd)


def fmaps_to_kmajor(fmaps, out=None):
    """DepthVideo.fmaps [buffer, rig, 128, h, w] f16 -> K-major [buffer*rig, h*w, 128] (done once
    per inserted keyframe; `out` lets the caller convert just the new rows in place)."""
    if not fmaps.is_cuda or fmaps.dtype != torch.float16:
        raise RuntimeError("fmaps_to_kmajor: CUDA float16 tensor required")
    f = fmaps.contiguous()
    h, w = f.shape[-2], f.shape[-1]
    F = f.numel() // (128 * h * w)
    if out is None:
        out = torch.empty((F, h * w, 128), dtype=torch.float16, device=f.device)
    _lib.call("fmaps_to_kmajor", f, out, F, 128, h, w)
    return out


class AltCorrBlock:
    """Windowed correlation without a volume (global BA / `update_lowmem`): same constructor and call
    signature as src/modules/corr.py:97-145.  `pyramid[l]` = NHWC feature maps of level l, pre-scaled by
    1/4 and 2x2 average-pooled l times, shape [B, N, H >> l, W >> l, C]."""

    def __init__(self, fmaps, num_levels=4, radius=3):
        self.num_levels, self.radius = num_levels, radius
        b, n, c, h, w = fmaps.shape
        level = fmaps.reshape(b * n, c, h, w) * 0.25            # exact power-of-two scaling, == fmaps / 4.0
        self.pyramid = []
        for lvl in range(num_levels):
            nhwc = level.permute(0, 2, 3, 1).contiguous()
            self.pyramid.append(nhwc.view(b, n, h >> lvl, w >> lvl, c))
            if lvl + 1 < num_levels:
                level = F.avg_pool2d(level, kernel_size=2, stride=2)

    def __call__(self, coords, ii, jj):
        """coords [B, N, H, W, 2] (what FactorGraph.update_lowmem passes) or [B, N, H, W, S, 2] (S coordinate
        sets per edge, the reference's general form): [B, N, L*(2r+1)^2, H, W(, S)] in float32."""
        if not coords.is_cuda:
            raise RuntimeError("AltCorrBlock: CUDA tensors required (no CPU fallback)")
        if coords.dim() == 5:
            return self._fused(coords, ii, jj)
        return torch.stack([self._fused(coords[..., s, :], ii, jj) for s in range(coords.shape[-2])], dim=-1)

    def _fused(self, coords, ii, jj):
        """one launch for all levels, feature maps indexed per edge on the device."""
        B, N, H, W, _ = coords.shape
        if B != 1:
            raise RuntimeError("AltCorrBlock fused path expects batch 1 (as GO-SLAM uses it)")
        C = self.pyramid[0].shape[-1]
        dev = coords.device
        rd = 2 * self.radius + 1
        out = torch.empty((1, N, self.num_levels * rd * rd, H, W), dtype=torch.float32, device=dev)
        pyr = [p.contiguous() if p.dtype == torch.float16 else p.half().contiguous() for p in self.pyramid]
        ii = torch.as_tensor(ii, device=dev).long().contiguous()
        jj = torch.as_tensor(jj, device=dev).long().contiguous()
        c = coords.reshape(N, H, W, 2).float().contiguous()
        _lib.call("altcorr_pyramid", _ptr_array(pyr), self.num_levels, c, ii, jj, out, N, H, W, C, int(self.radius))
        return out
