"""Reference spot sums (test helper, numpy only): what the `[n_tiles, 16]` summary of a grid launch
must hold, given the launch's per-ray ``status``, transverse aberration ``ax``, ``ay`` and ``op``.

Column layout (engine.SUMMARY_FIELDS): 0-4 ray counts by status class (0, 1, 2, 3, anything else),
5-9 the sums of x, y, x*x, y*y, x*y, 10-13 min x, max x, min y, max y, 14 the sum of op, 15 zero.
Only status-0 rays enter columns 5-14.

Two references:

* ``exact_summary``: counts, ``np.fmin`` / ``np.fmax`` (NaN skipped, +-inf for a tile without a
  status-0 ray) and the six sums correctly rounded (``math.fsum``) over the very doubles the kernel
  adds.  The products x*x, y*y, x*y are rounded once, as the kernel forms them (the library is built
  with ``-fmad=false``), so the only error left in a kernel sum is that of its additions;
  ``sum_bound`` bounds it by gamma_d * sum |x_i|, gamma_d = d u / (1 - d u), u = 2^-53, with d the
  depth of the addition chain (plus one for the rounding of the fsum itself).

* ``ordered_summary``: the same six sums added in the order the library documents, in float64:

  1. A work item (32 consecutive rays of a chunk; one warp) is summed by the halving tree
     ``s1[i] = x[i] + x[i+16]`` (i < 16), ``s2[i] = s1[i] + s1[i+8]``, ``s3[i] = s2[i] + s2[i+4]``,
     ``s4[i] = s3[i] + s3[i+2]``, ``s4[0] + s4[1]``; lanes without a status-0 ray hold +0.0.
     ``warp_record_from_regs`` forms exactly this tree with ``shfl_down`` (lane i adds lane
     i + off for off = 16, 8, 4, 2, 1; lane 0's result).  ``item_sums_store`` uses an xor butterfly:
     at step ``off`` lane l adds its own value and that of lane l ^ off.  For l < l ^ off this is
     ``v[l] + v[l + off]``; for the partner it is ``v[l] + v[l - off]``, the same double because
     IEEE addition is commutative.  By induction, after the steps 16, 8, ..., off every lane l holds
     the tree value at index ``l mod off`` of the value it keeps, so the lanes that store the
     result hold ``s4[0] + s4[1]``.  Handing half of the values to the partner at the 16 / 8 / 4
     steps only moves which lane holds which column; it adds nothing.
  2. ``reduce_tile`` takes the tile's entries (per-chunk record slots, or work items), splits them
     into RT_RED_SPLIT = 16 contiguous parts of ceil(n / 16); within a part, thread t of 256 adds
     entries t, t + 256, ... in ascending order starting from +0.0; a halving tree over the 256
     thread sums (``t[i] += t[i + off]``, off = 128 ... 1) gives the part's partial; the 16
     partials are added in part order, ``((p0 + p1) + p2) + ...``.
  3. The entries.  Per-chunk record regime (a launch with ``chunks_per_tile <= gridDim.x``): the
     ``sl * 8`` record slots of the tile, sl = min(chunks_per_tile, 2048), slot = local chunk * 8 +
     warp, i.e. the tile's work items in order; slots of chunks outside the launch's chunk range
     are skipped but still count for the part boundaries.  Work-item regime (otherwise, dynamic
     schedule): only the tile's items inside ``[chunk_begin, chunk_end)``, in order.
  4. ``combine``: partial summaries (pieces of ``rt_trace_grid_to_host``, shards) are added in
     part order, ``k_combine_summaries``' loop.

The regime of a launch follows from its CTA count ``min(SMs x resident CTAs, chunk_end -
chunk_begin, 2048)``; ``regime`` names the shapes where it is certain.  The static schedule's
per-CTA regime (``B200RT_STATIC=1`` and no per-chunk records) adds rays in per-thread chains whose
split depends on the CTA count; there only ``sum_bound`` applies."""
import math

import numpy as np

CHUNK = 256              # rays per chunk (RT_BLOCK)
ITEM = 32                # rays per work item (one warp)
WARPS = CHUNK//ITEM      # work items per chunk (RT_WARPS)
RED_SPLIT = 16           # reduce CTAs per tile (RT_RED_SPLIT)
RED_THREADS = 256        # threads per reduce CTA (RT_RED_THREADS)
MAX_GRID = 2048          # CTA cap of a launch and of record slots per tile (RT_MAX_GRID)
SUM_COLS = (5, 6, 7, 8, 9, 14)
MIN_COLS, MAX_COLS = (10, 12), (11, 13)
U = 2.0**-53


class Shape:
    """The grid shape of one launch: tiles of ``rays_per_tile`` rays, ``chunks_per_tile`` chunks
    each, chunk range ``[chunk_begin, chunk_end)``."""

    def __init__(self, rays_per_tile, n_tiles, chunk_begin=0, chunk_end=None):
        self.rays_per_tile, self.n_tiles = int(rays_per_tile), int(n_tiles)
        self.chunks_per_tile = -(-self.rays_per_tile//CHUNK)
        self.n_chunks = self.n_tiles*self.chunks_per_tile
        self.chunk_begin = int(chunk_begin)
        self.chunk_end = self.n_chunks if chunk_end is None else int(chunk_end)
        assert 0 <= self.chunk_begin <= self.chunk_end <= self.n_chunks

    @classmethod
    def of(cls, grid, chunk_begin=0, chunk_end=None):
        return cls(grid.rays_per_tile, grid.n_tiles, chunk_begin, chunk_end)

    def sub(self, chunk_begin, chunk_end):
        return Shape(self.rays_per_tile, self.n_tiles, chunk_begin, chunk_end)

    def first_ray(self, chunk):
        tile, lc = divmod(chunk, self.chunks_per_tile)
        return tile*self.rays_per_tile + min(lc*CHUNK, self.rays_per_tile)

    @property
    def n_rays(self):
        return self.first_ray(self.chunk_end) - self.first_ray(self.chunk_begin)

    def tile_range(self, tile):
        """chunks of ``tile`` inside the launch's range, as local chunk indices [l0, l1)"""
        base = tile*self.chunks_per_tile
        c0 = max(base, self.chunk_begin)
        c1 = max(min(base + self.chunks_per_tile, self.chunk_end), c0)
        return c0 - base, c1 - base


def regime(shape, sm_count, max_ctas_per_sm):
    """'records' | 'items' for the launch over ``shape``'s chunk range ('empty' for no chunks), or
    None where it depends on the occupancy the runtime reports.  ``max_ctas_per_sm``: an upper bound of resident
    256-thread CTAs per SM (threads and shared memory of the summary kernels)."""
    n = shape.chunk_end - shape.chunk_begin
    cpt = shape.chunks_per_tile
    if n == 0:
        return 'empty'
    if cpt <= min(sm_count, n):
        return 'records'
    if cpt > min(sm_count*max_ctas_per_sm, n, MAX_GRID):
        return 'items'
    return None


def _tile_values(shape, status, ax, ay, op):
    """per tile: (ok mask, the six summands) of the launch's rays, in ray order"""
    status = np.asarray(status)
    assert len(status) == shape.n_rays
    base = shape.first_ray(shape.chunk_begin)
    ok = status == 0
    zero = np.zeros(len(status))
    ax, ay, op = (np.where(ok, np.asarray(v, dtype=np.float64), zero) for v in (ax, ay, op))
    with np.errstate(all='ignore'):
        six = np.stack([ax, ay, ax*ax, ay*ay, ax*ay, op], axis=1)
    six[~ok] = 0.0
    for t in range(shape.n_tiles):
        a = max(shape.first_ray(t*shape.chunks_per_tile), shape.first_ray(shape.chunk_begin)) - base
        b = min(shape.first_ray((t + 1)*shape.chunks_per_tile), shape.first_ray(shape.chunk_end)) - base
        b = max(a, b)
        yield t, status[a:b], ok[a:b], six[a:b]


def identity_summary(n_tiles):
    s = np.zeros((n_tiles, 16))
    s[:, list(MIN_COLS)] = np.inf
    s[:, list(MAX_COLS)] = -np.inf
    return s


def _counts_minmax(s, t, st, ok, six):
    cls = np.where((st >= 0) & (st <= 3), st, 4)
    s[t, 0:5] = np.bincount(cls, minlength=5)[:5]
    if ok.any():
        with np.errstate(invalid='ignore'):
            x, y = six[ok, 0], six[ok, 1]
            s[t, 10], s[t, 11] = np.fmin.reduce(x, initial=np.inf), np.fmax.reduce(x, initial=-np.inf)
            s[t, 12], s[t, 13] = np.fmin.reduce(y, initial=np.inf), np.fmax.reduce(y, initial=-np.inf)


def exact_summary(shape, status, ax, ay, op):
    """counts, fmin / fmax and correctly rounded sums of the launch's rays, ``[n_tiles, 16]``;
    also returns ``[n_tiles, 6]`` sums of |summand| for ``sum_bound``"""
    s = identity_summary(shape.n_tiles)
    absum = np.zeros((shape.n_tiles, 6))
    for t, st, ok, six in _tile_values(shape, status, ax, ay, op):
        _counts_minmax(s, t, st, ok, six)
        for j, c in enumerate(SUM_COLS):
            v = six[ok, j]
            s[t, c] = math.fsum(v) if np.isfinite(v).all() else np.sum(v)
            absum[t, j] = math.fsum(np.abs(v)) if np.isfinite(v).all() else np.inf
    return s, absum


def chain_depth(shape, regime_, pieces=1, static=False):
    """depth of the kernel's addition chain for one tile: the item tree (5), a thread's run
    through its part, the 256-thread tree (8), the 16 partials (15), the combine of the pieces;
    the static schedule's per-CTA regime adds a per-thread run over the chunks of the tile"""
    cpt = shape.chunks_per_tile
    n = min(cpt, MAX_GRID)*WARPS if regime_ == 'records' or static else cpt*WARPS
    per = -(-n//RED_SPLIT)
    d = 5 + -(-per//RED_THREADS) + 8 + (RED_SPLIT - 1) + (pieces - 1)
    if static:
        d += cpt
    return d + 1                      # + the rounding of the correctly rounded reference


def sum_bound(absum, depth):
    """gamma_d * sum |x_i|"""
    g = depth*U/(1.0 - depth*U)
    return g*absum


def item_tree(v):
    """the halving tree of one work item over axis -2 (32 lanes)"""
    assert v.shape[-2] == ITEM
    half = ITEM//2
    while half >= 1:
        v = v[..., :half, :] + v[..., half:2*half, :]
        half //= 2
    return v[..., 0, :]


def reduce_entries(e, valid):
    """``reduce_tile`` over entries ``e`` ``[n, k]`` (``valid``: entries that are added)"""
    n, k = e.shape
    e = np.where(valid[:, None], e, 0.0)    # x + (+0.0) == x: x starts at +0.0 and is never -0.0
    per = -(-n//RED_SPLIT)
    parts = []
    for p in range(RED_SPLIT):
        r0, r1 = min(p*per, n), min(p*per + per, n)
        m = r1 - r0
        rows = -(-m//RED_THREADS)
        blk = np.zeros((max(rows, 1)*RED_THREADS, k))
        blk[:m] = e[r0:r1]
        blk = blk.reshape(-1, RED_THREADS, k)
        x = np.zeros((RED_THREADS, k))
        for r in range(blk.shape[0]):
            x = x + blk[r]
        off = RED_THREADS//2
        while off >= 1:
            x = np.concatenate([x[:off] + x[off:2*off], x[2*off:]])
            off //= 2
        parts.append(x[0])
    v = parts[0]
    for p in parts[1:]:
        v = v + p
    return v


def tile_items(shape, t, ok, six):
    """the tile's work-item sums ``[chunks_per_tile * 8, 6]`` (items outside the range: 0) and
    the in-range mask"""
    cpt = shape.chunks_per_tile
    l0, l1 = shape.tile_range(t)
    lanes = np.zeros((cpt*CHUNK, 6))
    start = l0*CHUNK
    lanes[start:start + len(six)] = six
    items = item_tree(lanes.reshape(cpt*WARPS, ITEM, 6))
    inr = np.zeros(cpt*WARPS, bool)
    inr[l0*WARPS:l1*WARPS] = True
    return items, inr


def ordered_summary(shape, status, ax, ay, op, regime_):
    """the summary a launch over ``shape`` returns, its six sums in the documented order"""
    s = identity_summary(shape.n_tiles)
    if shape.chunk_end == shape.chunk_begin:
        return s
    assert regime_ in ('records', 'items')
    for t, st, ok, six in _tile_values(shape, status, ax, ay, op):
        _counts_minmax(s, t, st, ok, six)
        items, inr = tile_items(shape, t, ok, six)
        with np.errstate(invalid='ignore'):
            if regime_ == 'records':
                assert shape.chunks_per_tile <= MAX_GRID
                v = reduce_entries(items, inr)
            else:
                v = reduce_entries(items[inr], np.ones(int(inr.sum()), bool))
        s[t, list(SUM_COLS)] = v
    return s


def combine(parts):
    """``k_combine_summaries``: parts added (min / max taken) in part order"""
    out = np.array(parts[0], dtype=np.float64)
    for p in parts[1:]:
        with np.errstate(invalid='ignore'):
            out[:, :10] = out[:, :10] + p[:, :10]
            out[:, 14:] = out[:, 14:] + p[:, 14:]
            out[:, list(MIN_COLS)] = np.fmin(out[:, list(MIN_COLS)], p[:, list(MIN_COLS)])
            out[:, list(MAX_COLS)] = np.fmax(out[:, list(MAX_COLS)], p[:, list(MAX_COLS)])
    return out


def spot_reference(x, y):
    """centroid, variance (squared RMS radius) by two passes of correctly rounded sums, and
    a = (sum x^2 + sum y^2) / n, the size of the terms the one-pass formula cancels:
    kappa = a / var"""
    n = len(x)
    cx, cy = math.fsum(x)/n, math.fsum(y)/n
    dx, dy = x - cx, y - cy
    var = math.fsum(np.concatenate([dx*dx, dy*dy]))/n
    a = math.fsum(np.concatenate([x*x, y*y]))/n
    return cx, cy, var, a
