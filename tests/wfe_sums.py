"""Reference wavefront-error sums (test helper, numpy only): what the ``[n_tiles, RT_WFE_DOUBLES]``
record of ``rt_trace_grid_wfe`` must hold, given the launch's per-ray ``status``, OPD ``W`` and the
rays' relative pupil coordinates ``x``, ``y``.

Column layout (engine.WFE_FIELDS, include/b200rt.h): 0-4 ray counts by status class, 5 / 6 min / max
W (fmin / fmax), 7-19 the 13 sums of W, W*W, x*W, y*W, r2*W, x, y, x*x, x*y, y*y, x*r2, y*r2, r2*r2
with r2 = x*x + y*y (every product rounded once, as the kernel forms them: the library is built
with ``-fmad=false``), 20-23 zero.  Only status-0 rays enter columns 5-19.

The sums are added as the spot sums of ``tests/spot_sums.py`` in their work-item regime (DESIGN.md
section 4): the halving tree over the 32 rays of a work item (``wfe_item_sums_store``: the 16-slot
transposition tree), ``reduce_tile`` over the tile's work items inside the chunk range, partial
records combined in part order.  ``Shape``, ``item_tree``, ``reduce_entries``, ``chain_depth`` and
``sum_bound`` of ``spot_sums`` take any number of columns and are used as they are; ``combine``
is restated here for this record layout."""
import math

import numpy as np

from spot_sums import CHUNK, ITEM, WARPS, Shape, item_tree, reduce_entries, chain_depth, sum_bound  # noqa: F401

WIDTH = 24
SUM_COLS = tuple(range(7, 20))
MIN_COL, MAX_COL = 5, 6
N_SUMS = len(SUM_COLS)


def summands(w, x, y, ok=None):
    """``[n, 13]`` summands in the kernel's column order; rays outside ``ok`` hold +0.0"""
    w, x, y = (np.asarray(v, dtype=np.float64) for v in (w, x, y))
    with np.errstate(all='ignore'):
        r2 = x*x + y*y
        v = np.stack([w, w*w, x*w, y*w, r2*w, x, y, x*x, x*y, y*y, x*r2, y*r2, r2*r2], axis=1)
    if ok is not None:
        v[~np.asarray(ok, bool)] = 0.0
    return v


def grid_pupil_xy(spec, shape):
    """per-ray (x, y) of the launch's rays: the grid's pupil tables as the kernel reads them
    (a product grid without vignetting, the layout ``wavefront_error`` builds)"""
    assert not spec.paired and not spec.apply_vignetting
    xs, ys = [], []
    for t in range(shape.n_tiles):
        f = t//spec.n_wvls
        gx, gy = np.meshgrid(spec.pupil_x[f], spec.pupil_y[f], indexing='ij')
        xs.append(gx.ravel())
        ys.append(gy.ravel())
    x, y = np.concatenate(xs), np.concatenate(ys)
    a, b = shape.first_ray(shape.chunk_begin), shape.first_ray(shape.chunk_end)
    return x[a:b], y[a:b]


def identity(n_tiles):
    s = np.zeros((n_tiles, WIDTH))
    s[:, MIN_COL] = np.inf
    s[:, MAX_COL] = -np.inf
    return s


def _tiles(shape, status, w, x, y):
    status = np.asarray(status)
    assert len(status) == shape.n_rays
    base = shape.first_ray(shape.chunk_begin)
    ok = status == 0
    v = summands(w, x, y, ok)
    w = np.asarray(w, dtype=np.float64)
    for t in range(shape.n_tiles):
        a = max(shape.first_ray(t*shape.chunks_per_tile), base) - base
        b = min(shape.first_ray((t + 1)*shape.chunks_per_tile), shape.first_ray(shape.chunk_end)) - base
        b = max(a, b)
        yield t, status[a:b], ok[a:b], w[a:b], v[a:b]


def _counts_minmax(s, t, st, ok, w):
    cls = np.where((st >= 0) & (st <= 3), st, 4)
    s[t, 0:5] = np.bincount(cls, minlength=5)[:5]
    if ok.any():
        s[t, MIN_COL] = np.fmin.reduce(w[ok], initial=np.inf)
        s[t, MAX_COL] = np.fmax.reduce(w[ok], initial=-np.inf)


def exact_summary(shape, status, w, x, y):
    """counts, fmin / fmax and correctly rounded sums; also ``[n_tiles, 13]`` sums of |summand|"""
    s = identity(shape.n_tiles)
    absum = np.zeros((shape.n_tiles, N_SUMS))
    for t, st, ok, wt, v in _tiles(shape, status, w, x, y):
        _counts_minmax(s, t, st, ok, wt)
        for j, c in enumerate(SUM_COLS):
            col = v[ok, j]
            fin = np.isfinite(col).all()
            s[t, c] = math.fsum(col) if fin else np.sum(col)
            absum[t, j] = math.fsum(np.abs(col)) if fin else np.inf
    return s, absum


def tile_items(shape, t, v):
    """the tile's work-item sums ``[chunks_per_tile * 8, 13]`` and the in-range mask"""
    cpt = shape.chunks_per_tile
    l0, l1 = shape.tile_range(t)
    lanes = np.zeros((cpt*CHUNK, N_SUMS))
    lanes[l0*CHUNK:l0*CHUNK + len(v)] = v
    with np.errstate(invalid='ignore'):
        items = item_tree(lanes.reshape(cpt*WARPS, ITEM, N_SUMS))
    inr = np.zeros(cpt*WARPS, bool)
    inr[l0*WARPS:l1*WARPS] = True
    return items, inr


def ordered_summary(shape, status, w, x, y):
    """the record a launch over ``shape`` returns, its 13 sums in the documented order"""
    s = identity(shape.n_tiles)
    if shape.chunk_end == shape.chunk_begin:
        return s
    for t, st, ok, wt, v in _tiles(shape, status, w, x, y):
        _counts_minmax(s, t, st, ok, wt)
        items, inr = tile_items(shape, t, v)
        with np.errstate(invalid='ignore'):
            s[t, list(SUM_COLS)] = reduce_entries(items[inr], np.ones(int(inr.sum()), bool))
    return s


def combine(parts):
    """``k_combine_wfe``: parts added (min / max taken) in part order"""
    out = np.array(parts[0], dtype=np.float64)
    for p in parts[1:]:
        with np.errstate(invalid='ignore'):
            out[:, :5] = out[:, :5] + p[:, :5]
            out[:, 7:] = out[:, 7:] + p[:, 7:]
            out[:, MIN_COL] = np.fmin(out[:, MIN_COL], p[:, MIN_COL])
            out[:, MAX_COL] = np.fmax(out[:, MAX_COL], p[:, MAX_COL])
    return out


def shuffle_tree_lanes(v):
    """lane-by-lane simulation of ``wfe_item_sums_store``: ``v`` ``[32, 13]`` lane values ->
    the 13 values the storing lanes write"""
    assert v.shape == (ITEM, N_SUMS)
    vals = np.zeros((ITEM, 16))
    vals[:, :N_SUMS] = v
    lanes = range(ITEM)
    h = lambda l, b: bool(l & b)        # noqa: E731
    a = np.zeros((ITEM, 8))
    for l in lanes:
        p = l ^ 16
        for k in range(8):
            mine = vals[l, 8 + k] if h(l, 16) else vals[l, k]
            got = vals[p, k] if h(p, 16) else vals[p, 8 + k]
            a[l, k] = mine + got
    b = np.zeros((ITEM, 4))
    for l in lanes:
        p = l ^ 8
        for k in range(4):
            b[l, k] = (a[l, 4 + k] if h(l, 8) else a[l, k]) + (a[p, k] if h(p, 8) else a[p, 4 + k])
    c = np.zeros((ITEM, 2))
    for l in lanes:
        p = l ^ 4
        for k in range(2):
            c[l, k] = (b[l, 2 + k] if h(l, 4) else b[l, k]) + (b[p, k] if h(p, 4) else b[p, 2 + k])
    e = np.zeros(ITEM)
    for l in lanes:
        p = l ^ 2
        e[l] = (c[l, 1] if h(l, 2) else c[l, 0]) + (c[p, 0] if h(p, 2) else c[p, 1])
    f = np.array([e[l] + e[l ^ 1] for l in lanes])
    out = np.full(16, np.nan)
    for l in lanes:
        if l & 1 == 0:
            idx = ((l >> 4) & 1)*8 + ((l >> 3) & 1)*4 + ((l >> 2) & 1)*2 + ((l >> 1) & 1)
            out[idx] = f[l]
    return out[:N_SUMS]
