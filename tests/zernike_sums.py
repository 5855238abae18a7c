"""Reference Zernike moments (test helper, numpy only): what the ``[n_tiles, RT_ZERN_DOUBLES]``
record of ``rt_grid_zernike`` must hold, given the launch's per-ray ``status``, OPD ``W`` and the
rays' relative pupil coordinates ``x``, ``y``.

Column layout (include/b200rt.h): 0-4 ray counts by status class (0, 1, 2, 3, anything else) over
every ray, 5 n_used, 6 / 7 min / max W over the used rays (fmin / fmax), 8 zero, 9 + j(j+1)/2 + i
(i <= j <= J) the sum of a_i*a_j over the used rays with a = [W, Z_1 ... Z_J], later columns zero.
A ray is used when its status is 0 and x*x + y*y <= 1.

The sums in the documented order (DESIGN.md section 4):

1. a per ray: ``engine.zernike_terms``, the numpy restatement of csrc/rt_zernike.cuh; +0.0 in every
   column of a ray that is not used.  Each product a_i*a_j is rounded once (``-fmad=false``).
2. a chunk (256 consecutive rays of one tile): every entry added one after another in ray order,
   starting from +0.0.  ``np.cumsum`` along the ray axis after a leading +0.0 row is exactly that
   chain; ``np.sum`` would add pairwise.  Rays past the end of a tile's last chunk add +0.0,
   which leaves a chain that started at +0.0 unchanged.
3. a tile: its chunk sums inside the launch's chunk range, added in chunk order from +0.0
   (``k_reduce_zernike``), ``np.cumsum`` again.
4. ``combine``: partial records (chunk ranges, shards) added in part order (``k_combine_zernike``).
"""
import math

import numpy as np

from spot_sums import CHUNK, U, Shape  # noqa: F401
from rayoptics_b200 import engine as E

WIDTH = 752
HEAD = 9
MIN_COL, MAX_COL = 6, 7
COUNT_COLS = (0, 1, 2, 3, 4, 5)


def triangle(n_terms):
    """(i, j) of the packed Gram block in column order: column j-major, i <= j"""
    return [(i, j) for j in range(n_terms + 1) for i in range(j + 1)]


def sum_cols(n_terms):
    return list(range(HEAD, HEAD + (n_terms + 1)*(n_terms + 2)//2))


def used_mask(status, x, y):
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    return (np.asarray(status) == 0) & (x*x + y*y <= 1.0)


def augmented(status, w, x, y, n_terms, used=None):
    """``[n, n_terms + 1]`` rows [W, Z_1 ...]; +0.0 for rays that are not used"""
    if used is None:
        used = used_mask(status, x, y)
    a = np.concatenate([np.asarray(w, dtype=np.float64)[:, None], E.zernike_terms(x, y, n_terms)], axis=1)
    a[~used] = 0.0
    return a


def products(a, n_terms, tri=None):
    i, j = np.array(tri or triangle(n_terms)).T
    with np.errstate(all='ignore'):
        return a[..., i]*a[..., j]


def chained(v, axis):
    """the sum along ``axis`` added one after another from +0.0"""
    v = np.moveaxis(v, axis, 0)
    with np.errstate(all='ignore'):
        return np.cumsum(np.concatenate([np.zeros((1,) + v.shape[1:]), v]), axis=0)[-1]


def identity(n_tiles):
    s = np.zeros((n_tiles, WIDTH))
    s[:, MIN_COL] = np.inf
    s[:, MAX_COL] = -np.inf
    return s


def _tiles(shape, status, w, x, y):
    """per tile of the launch: (tile, first local chunk, its rays' slice of the launch's arrays)"""
    base = shape.first_ray(shape.chunk_begin)
    for t in range(shape.n_tiles):
        l0, l1 = shape.tile_range(t)
        if l1 == l0:
            continue
        a = shape.first_ray(t*shape.chunks_per_tile + l0) - base
        b = shape.first_ray(t*shape.chunks_per_tile + l1) - base
        yield t, l0, l1, slice(a, b)


def _head(s, t, st, used, w):
    cls = np.where((st >= 0) & (st <= 3), st, 4)
    s[t, 0:5] = np.bincount(cls, minlength=5)[:5]
    s[t, 5] = used.sum()
    s[t, MIN_COL] = np.fmin.reduce(w[used], initial=np.inf)
    s[t, MAX_COL] = np.fmax.reduce(w[used], initial=-np.inf)


def chunk_sums(a, n_chunks, n_terms, reverse_rays=False, tri=None, batch=16):
    """``[n_chunks, n_entries]`` per-chunk chains over rows ``a`` (the chunks' rays in order; the last
    chunk may be short)"""
    n_e = len(tri or triangle(n_terms))
    out = np.empty((n_chunks, n_e))
    pad = np.zeros((n_chunks*CHUNK, a.shape[1]))
    pad[:len(a)] = a
    pad = pad.reshape(n_chunks, CHUNK, a.shape[1])
    if reverse_rays:
        pad = pad[:, ::-1]
    for c in range(0, n_chunks, batch):
        out[c:c + batch] = chained(products(pad[c:c + batch], n_terms, tri), axis=1)
    return out


def ordered_summary(shape, status, w, x, y, n_terms, reverse_rays=False, drop_chunk=None, transposed=False,
                    strict=False):
    """the record a launch over ``shape`` returns, its sums in the documented order.  The keyword
    arguments make plausible mistakes on purpose (tests that they change the bits): rays added in
    reverse order, one chunk dropped, the triangle packed row by row, ``<`` for ``<=``."""
    status = np.asarray(status)
    w, x, y = (np.asarray(v, dtype=np.float64) for v in (w, x, y))
    assert len(status) == shape.n_rays == len(w) == len(x) == len(y)
    s = identity(shape.n_tiles)
    if shape.chunk_end == shape.chunk_begin:
        return s
    used = used_mask(status, x, y) if not strict else (status == 0) & (x*x + y*y < 1.0)
    tri = triangle(n_terms)
    if transposed:      # row-major packing of the upper triangle
        tri = [(i, j) for i in range(n_terms + 1) for j in range(i, n_terms + 1)]
    cols = sum_cols(n_terms)
    for t, l0, l1, sl in _tiles(shape, status, w, x, y):
        _head(s, t, status[sl], used[sl], w[sl])
        s[t, 8] = 0.0
        a = augmented(status[sl], w[sl], x[sl], y[sl], n_terms, used[sl])
        per_chunk = chunk_sums(a, l1 - l0, n_terms, reverse_rays, tri)
        if drop_chunk is not None:
            per_chunk = np.delete(per_chunk, drop_chunk % len(per_chunk), axis=0)
        s[t, cols] = chained(per_chunk, axis=0)
    return s


def exact_summary(shape, status, w, x, y, n_terms):
    """counts, fmin / fmax and correctly rounded sums; also ``[n_tiles, n_entries]`` sums of
    |product|"""
    status = np.asarray(status)
    w, x, y = (np.asarray(v, dtype=np.float64) for v in (w, x, y))
    s = identity(shape.n_tiles)
    cols = sum_cols(n_terms)
    absum = np.zeros((shape.n_tiles, len(cols)))
    used = used_mask(status, x, y)
    for t, l0, l1, sl in _tiles(shape, status, w, x, y):
        _head(s, t, status[sl], used[sl], w[sl])
        p = products(augmented(status[sl], w[sl], x[sl], y[sl], n_terms, used[sl])[used[sl]], n_terms)
        for e, c in enumerate(cols):
            col = p[:, e]
            fin = np.isfinite(col).all()
            s[t, c] = math.fsum(col) if fin else np.sum(col)
            absum[t, e] = math.fsum(np.abs(col)) if fin else np.inf
    return s, absum


def chain_depth(shape):
    """additions on the way to one tile entry: a chunk's 256 rays, the tile's chunks, and the
    rounding of the correctly rounded reference"""
    return CHUNK + shape.chunks_per_tile + 1


def sum_bound(absum, depth):
    """gamma_d * sum |x_i|"""
    return depth*U/(1.0 - depth*U)*absum


def combine(parts):
    """``k_combine_zernike``: parts added (min / max taken) in part order"""
    out = np.array(parts[0], dtype=np.float64)
    for p in parts[1:]:
        with np.errstate(invalid='ignore'):
            out[:, :6] = out[:, :6] + p[:, :6]
            out[:, 8:] = out[:, 8:] + p[:, 8:]
            out[:, MIN_COL] = np.fmin(out[:, MIN_COL], p[:, MIN_COL])
            out[:, MAX_COL] = np.fmax(out[:, MAX_COL], p[:, MAX_COL])
    return out


def grid_pupil_xy(spec, shape):
    """per-ray (x, y) of the launch's rays: the grid's pupil tables as the kernel reads them (a
    product grid without vignetting)"""
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


def same_bits(got, want, n_terms, what=''):
    """counts and sums bit for bit (NaN: both NaN), min / max by ==, every other column 0"""
    cols = list(COUNT_COLS) + [8] + sum_cols(n_terms)
    g, w = got[:, cols], want[:, cols]
    assert (np.isnan(g) == np.isnan(w)).all(), what
    m = ~np.isnan(w)
    assert g[m].view(np.uint64).tolist() == w[m].view(np.uint64).tolist(), what
    assert (got[:, [MIN_COL, MAX_COL]] == want[:, [MIN_COL, MAX_COL]]).all(), what
    rest = np.ones(WIDTH, bool)
    rest[cols + [MIN_COL, MAX_COL]] = False
    assert (got[:, rest] == 0.0).all() and not np.signbit(got[:, rest]).any(), what
