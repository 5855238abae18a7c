"""Reference tolerance records (test helper, numpy only): what the ``[n_tiles, RT_TOL_DOUBLES]`` record
of one variant of ``rt_trace_grid_variants`` must hold, given the whole grid's per-ray ``status``,
transverse aberration ``ax``, ``ay``, ``op`` and last-segment direction ``dx``, ``dy``, ``dz``.

Columns 0-15 are ``rt_trace_grid``'s summary (``spot_sums.ordered_summary``; over the whole grid
its two regimes add in the same order); 16-21 the sums of ux, uy, ux*ux, uy*uy, ax*ux, ay*uy with
ux = dx/dz, uy = dy/dz (one IEEE division each, every product rounded once), added by the halving
tree of a work item and ``reduce_tile`` over the tile's items in item order (DESIGN.md section 4);
22-23 zero.  Only status-0 rays enter the sums."""
import numpy as np

from spot_sums import Shape, item_tree, reduce_entries, ordered_summary, CHUNK, WARPS, ITEM  # noqa: F401

WIDTH = 24
SLOPE_COLS = tuple(range(16, 22))


def slope_summands(ax, ay, dx, dy, dz, ok):
    """``[n, 6]`` summands of columns 16-21; rays outside ``ok`` hold +0.0"""
    ax, ay, dx, dy, dz = (np.asarray(v, dtype=np.float64) for v in (ax, ay, dx, dy, dz))
    with np.errstate(all='ignore'):
        ux, uy = dx/dz, dy/dz
        v = np.stack([ux, uy, ux*ux, uy*uy, ax*ux, ay*uy], axis=1)
    v[~np.asarray(ok, bool)] = 0.0
    return v


def record(shape, status, ax, ay, op, dx, dy, dz):
    """the record of one variant over the whole grid ``shape``"""
    assert shape.chunk_begin == 0 and shape.chunk_end == shape.n_chunks
    status = np.asarray(status)
    out = np.zeros((shape.n_tiles, WIDTH))
    out[:, :16] = ordered_summary(shape, status, ax, ay, op, 'items')
    v = slope_summands(ax, ay, dx, dy, dz, status == 0)
    cpt, rpt = shape.chunks_per_tile, shape.rays_per_tile
    for t in range(shape.n_tiles):
        lanes = np.zeros((cpt*CHUNK, 6))
        lanes[:rpt] = v[t*rpt:(t + 1)*rpt]
        with np.errstate(invalid='ignore'):
            items = item_tree(lanes.reshape(cpt*WARPS, ITEM, 6))
            out[t, list(SLOPE_COLS)] = reduce_entries(items, np.ones(len(items), bool))
    return out
