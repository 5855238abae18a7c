"""CPU: the spot-sum references of tests/spot_sums.py.

* ``ordered_summary`` (the library's addition order) stays within ``sum_bound`` of the correctly
  rounded ``exact_summary`` on adversarial data: magnitudes from 1e-9 to 1e3, heavy cancellation,
  signed zeros, rejected rays, all-rejected and one-ray tiles, partial items, chunks and ranges.
* Its item tree is the literal lane arithmetic of ``item_sums_store`` (xor butterfly) and of
  ``warp_record_from_regs`` (``shfl_down``), simulated lane by lane.
* Each plausible mistake of the kernel's reduction, applied to the restatement, changes the bits
  of the sums on this data, so the bit-for-bit GPU comparison (test_gpu_spot_sums.py) catches it.
* On the oracle's per-ray grid outputs, ``exact_summary``'s counts and min / max are what
  ``test_cuda_grid_matches_oracle`` computes."""
import numpy as np
import pytest

import spot_sums as S
from conftest import load_model


def synthetic(n, rng, p_rejected=0.2):
    """per-ray (status, ax, ay, op) that make floating-point sums hard"""
    mag = 10.0**rng.uniform(-9, 3, n)
    ax = mag*rng.choice([-1.0, 1.0], n)
    ay = 10.0**rng.uniform(-9, 3, n)*rng.choice([-1.0, 1.0], n)
    # heavy cancellation: every other ray is the negated neighbour plus a tiny offset
    k = np.arange(1, n, 2)
    ax[k] = -ax[k - 1]*(1 + 1e-12*rng.standard_normal(len(k)))
    ay[k] = -ay[k - 1] + 1e-9*rng.standard_normal(len(k))
    z = rng.random(n) < 0.03
    ax[z] = rng.choice([0.0, -0.0], z.sum())
    ay[rng.random(n) < 0.03] = -0.0
    op = 1e3 + 10.0**rng.uniform(-9, 1, n)*rng.choice([-1.0, 1.0], n)
    status = np.where(rng.random(n) < p_rejected, rng.integers(1, 6, n), 0).astype(np.int32)
    return status, ax, ay, op


def cases():
    """(shape, per-ray data) covering the shapes where reductions go wrong"""
    rng = np.random.default_rng(2024)
    out = []

    def add(rays_per_tile, n_tiles, c0=0, c1=None, reject_tile=None):
        sh = S.Shape(rays_per_tile, n_tiles, c0, c1)
        st, ax, ay, op = synthetic(sh.n_rays, rng)
        if reject_tile is not None:
            a = sh.first_ray(reject_tile*sh.chunks_per_tile) - sh.first_ray(c0)
            b = sh.first_ray((reject_tile + 1)*sh.chunks_per_tile) - sh.first_ray(c0)
            st[a:b] = 3
        out.append((sh, (st, ax, ay, op)))
    add(1000, 4, reject_tile=2)               # partial last chunk (232 rays) and item (8 rays)
    add(1000, 4, 1, 11)                       # range starting / ending inside tiles
    add(1000, 4, 6, 7)                        # one chunk
    add(1, 5)                                 # one ray per tile
    add(1089, 3, 2, 13)                       # 33^2: 5 chunks per tile, 65-ray last chunk
    add(600*256 + 77, 2)                      # 601 chunks per tile: threads add 2 items per part
    add(600*256 + 77, 2, 200, 1000)
    add(2100*256 + 5, 1, 3, 2101)             # more chunks per tile than record slots
    return out


CASES = cases()


def test_shapes_cover_the_edges():
    shapes = [sh for sh, _ in CASES]
    assert any(sh.rays_per_tile % S.CHUNK and sh.rays_per_tile % S.ITEM for sh in shapes)
    assert any(sh.rays_per_tile == 1 for sh in shapes)
    assert any(sh.chunks_per_tile > S.MAX_GRID for sh in shapes)
    assert any(sh.chunk_begin % sh.chunks_per_tile and sh.chunk_end % sh.chunks_per_tile for sh in shapes)
    assert any(sh.chunk_end - sh.chunk_begin == 1 for sh in shapes)
    assert any(-(-sh.chunks_per_tile*S.WARPS//S.RED_SPLIT) > S.RED_THREADS for sh in shapes)


def regimes(sh):
    return ['items'] if sh.chunks_per_tile > S.MAX_GRID else ['records', 'items']


@pytest.mark.parametrize('i', range(len(CASES)))
def test_ordered_within_bound_of_exact(i):
    sh, data = CASES[i]
    exact, absum = S.exact_summary(sh, *data)
    for rg in regimes(sh):
        got = S.ordered_summary(sh, *data, rg)
        assert (got[:, 0:5] == exact[:, 0:5]).all() and (got[:, 10:14] == exact[:, 10:14]).all()
        assert (got[:, 15] == 0).all()
        cols = list(S.SUM_COLS)
        err = np.abs(got[:, cols] - exact[:, cols])
        assert (err <= S.sum_bound(absum, S.chain_depth(sh, rg))).all(), rg
        assert (got[:, 0:5].sum() == sh.n_rays)
    st = data[0]
    if (st == 0).sum() == 0:
        assert (exact[:, 10] == np.inf).all()


def test_identities():
    sh = S.Shape(1000, 4, 5, 5)
    z = np.zeros(0)
    got = S.ordered_summary(sh, z.astype(np.int32), z, z, z, 'items')
    assert (got[:, [10, 12]] == np.inf).all() and (got[:, [11, 13]] == -np.inf).all()
    assert (got[:, list(S.SUM_COLS)].view(np.uint64) == 0).all() and (got[:, 0:5] == 0).all()
    sh, data = CASES[0]                        # tile 2: rays, none of them at the image
    got = S.ordered_summary(sh, *data, 'records')
    assert got[2, 3] == sh.rays_per_tile and got[2, 0] == 0
    assert got[2, 10] == np.inf and got[2, 13] == -np.inf
    assert (got[2, list(S.SUM_COLS)].view(np.uint64) == 0).all()


def test_exact_when_every_sum_is_exact():
    """small integers: every order gives the exact sums, so the bookkeeping (which rays, which
    tile, which column) is checked apart from the order"""
    rng = np.random.default_rng(5)
    for sh, data in CASES:
        st = data[0]
        ax, ay = rng.integers(-50, 50, len(st)).astype(float), rng.integers(-50, 50, len(st)).astype(float)
        op = rng.integers(0, 1000, len(st)).astype(float)
        exact, _ = S.exact_summary(sh, st, ax, ay, op)
        for rg in regimes(sh):
            got = S.ordered_summary(sh, st, ax, ay, op, rg)
            assert np.array_equal(got, exact), rg


def test_full_range_regimes_agree():
    """over a full range with chunks_per_tile <= 2048 records and items give the same order"""
    for sh, data in CASES:
        if sh.chunk_begin == 0 and sh.chunk_end == sh.n_chunks and sh.chunks_per_tile <= S.MAX_GRID:
            a = S.ordered_summary(sh, *data, 'records')
            b = S.ordered_summary(sh, *data, 'items')
            assert a.tobytes() == b.tobytes()


def test_partial_ranges_regimes_differ():
    sh, data = CASES[6]
    a = S.ordered_summary(sh, *data, 'records')
    b = S.ordered_summary(sh, *data, 'items')
    assert a.tobytes() != b.tobytes()


# ------------------------------------------------------------ the item tree, lane by lane
def butterfly(v):
    """item_sums_store, lane for lane: v [32, 6] -> what lanes 4g store at dst[idx]"""
    lane = np.arange(32)
    v8 = np.concatenate([v, np.zeros((32, 2))], axis=1)

    def shfl(x, m):
        return x[lane ^ m]
    h16, h8, h4 = (lane & 16) > 0, (lane & 8) > 0, (lane & 4) > 0
    sel = lambda c, a, b: np.where(c, a, b)  # noqa: E731
    a = [sel(h16, v8[:, j + 4], v8[:, j]) + shfl(sel(h16, v8[:, j], v8[:, j + 4]), 16) for j in range(4)]
    b0 = sel(h8, a[2], a[0]) + shfl(sel(h8, a[0], a[2]), 8)
    b1 = sel(h8, a[3], a[1]) + shfl(sel(h8, a[1], a[3]), 8)
    c = sel(h4, b1, b0) + shfl(sel(h4, b0, b1), 4)
    c = c + shfl(c, 2)
    c = c + shfl(c, 1)
    idx = ((lane >> 4) & 1)*4 + ((lane >> 3) & 1)*2 + ((lane >> 2) & 1)
    out = np.full(6, np.nan)
    for ln in range(0, 32, 4):
        if idx[ln] < 6:
            out[idx[ln]] = c[ln]
    return out


def shfl_down(v):
    """warp_record_from_regs / the focus records: x += shfl_down(x, off), lane 0's value"""
    x = v.copy()
    for off in (16, 8, 4, 2, 1):
        y = np.concatenate([x[off:], x[-off:]])          # lanes past 31 read their own value
        x = x + y
    return x[0]


def test_item_tree_is_the_lane_arithmetic():
    rng = np.random.default_rng(8)
    for _ in range(300):
        st, ax, ay, op = synthetic(32, rng)
        sh = S.Shape(32, 1)
        ok = st == 0
        six = np.stack([ax, ay, ax*ax, ay*ay, ax*ay, op], axis=1)
        six[~ok] = 0.0
        want = S.item_tree(six[None])[0]
        assert want.tobytes() == butterfly(six).tobytes()
        assert want.tobytes() == shfl_down(six).tobytes()
        got = S.ordered_summary(sh, st, ax, ay, op, 'records')
        assert got[0, list(S.SUM_COLS)].tobytes() == want.tobytes()


# ------------------------------------------------------------ mutation sensitivity
def drop_last_item(orig):
    def f(shape, t, ok, six):
        items, inr = orig(shape, t, ok, six)
        k = np.nonzero(inr)[0]
        if len(k):
            items = items.copy()
            items[k[-1]] = 0.0
        return items, inr
    return f


def count_item_twice(orig):
    def f(shape, t, ok, six):
        items, inr = orig(shape, t, ok, six)
        k = np.nonzero(inr)[0]
        if len(k):
            j = k[len(k)//2]
            items = np.insert(items, j, items[j], axis=0)
            inr = np.insert(inr, j, True)
        return items, inr
    return f


def no_range_clamp(orig):
    def f(shape, t, ok, six):
        items, inr = orig(shape, t, ok, six)
        return items, np.ones_like(inr)
    return f


def pair_8_before_16(orig):
    def f(v):
        order = [8, 16, 4, 2, 1]
        idx = np.arange(32)
        for off in order:
            lo = idx[(idx & off) == 0]
            v2 = v[..., lo, :] + v[..., lo + off, :]
            v = np.zeros(v.shape[:-2] + (32,) + v.shape[-1:])
            v[..., lo, :] = v2
        return v[..., 0, :]
    return f


def swap_columns(orig):
    def f(v):
        r = orig(v)
        return r[..., [1, 0, 2, 3, 4, 5]]
    return f


def reduce_variant(e, valid, shift=0, tree=False):
    """reduce_tile's order written out again, with two of its decisions open: the boundary
    between parts 0 and 1 moved by ``shift``; the 16 partials added as a tree"""
    n, k = e.shape
    e = np.where(valid[:, None], e, 0.0)
    per = -(-n//S.RED_SPLIT)
    bounds = [min(p*per, n) for p in range(S.RED_SPLIT + 1)]
    bounds[1] = min(max(bounds[1] + shift, 0), n)
    parts = []
    for p in range(S.RED_SPLIT):
        blk = e[bounds[p]:max(bounds[p + 1], bounds[p])]
        x = np.zeros((S.RED_THREADS, k))
        for r0 in range(0, len(blk), S.RED_THREADS):
            row = np.zeros((S.RED_THREADS, k))
            row[:len(blk) - r0] = blk[r0:r0 + S.RED_THREADS]
            x = x + row
        off = S.RED_THREADS//2
        while off >= 1:
            x = np.concatenate([x[:off] + x[off:2*off], x[2*off:]])
            off //= 2
        parts.append(x[0])
    if tree:
        while len(parts) > 1:
            parts = [parts[i] + parts[i + 1] for i in range(0, len(parts), 2)]
        return parts[0]
    v = parts[0]
    for p in parts[1:]:
        v = v + p
    return v


def shift_part_boundary(orig):
    return lambda e, valid: reduce_variant(e, valid, shift=1)


def partials_as_tree(orig):
    return lambda e, valid: reduce_variant(e, valid, tree=True)


MUTATIONS = [('tile_items', drop_last_item), ('tile_items', count_item_twice), ('item_tree', pair_8_before_16),
             ('reduce_entries', shift_part_boundary), ('reduce_entries', partials_as_tree),
             ('item_tree', swap_columns), ('tile_items', no_range_clamp)]


def sums_of_all_cases(rg_of=lambda sh: 'items'):
    out = []
    for sh, data in CASES:
        out.append(S.ordered_summary(sh, *data, rg_of(sh))[:, list(S.SUM_COLS)])
    return np.concatenate(out).tobytes()


@pytest.mark.parametrize('target,mutation', MUTATIONS, ids=[m.__name__ for _, m in MUTATIONS])
def test_mutation_changes_the_bits(monkeypatch, target, mutation):
    base = sums_of_all_cases()
    monkeypatch.setattr(S, target, mutation(getattr(S, target)))
    assert sums_of_all_cases() != base


def test_reduce_variant_unmutated_is_reduce_entries():
    """the harness of the two reduce_tile mutations is the restatement itself when not mutated"""
    rng = np.random.default_rng(1)
    for n in (1, 15, 17, 300, 4808, 18432):
        e = rng.standard_normal((n, 6))*10.0**rng.uniform(-9, 3, (n, 1))
        valid = rng.random(n) < 0.9
        assert reduce_variant(e, valid).tobytes() == S.reduce_entries(e, valid).tobytes()


def test_combine_in_reverse_changes_the_bits():
    sh, data = CASES[5]
    cuts = [0, 300, 301, 900, sh.n_chunks]
    parts = []
    base = sh.first_ray(0)
    for a, b in zip(cuts[:-1], cuts[1:]):
        sub = sh.sub(a, b)
        sl = slice(sh.first_ray(a) - base, sh.first_ray(b) - base)
        parts.append(S.ordered_summary(sub, *(v[sl] for v in data), 'items'))
    fwd, rev = S.combine(parts), S.combine(parts[::-1])
    assert fwd[:, list(S.SUM_COLS)].tobytes() != rev[:, list(S.SUM_COLS)].tobytes()
    assert (fwd[:, 0:5] == rev[:, 0:5]).all() and (fwd[:, 10:14] == rev[:, 10:14]).all()
    exact, absum = S.exact_summary(sh, *data)
    d = S.chain_depth(sh, 'items', pieces=len(parts))
    assert (np.abs(fwd[:, list(S.SUM_COLS)] - exact[:, list(S.SUM_COLS)]) <= S.sum_bound(absum, d)).all()


# ------------------------------------------------------------ oracle grids
@pytest.mark.parametrize('name,num', [('singlet', 7), ('dblgauss', 24), ('exotic', 16),
                                      ('diffractive_wild', 24)])
def test_exact_counts_and_extrema_on_oracle_grids(oracle, name, num):
    """what test_cuda_grid_matches_oracle computes per tile from the oracle's grid trace"""
    from rayoptics_b200 import _abi, engine as E, table as T
    opm = load_model(name)
    descs, n_by_wvl, wvls = T.describe_model(opm.seq_model)
    spec = E.grid_spec_for_model(opm, num)
    opts = _abi.make_opts(first_surf=1, last_surf=len(descs) - 2, check_apertures=True)
    g = oracle.trace_grid(spec.c_spec(), descs, n_by_wvl, 0, spec.n_rays, opts, n_threads=8, wvls=wvls)
    st, (ax, ay), op = g['status'], g['abr'], g['op']
    sh = S.Shape(spec.rays_per_tile, spec.n_tiles)
    exact, _ = S.exact_summary(sh, st, ax, ay, op)
    per = spec.rays_per_tile
    for t in range(spec.n_tiles):
        sl = slice(t*per, (t + 1)*per)
        s, ok = st[sl], st[sl] == 0
        assert exact[t, 0] == ok.sum() and exact[t, 1] == (s == 1).sum()
        assert exact[t, 2] == (s == 2).sum() and exact[t, 3] == (s == 3).sum()
        assert exact[t, 4] == (s > 3).sum()
        x, y = ax[sl][ok], ay[sl][ok]
        if ok.any() and not np.isnan(x).all():
            assert exact[t, 10] == np.nanmin(x) and exact[t, 11] == np.nanmax(x)
            assert exact[t, 12] == np.nanmin(y) and exact[t, 13] == np.nanmax(y)
        if np.isnan(x).any():                   # NaN aberrations of status-0 rays: sums NaN
            assert np.isnan(exact[t, [5, 7, 9]]).all()
    assert exact[:, 0:5].sum() == spec.n_rays
    if name == 'diffractive_wild':
        assert exact[:, 4].sum() > 0 and np.isnan(exact[:, 5]).any()
