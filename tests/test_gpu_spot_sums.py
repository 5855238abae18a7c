"""GPU: the `[n_tiles, 16]` spot sums of grid launches against references of the same operation.

Every launch also returns its per-ray status, aberrations and op, which are checked against the
oracle (bit for bit; tolerance parity for phase elements).  From those per-ray values
`tests/spot_sums.py` builds the summary the launch must return:

* counts (columns 0-4) exactly, column 15 zero;
* min / max (10-13) by == against fmin / fmax (either signed zero may come back);
* the six sums (5-9, 14) bit for bit against ``ordered_summary`` (the addition order the library
  documents) and within ``sum_bound`` of the correctly rounded sums.

The regime of each launch (per-chunk records or work items) is derived from its shape and the
device's SM count and occupancy limits, and asserted to be the one the case is meant to test.
The static schedule's per-CTA records depend on the CTA count the launch picked: bound only.
``spot_statistics`` (centroid, RMS radius) of every checked tile is compared with a two-pass
reference within a tolerance that follows from the cancellation of the one-pass formula."""
import numpy as np
import pytest
import torch

import spot_sums as S
from conftest import load_model
from rayoptics_b200 import _abi, engine as E, table as T, waveabr as W

pytestmark = pytest.mark.gpu

RT_ACC_BYTES = 15*256*8          # per-thread accumulators of every summary launch (shared memory)
WORST = {'kappa': 0.0, 'where': None, 'tiles': 0}


def sm_limits():
    """SM count and an upper bound of the 256-thread summary CTAs resident per SM"""
    p = torch.cuda.get_device_properties(0)
    by_threads = p.max_threads_per_multi_processor//S.CHUNK
    by_smem = p.shared_memory_per_multiprocessor//(RT_ACC_BYTES + 1024)     # + 1 KB reserved per CTA
    return p.multi_processor_count, min(by_threads, by_smem)


def regime_of(shape):
    return S.regime(shape, *sm_limits())


def np_(t):
    return t.detach().cpu().numpy()


_TABLES = {}


def table(name, fresh=False):
    """the model's table, shared by the tests; ``fresh``: a new one (created under the caller's
    environment, e.g. B200RT_STATIC / B200RT_NO_LEAN)"""
    if fresh:
        return T.SurfaceTable.from_model(load_model(name).seq_model, device=0)
    if name not in _TABLES:
        opm = load_model(name)
        _TABLES[name] = (opm, T.SurfaceTable.from_model(opm.seq_model, device=0))
    return _TABLES[name][1]


def model(name):
    table(name)
    return _TABLES[name][0]


def same_bits(a, b):
    """equal as bit patterns, NaNs by NaN-ness"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nan = np.isnan(a)
    return (nan == np.isnan(b)).all() and (a[~nan].view(np.uint64) == b[~nan].view(np.uint64)).all()


def check_rays(oracle, tab, grid, c0, c1, got, chunks=None, tol=0.0):
    """per-ray outputs of chunks [c0, c1) (or of the listed chunks) against the oracle"""
    opts = _abi.make_opts(first_surf=1, last_surf=tab.n_ifc - 2, check_apertures=True)
    base = grid.first_ray_of_chunk(c0)
    spans = [(c0, c1)] if chunks is None else [(int(c), int(c) + 1) for c in chunks]
    for ca, cb in spans:
        a, b = grid.first_ray_of_chunk(ca), grid.first_ray_of_chunk(cb)
        if a == b:
            continue
        ref = oracle.trace_grid(grid.c_spec(), tab.descs, tab.n_by_wvl, a, b, opts, n_threads=8,
                                wvls=tab.wvls)
        ref['p'], ref['d'] = ref['last'][0:3], ref['last'][3:6]
        sl = slice(a - base, b - base)
        for key, v in got.items():
            g, r = v[..., sl], ref[key]
            if key == 'status' or tol == 0.0:
                assert same_bits(g, r) if key != 'status' else (g == r).all(), (key, ca, cb)
            else:                                # phase elements: rays at the image, op 1e3 x tol
                ok = ref['status'] == 0
                g, r = g[..., ok], r[..., ok]
                assert (np.isnan(g) == np.isnan(r)).all(), key
                np.testing.assert_allclose(g, r, rtol=0, atol=tol*(1e3 if key == 'op' else 1), err_msg=key)


def check_summary(summ, shape, status, ax, ay, op, regime, pieces=1, static=False, what=''):
    """a launch's summary (numpy [n_tiles, 16]) against both references of its per-ray values;
    ``regime``: 'records' / 'items' (bit for bit) or None (bound only)"""
    exact, absum = S.exact_summary(shape, status, ax, ay, op)
    assert (summ[:, 0:5] == exact[:, 0:5]).all(), what
    assert (summ[:, 15].view(np.uint64) == 0).all(), what
    assert (summ[:, 10:14] == exact[:, 10:14]).all(), what
    cols = list(S.SUM_COLS)
    if regime is not None:
        want = S.ordered_summary(shape, status, ax, ay, op, regime)
        assert same_bits(summ[:, cols], want[:, cols]), (what, regime)
    d = S.chain_depth(shape, regime or 'records', pieces, static)
    got, ex = summ[:, cols], exact[:, cols]
    nan = np.isnan(ex)
    assert (np.isnan(got) == nan).all(), what
    with np.errstate(invalid='ignore'):
        err = np.abs(got - ex)
    assert (err[~nan] <= S.sum_bound(absum, d)[~nan]).all(), (what, d)
    check_statistics(summ, shape, status, ax, ay, d, what)


def check_statistics(summ, shape, status, ax, ay, d, what):
    """spot_statistics of the summary against a two-pass reference.  Centroid: the error of a sum
    over n, (d + 3) u sum|x| / n.  Variance (squared RMS radius) by the one-pass formula
    (sum x^2 + sum y^2) / n - (cx^2 + cy^2): the sums carry gamma_d relative errors, the centroid
    terms twice that, so |var - var_ref| <= (3 d + 10) u a with a = (sum x^2 + sum y^2) / n,
    i.e. a relative error of (3 d + 10) u kappa, kappa = a / var."""
    st = E.spot_statistics(summ)
    rms = st['rms_radius']
    base = shape.first_ray(shape.chunk_begin)
    status = np.asarray(status)
    for t in range(shape.n_tiles):
        a = max(shape.first_ray(t*shape.chunks_per_tile), base) - base
        b = min(shape.first_ray((t + 1)*shape.chunks_per_tile), shape.first_ray(shape.chunk_end)) - base
        if b <= a:
            continue
        ok = status[a:b] == 0
        x, y = np.asarray(ax[a:b])[ok], np.asarray(ay[a:b])[ok]
        if len(x) == 0 or not (np.isfinite(x).all() and np.isfinite(y).all()):
            continue
        cx, cy, var, aa = S.spot_reference(x, y)
        n = len(x)
        assert abs(st['centroid_x'][t] - cx) <= (d + 3)*S.U*np.abs(x).sum()/n, (what, t)
        assert abs(st['centroid_y'][t] - cy) <= (d + 3)*S.U*np.abs(y).sum()/n, (what, t)
        assert abs(rms[t]**2 - var) <= (3*d + 10)*S.U*aa*(1 + 4*S.U), (what, t)
        WORST['tiles'] += 1
        if var > 0 and aa/var > WORST['kappa']:
            WORST['kappa'], WORST['where'] = aa/var, (what, t)


def trace_and_check(oracle, tab, grid, c0, c1, want_regime, outputs=('status', 'abr', 'op'),
                    full=False, sample=None, tol=0.0, static=False, what=''):
    """one rt_trace_grid launch with per-ray outputs and summary; both checked"""
    shape = S.Shape.of(grid, c0, c1)
    rg = regime_of(shape)
    assert rg == want_regime, (what, c0, c1, rg)
    r = E.trace_grid(tab, grid, c0, c1, outputs=outputs, full=full)
    torch.cuda.synchronize()
    got = {k: np_(getattr(r, k)) for k in outputs if k in ('status', 'abr', 'op', 'p', 'd')}
    if c1 > c0:
        chunks = None if sample is None else np.random.default_rng(5).integers(c0, c1, sample)
        check_rays(oracle, tab, grid, c0, c1, got, chunks, tol)
    summ = np_(r.summary)
    if c1 == c0:
        assert same_bits(summ, S.identity_summary(grid.n_tiles)), what
        return summ, got
    check_summary(summ, shape, got['status'], got['abr'][0], got['abr'][1], got['op'],
                  None if static and rg == 'items' else rg, static=static, what=what)
    return summ, got


# ---------------------------------------------------------------- kernel instances x ranges
RANGES_48 = [  # num = 48: 9 tiles of 9 chunks
    (lambda n: (0, n), 'records'),
    (lambda n: (3, n - 5), 'records'),           # starts and ends inside a tile
    (lambda n: (40, 41), 'items'),               # one chunk
    (lambda n: (10, 15), 'items'),               # shorter than a tile's chunks, inside one tile
    (lambda n: (4, 4), 'empty'),                 # no chunks: identities
]


@pytest.mark.parametrize('name', ['dblgauss', 'cellphone', 'evenasph', 'threemir', 'exotic', 'relay_na'])
def test_kernel_instances_over_chunk_ranges(oracle, name):
    """lean (dblgauss), lean POLY (cellphone, evenasph), general staged (threemir, exotic),
    angular pupil (relay_na)"""
    tab = table(name)
    grid = E.grid_for_model(model(name), tab, 48)
    assert grid.chunks_per_tile == 9
    for rng, want in RANGES_48:
        c0, c1 = rng(grid.n_chunks)
        summ, got = trace_and_check(oracle, tab, grid, c0, c1, want, what=(name, c0, c1))
        if c1 - c0 == grid.n_chunks:
            assert summ[:, 0].sum() > 0 and summ[:, 0:5].sum() == grid.n_rays
    grid.close()


@pytest.mark.parametrize('kind', [1, 2])
@pytest.mark.parametrize('name', ['dblgauss', 'threemir'])
def test_output_kinds_with_summary(oracle, name, kind):
    tab = table(name)
    grid = E.grid_for_model(model(name), tab, 24)          # 3 chunks per tile
    outs = ('status', 'abr', 'op') + (('nrml', 'dst') if kind == 1 else ())
    for c0, c1, want in ((0, grid.n_chunks, 'records'), (4, 6, 'items')):
        trace_and_check(oracle, tab, grid, c0, c1, want, outputs=outs, full=kind == 2, what=(name, kind))
    grid.close()


@pytest.mark.parametrize('general', [False, True])
def test_opd_with_summary(oracle, monkeypatch, general):
    opm = model('dblgauss')
    if general:
        monkeypatch.setenv('B200RT_NO_LEAN', '1')
        tab = table('dblgauss', fresh=True)
        monkeypatch.delenv('B200RT_NO_LEAN')
    else:
        tab = table('dblgauss')
    osp, sm = opm.optical_spec, opm.seq_model
    fields, wvls = list(osp.fov.fields), list(sm.wvlns)
    wave, ref_img, _ = W.setup_tiles(opm, tab, fields, wvls, 0.0)
    recs, eprad, z_pupil = osp.grid_fields(fields)
    xs = E.accumulated_steps(-1.0, 1.0, 24)
    grid = E.PupilGrid(recs, [tab.wvl_index(w) for w in wvls], xs, xs, eprad, z_pupil,
                       ref_img=ref_img, flip_z_dir=sm.z_dir[0], wave=wave, device=0)
    for c0, c1, want in ((0, grid.n_chunks, 'records'), (4, 6, 'items')):
        summ, got = trace_and_check(oracle, tab, grid, c0, c1, want, outputs=('status', 'abr', 'op', 'opd'),
                                    what=('opd', general))
    grid.close()


# ---------------------------------------------------------------- regimes at size
def test_work_items_at_512(oracle):
    """the bench / spot_diagram shape: 9 tiles of 512^2 rays, 1024 chunks per tile"""
    tab = table('dblgauss')
    grid = E.grid_for_model(model('dblgauss'), tab, 512)
    n = grid.n_chunks
    for c0, c1 in ((0, n), (500, n - 700)):
        trace_and_check(oracle, tab, grid, c0, c1, 'items', sample=12, what=(512, c0, c1))
    grid.close()


def test_more_chunks_per_tile_than_record_slots(oracle):
    """768^2 rays of one field and wavelength: 2304 chunks per tile > RT_MAX_GRID"""
    opm = model('dblgauss')
    tab = table('dblgauss')
    grid = E.grid_for_model(opm, tab, 768, fields=[opm.optical_spec.fov.fields[-1]],
                            wvls=[opm.seq_model.central_wavelength()])
    assert grid.n_tiles == 1 and grid.chunks_per_tile == 2304
    for c0, c1 in ((0, grid.n_chunks), (300, 2000)):
        trace_and_check(oracle, tab, grid, c0, c1, 'items', sample=8, what=(768, c0, c1))
    grid.close()


# ---------------------------------------------------------------- shapes
def test_one_ray_per_tile(oracle):
    tab = table('dblgauss')
    grid = E.grid_for_model(model('dblgauss'), tab, 1)
    assert grid.rays_per_tile == 1
    trace_and_check(oracle, tab, grid, 0, grid.n_chunks, 'records', what='num=1')
    trace_and_check(oracle, tab, grid, 2, 7, 'records', what='num=1')
    grid.close()


def test_partial_last_chunk_and_item(oracle):
    """33^2 = 1089 rays per tile: 5 chunks, the last holds 65 rays (2 items + 1 ray)"""
    tab = table('evenasph')
    grid = E.grid_for_model(model('evenasph'), tab, 33)
    assert grid.chunks_per_tile == 5
    for c0, c1, want in ((0, grid.n_chunks, 'records'), (7, 11, 'items'), (9, 10, 'items'),
                         (4, grid.n_chunks - 3, 'records')):
        trace_and_check(oracle, tab, grid, c0, c1, want, what=(33, c0, c1))
    grid.close()


def paired_grid(opm, tab, px, py):
    osp, sm = opm.optical_spec, opm.seq_model
    fields = list(osp.fov.fields)
    recs, eprad, z_pupil = osp.grid_fields(fields)
    g0 = E.grid_for_model(opm, tab, 1)
    ref = g0.ref_img
    g0.close()
    return E.PupilGrid(recs, [tab.wvl_index(w) for w in sm.wvlns], px, py, eprad, z_pupil, ref_img=ref,
                       flip_z_dir=sm.z_dir[0], paired=True, device=0)


def test_paired_list_not_a_multiple_of_32(oracle):
    opm, tab = model('dblgauss'), table('dblgauss')
    rng = np.random.default_rng(17)
    m = 1000
    px, py = rng.uniform(-1.1, 1.1, m), rng.uniform(-1.1, 1.1, m)
    py[:9] = [0.0, -0.0, 0.0, 1.0, -1.0, 0.5, -0.5, 0.0, 0.0]
    px[:9] = [0.0, 0.0, -0.0, 0.0, 0.0, 0.5, -0.5, 1.0, -1.0]
    grid = paired_grid(opm, tab, px, py)
    assert grid.rays_per_tile == m and grid.chunks_per_tile == 4
    for c0, c1, want in ((0, grid.n_chunks, 'records'), (5, 7, 'items'), (3, grid.n_chunks - 2, 'records')):
        trace_and_check(oracle, tab, grid, c0, c1, want, what=('paired', c0, c1))
    grid.close()


def test_tiles_where_no_ray_arrives(oracle):
    opm, tab = model('dblgauss'), table('dblgauss')
    grid = E.grid_for_model(opm, tab, 24, pupil_range=(3.0, 4.0))
    for c0, c1, want in ((0, grid.n_chunks, 'records'), (4, 6, 'items')):
        summ, _ = trace_and_check(oracle, tab, grid, c0, c1, want, what=('none', c0, c1))
        hit = summ[:, 0:5].sum(axis=1) > 0
        assert hit.any() and (summ[hit, 0] == 0).all()
        assert (summ[:, [10, 12]] == np.inf).all() and (summ[:, [11, 13]] == -np.inf).all()
        assert (summ[:, list(S.SUM_COLS)].view(np.uint64) == 0).all()
    grid.close()


def test_status_4_and_nan_aberrations(oracle):
    """diffractive_wild: evanescent rays (status 4) go to column 4; grating rays with NaN directions
    keep status 0, so their NaN aberrations make the tile's sums NaN while fmin / fmax skip them"""
    opm, tab = model('diffractive_wild'), table('diffractive_wild')
    grid = E.grid_for_model(opm, tab, 24)
    for c0, c1, want in ((0, grid.n_chunks, 'records'), (4, 6, 'items')):
        summ, got = trace_and_check(oracle, tab, grid, c0, c1, want, tol=1e-11, what=('wild', c0, c1))
        if c1 - c0 == grid.n_chunks:
            assert summ[:, 4].sum() > 0
            st, abr = got['status'], got['abr']
            nan_ok = (st == 0) & np.isnan(abr[0])
            assert nan_ok.any()
            tiles = np.unique(np.nonzero(nan_ok)[0]//grid.rays_per_tile)
            assert np.isnan(summ[tiles][:, [5, 7, 9]]).all()
            assert np.isfinite(summ[tiles][:, 10:14]).all()
    grid.close()


# ---------------------------------------------------------------- static schedule
def test_static_schedule(oracle, monkeypatch):
    """B200RT_STATIC=1: per-chunk records bit for bit; per-CTA records (per-thread shared-memory
    accumulators, acc_add / acc_flush) within the bound of a chain as long as the tile's chunks"""
    monkeypatch.setenv('B200RT_STATIC', '1')
    tabs = {name: table(name, fresh=True) for name in ('dblgauss', 'threemir')}
    monkeypatch.delenv('B200RT_STATIC')
    for name, tab in tabs.items():
        grid = E.grid_for_model(model(name), tab, 48)
        for rng, want in RANGES_48:
            c0, c1 = rng(grid.n_chunks)
            trace_and_check(oracle, tab, grid, c0, c1, want, static=True, what=('static', name, c0, c1))
        grid.close()
    tab = tabs['dblgauss']
    grid = E.grid_for_model(model('dblgauss'), tab, 512)
    trace_and_check(oracle, tab, grid, 0, grid.n_chunks, 'items', sample=6, static=True, what='static 512')
    grid.close()


# ---------------------------------------------------------------- entry points
def piece_ranges(c0, c1, n):
    n = max(1, min(n, c1 - c0))
    return [(c0 + (c1 - c0)*i//n, c0 + (c1 - c0)*(i + 1)//n) for i in range(n)]


@pytest.mark.parametrize('num,rng,pieces', [(48, None, 1), (48, None, 2), (48, None, 8), (48, (3, 60), 8),
                                            (512, None, 8)])
def test_trace_grid_to_host(oracle, num, rng, pieces):
    """rt_trace_grid_to_host: each piece is a launch of its own regime, the pieces combined in order"""
    tab = table('dblgauss')
    grid = E.grid_for_model(model('dblgauss'), tab, num)
    c0, c1 = rng if rng is not None else (0, grid.n_chunks)
    n = grid.rays_in_chunks(c0, c1)
    ref = E.trace_grid(tab, grid, c0, c1, outputs=('status', 'abr', 'op'), summary=False)
    h = torch.empty((2, n), dtype=torch.float64).pin_memory()
    summ, _ = E.trace_grid_to_host(tab, grid, h, c0, c1, pieces=pieces)
    torch.cuda.synchronize()
    st, abr, op = np_(ref.status), np_(ref.abr), np_(ref.op)
    hs, _ = E.decode_nan_status(h.numpy())
    assert (hs == st).all() and same_bits(h.numpy()[:, st == 0], abr[:, st == 0])
    check_rays(oracle, tab, grid, c0, c1, {'status': st, 'abr': abr, 'op': op},
               chunks=None if num < 100 else np.random.default_rng(9).integers(c0, c1, 6))
    parts = []
    base = grid.first_ray_of_chunk(c0)
    for a, b in piece_ranges(c0, c1, pieces):
        sh = S.Shape.of(grid, a, b)
        rg = regime_of(sh)
        assert rg is not None, (a, b)
        sl = slice(grid.first_ray_of_chunk(a) - base, grid.first_ray_of_chunk(b) - base)
        parts.append(S.ordered_summary(sh, st[sl], abr[0, sl], abr[1, sl], op[sl], rg))
    if num == 48 and rng is not None:
        assert {regime_of(S.Shape.of(grid, a, b)) for a, b in piece_ranges(c0, c1, pieces)} == {'items'}
    want = S.combine(parts)
    summ = np_(summ)
    assert same_bits(summ, want)
    check_summary(summ, S.Shape.of(grid, c0, c1), st, abr[0], abr[1], op, None, pieces=len(parts),
                  what=('to_host', num, pieces))
    grid.close()


def div_maybe_zero(a, b):
    """the device's division of the aberration epilogue: IEEE a / b (0 / b a signed zero)"""
    with np.errstate(all='ignore'):
        q = np.float64(a)/b
    z = (a == 0.0) & (b == b) & (b != 0.0)
    return np.where(z, np.copysign(0.0, np.copysign(1.0, a)*np.copysign(1.0, b)), q)


@pytest.mark.parametrize('name', ['dblgauss', 'threemir'])
def test_trace_grid_focus_planes(oracle, name):
    """rt_trace_grid_focus: plane k's summary against references built from the per-ray p, d,
    status, op: ax = (p.x + (foc/d.z) d.x) - rx with rx from chief_ref_focus"""
    opm, tab = model(name), table(name)
    foc = [0.0, -0.05, 0.1]
    wi = tab.wvl_index(opm.seq_model.central_wavelength())
    for num, rng, want in ((16, lambda n: (0, n), 'records'), (48, lambda n: (10, 15), 'items'),
                           (48, lambda n: (3, n - 5), 'records')):
        grid = E.grid_for_model(opm, tab, num, ref_img=None)
        c0, c1 = rng(grid.n_chunks)
        shape = S.Shape.of(grid, c0, c1)
        assert regime_of(shape) == want
        ref = grid.chief_ref_focus(tab, wi, foc)
        res = E.BundleResult(grid.rays_in_chunks(c0, c1), tab.n_ifc, torch.device('cuda', 0),
                             ('p', 'd', 'status', 'op'))
        summ = np_(E.trace_grid_focus(tab, grid, foc, c0, c1, ref_img=ref, res=res))
        torch.cuda.synchronize()
        got = {k: np_(getattr(res, k)) for k in ('p', 'd', 'status', 'op')}
        check_rays(oracle, tab, grid, c0, c1, got)
        p, d = got['p'], got['d']
        ref = np_(ref)
        tiles = (np.arange(grid.n_rays)//grid.rays_per_tile)[grid.first_ray_of_chunk(c0):grid.first_ray_of_chunk(c1)]
        f = tiles//grid.n_wvls
        for k, fk in enumerate(foc):
            dist = div_maybe_zero(np.float64(fk), d[2])
            with np.errstate(all='ignore'):
                ax = (p[0] + dist*d[0]) - ref[k, f, 0]
                ay = (p[1] + dist*d[1]) - ref[k, f, 1]
            check_summary(summ[k], shape, got['status'], ax, ay, got['op'], want, what=(name, num, k))
        grid.close()


def test_combine_shards_that_split_tiles(oracle):
    """rt_combine_summaries over shards cut inside tiles, each shard in its own regime; tile 1
    (chunks 9-17) is split over three shards, so the order of the combine shows in its bits"""
    tab = table('dblgauss')
    grid = E.grid_for_model(model('dblgauss'), tab, 48)
    cuts = [0, 7, 11, 12, 40, 41, grid.n_chunks]
    parts, want, sts, abrs, ops = [], [], [], [], []
    for (a, b), rg in zip(zip(cuts[:-1], cuts[1:]), ('items', 'items', 'items', 'records', 'items', 'records')):
        summ, got = trace_and_check(oracle, tab, grid, a, b, rg, what=('shard', a, b))
        parts.append(torch.from_numpy(summ).cuda())
        want.append(S.ordered_summary(S.Shape.of(grid, a, b), got['status'], got['abr'][0], got['abr'][1],
                                      got['op'], rg))
        sts.append(got['status']); abrs.append(got['abr']); ops.append(got['op'])
    comb = np_(E.combine_summaries(parts))
    assert same_bits(comb, S.combine(want))
    abr = np.concatenate(abrs, axis=1)
    check_summary(comb, S.Shape.of(grid), np.concatenate(sts), abr[0], abr[1], np.concatenate(ops), None,
                  pieces=len(parts), what='shards')
    grid.close()


def test_zz_report_cancellation():
    """the worst kappa = (sum x^2 + sum y^2) / (n var) met by the statistics checks above"""
    if WORST['tiles'] == 0:
        pytest.skip('no statistics checked in this session')
    print(f"\nspot_statistics: {WORST['tiles']} tiles checked, worst kappa {WORST['kappa']:.3g} at {WORST['where']}")
