"""GPU: rt_grid_zernike against the restatement of its sums (tests/zernike_sums.py) built from the
launch's own per-ray opd and status, on every trace family, and analyses.zernike_fit against
numpy lstsq on the reference's RayGrid maps, tile by tile.

Fixtures and the trace kernel each takes (as in test_gpu_wavefront_error.py): dblgauss, rc lean;
cellphone, evenasph lean POLY; exotic, fisheye, relay_na general; diffractive_wild general with
phase elements (status 4 and NaN OPDs)."""
import ctypes as C

import numpy as np
import pytest
import torch

import zernike_sums as ZS
from conftest import load_model
from test_zernike import check_against_lstsq, edge_points
from rayoptics_b200 import _abi, engine as E, analyses as A
from rayoptics_b200.table import SurfaceTable

pytestmark = pytest.mark.gpu

NAMES = ['dblgauss', 'rc', 'cellphone', 'evenasph', 'exotic', 'fisheye', 'relay_na', 'diffractive_wild']
TERMS = [1, 4, 16, 37]
_SETUP = {}


def setup(name, num):
    key = (name, num)
    if key not in _SETUP:
        opm = load_model(name)
        tab = SurfaceTable.from_model(opm.seq_model, device=0)
        fields = list(opm.optical_spec.field_of_view.fields)
        wvls = list(opm.seq_model.wvlns)
        args, kw = A.wavefront_grid_args(opm, tab, num, fields, wvls, opm.optical_spec.defocus.focus_shift)
        grid = E.PupilGrid(*args, device=0, **kw)
        _SETUP[key] = (opm, tab, grid, fields, wvls)
    return _SETUP[key]


def chunk_range(grid, which):
    n, cpt = grid.n_chunks, grid.chunks_per_tile
    return {'full': (0, n), 'mid': (cpt//2, n - max(cpt//3, 1)) if n > 2 else (0, n),
            'one': (n//2, n//2 + 1), 'empty': (n//2, n//2)}[which]


def launch(tab, grid, c0, c1, n_terms):
    n = grid.rays_in_chunks(c0, c1)
    res = E.BundleResult(n, tab.n_ifc, torch.device('cuda', 0), ('opd', 'status'))
    summ = E.trace_grid_zernike(tab, grid, n_terms, c0, c1, res=res).cpu().numpy()
    return summ, res.status.cpu().numpy(), res.opd.cpu().numpy()


def want_record(grid, c0, c1, status, opd, n_terms):
    shape = ZS.Shape.of(grid, c0, c1)
    x, y = ZS.grid_pupil_xy(grid, shape)
    return ZS.ordered_summary(shape, status, opd, x, y, n_terms), shape, x, y


def check_launch(name, num, which, n_terms):
    opm, tab, grid, fields, wvls = setup(name, num)
    c0, c1 = chunk_range(grid, which)
    summ, status, opd = launch(tab, grid, c0, c1, n_terms)
    assert summ.shape == (grid.n_tiles, _abi.RT_ZERN_DOUBLES)
    want, shape, x, y = want_record(grid, c0, c1, status, opd, n_terms)
    ZS.same_bits(summ, want, n_terms, (name, num, which, n_terms))
    if c1 == c0:
        assert np.array_equal(summ, ZS.identity(grid.n_tiles))
    return summ


@pytest.mark.parametrize('n_terms', TERMS)
@pytest.mark.parametrize('which', ['full', 'mid', 'one', 'empty'])
@pytest.mark.parametrize('num', [1, 33, 64])
@pytest.mark.parametrize('name', NAMES)
def test_record_equals_the_restatement(name, num, which, n_terms):
    check_launch(name, num, which, n_terms)


@pytest.mark.parametrize('name, which, n_terms', [('dblgauss', 'full', 37), ('dblgauss', 'mid', 16),
                                                  ('exotic', 'full', 37)])
def test_record_equals_the_restatement_512(name, which, n_terms):
    check_launch(name, 512, which, n_terms)


def adversarial_grid(num=64):
    """the double Gauss's grid with pupil tables that put rays exactly on r2 = 1, next to it and
    outside the disk"""
    opm, tab, _, fields, wvls = setup('dblgauss', num)
    args, kw = A.wavefront_grid_args(opm, tab, num, fields, wvls, 0.0)
    rng = np.random.default_rng(num)
    ex, ey = edge_points()
    px = np.concatenate([np.unique(ex), rng.uniform(-1.1, 1.1, num)])[:num]
    # every chunk (4 rows of 64) has a row x = 1, -1 or -0 (r2 = 1 with y = 0 or +-1) and a row x =
    # the double above 1
    px[::4] = np.resize([1.0, -1.0, -0.0], len(px[::4]))
    px[1::4] = np.nextafter(1.0, 2.0)
    py = np.concatenate([np.unique(ey), rng.uniform(-1.1, 1.1, num)])[:num]
    nf = len(fields)
    args = args[:2] + (np.tile(px, (nf, 1)), np.tile(py[::-1], (nf, 1))) + args[4:]
    return tab, E.PupilGrid(*args, device=0, **kw)


@pytest.mark.parametrize('n_terms', TERMS)
@pytest.mark.parametrize('which', ['full', 'mid', 'one'])
def test_caller_supplied_adversarial_arrays(which, n_terms):
    tab, grid = adversarial_grid()
    c0, c1 = chunk_range(grid, which)
    n = grid.rays_in_chunks(c0, c1)
    rng = np.random.default_rng(n + n_terms)
    w = rng.standard_normal(n)*10.0**rng.integers(-9, 4, n)
    w[rng.random(n) < 0.1] *= -1e3
    w[rng.random(n) < 0.05] = -0.0
    w[rng.random(n) < 0.05] = 0.0
    status = np.where(rng.random(n) < 0.8, 0, rng.integers(-2, 7, n)).astype(np.int32)
    x, y = ZS.grid_pupil_xy(grid, ZS.Shape.of(grid, c0, c1))
    r2 = x*x + y*y
    on = np.nonzero(r2 == 1.0)[0]
    near = np.nonzero((r2 > 1.0) & (r2 < 1 + 1e-15))[0]
    status[on[::2]] = 0                                      # used rays exactly on the edge
    status[near] = 0                                         # and status-0 rays just outside it
    if n > 2*grid.rays_per_tile:
        w[:300:37] = np.nan                                  # NaN OPDs in the first tile of the range only
    assert len(on) and len(near)
    dev = torch.device('cuda', 0)
    summ = E.grid_zernike(grid, c0, c1, n_terms, torch.as_tensor(status, device=dev),
                          torch.as_tensor(w, device=dev)).cpu().numpy()
    want = want_record(grid, c0, c1, status, w, n_terms)[0]
    ZS.same_bits(summ, want, n_terms, (which, n_terms))
    grid.close()


@pytest.mark.parametrize('name', ['dblgauss', 'exotic', 'diffractive_wild'])
def test_combine_over_ranges_that_split_tiles(name):
    opm, tab, grid, fields, wvls = setup(name, 33)
    n = grid.n_chunks
    cuts = [0, 3, grid.chunks_per_tile + 2, n - 1, n]
    for n_terms in (4, 37):
        parts, want = [], []
        for a, b in zip(cuts[:-1], cuts[1:]):
            summ, status, opd = launch(tab, grid, a, b, n_terms)
            parts.append(summ)
            want.append(want_record(grid, a, b, status, opd, n_terms)[0])
        got = E.combine_summaries(torch.as_tensor(np.stack(parts), device='cuda')).cpu().numpy()
        ZS.same_bits(got, ZS.combine(want), n_terms, (name, n_terms))


@pytest.mark.parametrize('name', ['dblgauss', 'fisheye'])
def test_sharded_zernike_fit(name):
    opm = load_model(name)
    num, n_terms = 40, 16
    s0 = A.zernike_fit(opm, num, n_terms, shard=(0, 2)).summary
    s1 = A.zernike_fit(opm, num, n_terms, shard=(1, 2)).summary
    opm_, tab, grid, fields, wvls = setup(name, num)
    from rayoptics_b200.parallel import shard_chunks
    want = []
    for r in range(2):
        a, b = shard_chunks(grid.n_chunks, r, 2)
        summ, status, opd = launch(tab, grid, a, b, n_terms)
        want.append(want_record(grid, a, b, status, opd, n_terms)[0])
    ZS.same_bits(s0, want[0], n_terms, 'rank 0')
    ZS.same_bits(s1, want[1], n_terms, 'rank 1')
    combined = E.combine_summaries(torch.as_tensor(np.stack([s0, s1]), device='cuda')).cpu().numpy()
    ZS.same_bits(combined, ZS.combine(want), n_terms, 'combined')
    whole = A.zernike_fit(opm, num, n_terms)
    assert (whole.n_used == combined[:, 5].reshape(whole.n_used.shape)).all()


@pytest.mark.parametrize('num', [33, 64, 512])
@pytest.mark.parametrize('name', ['dblgauss', 'rc', 'cellphone', 'exotic'])
def test_coefficients_equal_lstsq_on_raygrids(name, num):
    if num == 512 and name not in ('dblgauss', 'rc'):
        pytest.skip('512^2 on two fixtures')
    opm = load_model(name)
    fit = A.zernike_fit(opm, num, 37)
    fields, wvls = opm.optical_spec.field_of_view.fields, opm.seq_model.wvlns
    maps = [[A.RayGrid(opm, f=fi, wl=wl, num_rays=num).grid for wl in wvls] for fi in range(len(fields))]
    cpt = -(-num*num//ZS.CHUNK)
    check_against_lstsq(fit, opm, fields, wvls, maps, depth=ZS.CHUNK + cpt)


def test_four_launches():
    opm = load_model('dblgauss')
    A.zernike_fit(opm, 32, 37)
    n0 = E.launch_count()
    A.zernike_fit(opm, 32, 37)
    # chief rays, the opd trace, the moments, their reduction
    assert E.launch_count() - n0 == 4


def test_bad_arguments_launch_nothing():
    lib = _abi.load_library()
    opm, tab, grid, fields, wvls = setup('dblgauss', 8)
    dev = torch.device('cuda', 0)
    n = grid.rays_in_chunks(0, grid.n_chunks)
    st = torch.zeros(n, dtype=torch.int32, device=dev)
    w = torch.zeros(n, dtype=torch.float64, device=dev)
    summ = torch.empty((grid.n_tiles, _abi.RT_ZERN_DOUBLES), dtype=torch.float64, device=dev)
    scratch = torch.empty(lib.rt_grid_zernike_scratch_bytes(grid.handle, 0, grid.n_chunks, 37)//8,
                          dtype=torch.float64, device=dev)
    args, kw = A.wavefront_grid_args(opm, tab, 8, fields, wvls, 0.0)
    vign = E.PupilGrid(*args, device=0, **dict(kw, apply_vignetting=True))
    paired = E.PupilGrid(*args, device=0, **dict(kw, paired=True))
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())     # noqa: E731
    nc = grid.n_chunks
    n0 = E.launch_count()
    for g, c0, c1, J, s, o, sm, sc, msg in (
            (vign, 0, vign.n_chunks, 37, st, w, summ, scratch, 'vignett'),
            (paired, 0, paired.n_chunks, 37, st, w, summ, scratch, 'product grid'),
            (grid, 0, nc + 1, 37, st, w, summ, scratch, 'range'),
            (grid, 2, 1, 37, st, w, summ, scratch, 'range'),
            (grid, -1, nc, 37, st, w, summ, scratch, 'range'),
            (grid, 0, nc, 0, st, w, summ, scratch, 'n_terms'),
            (grid, 0, nc, 38, st, w, summ, scratch, 'n_terms'),
            (grid, 0, nc, 37, None, w, summ, scratch, 'required'),
            (grid, 0, nc, 37, st, None, summ, scratch, 'required'),
            (grid, 0, nc, 37, st, w, summ, None, 'required'),
            (grid, 0, nc, 37, st, w, None, scratch, 'summary')):
        rc = lib.rt_grid_zernike(g.handle, c0, c1, J, P(s), P(o), P(sm), P(sc), None)
        err = lib.rt_last_error().decode()
        assert rc == -1 and msg in err, (msg, rc, err)
    assert E.launch_count() == n0
    assert lib.rt_grid_zernike_scratch_bytes(grid.handle, 5, 4, 4) == 0
    assert lib.rt_grid_zernike_scratch_bytes(grid.handle, 0, 1, 38) == 0
    with pytest.raises(ValueError):
        E.grid_zernike(grid, 0, nc, 4, st[1:], w)
    with pytest.raises(ValueError):
        E.grid_zernike(grid, 0, nc, 4, st, w.float())
    assert E.launch_count() == n0
    vign.close()
    paired.close()


def test_decentered_image_gap_is_refused():
    """threemir decenters the last interface before the image: no OPD, so no Zernike fit
    (RT_ERR_UNSUPPORTED from the opd trace, before any device work)"""
    opm = load_model('threemir')
    tab = SurfaceTable.from_model(opm.seq_model, device=0)
    fields, wvls = list(opm.optical_spec.field_of_view.fields), list(opm.seq_model.wvlns)
    from test_analyses_vs_reference import OracleBackend
    args, kw = A.wavefront_grid_args(opm, None, 8, fields, wvls, 0.0, backend=OracleBackend(opm))
    args = (args[0], [tab.wvl_index(w) for w in wvls]) + args[2:]
    grid = E.PupilGrid(*args, device=0, **kw)
    n0 = E.launch_count()
    with pytest.raises(_abi.EngineError, match='-3'):
        E.trace_grid_zernike(tab, grid, 4)
    assert E.launch_count() == n0
    grid.close()
