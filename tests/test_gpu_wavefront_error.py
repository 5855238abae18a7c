"""GPU: rt_trace_grid_wfe against the restatement of its sums (tests/wfe_sums.py) built from the
launch's own per-ray values, and analyses.wavefront_error against numpy statistics of the
reference's RayGrid class, tile by tile.

Fixtures and the kernel family each takes: dblgauss, rc lean; cellphone, evenasph lean POLY;
exotic general (rotated transforms, aperture lists); fisheye general (wide-angle pupil); relay_na general
(angular pupil); diffractive_wild general (phase elements: status 4 and NaN OPDs)."""
import numpy as np
import pytest
import torch

import wfe_sums as WS
from conftest import load_model
from test_wavefront_error import check_against_numpy
from rayoptics_b200 import _abi, engine as E, analyses as A
from rayoptics_b200.table import SurfaceTable

pytestmark = pytest.mark.gpu

FAMILY = {'dblgauss': 'k_trace_grid_lean_wfe<false>', 'rc': 'k_trace_grid_lean_wfe<false>',
          'cellphone': 'k_trace_grid_lean_wfe<true>', 'evenasph': 'k_trace_grid_lean_wfe<true>',
          'exotic': 'k_trace_grid_wfe<true>', 'fisheye': 'k_trace_grid_wfe<true>',
          'relay_na': 'k_trace_grid_wfe<true>', 'diffractive_wild': 'k_trace_grid_wfe<true>'}
SUM_COLS = [0, 1, 2, 3, 4] + list(WS.SUM_COLS) + [20, 21, 22, 23]
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


def same_bits(got, want, what):
    """sums and counts bit for bit (NaN: both NaN), min / max by =="""
    g, w = got[:, SUM_COLS], want[:, SUM_COLS]
    assert (np.isnan(g) == np.isnan(w)).all(), what
    m = ~np.isnan(w)
    assert g[m].view(np.uint64).tolist() == w[m].view(np.uint64).tolist(), what
    assert (got[:, [WS.MIN_COL, WS.MAX_COL]] == want[:, [WS.MIN_COL, WS.MAX_COL]]).all(), what


def launch(tab, grid, c0, c1):
    n = grid.rays_in_chunks(c0, c1)
    res = E.BundleResult(n, tab.n_ifc, torch.device('cuda', 0), ('opd', 'status'))
    summ = E.trace_grid_wfe(tab, grid, c0, c1, res=res).cpu().numpy()
    return summ, res.status.cpu().numpy(), res.opd.cpu().numpy()


def check_launch(name, num, which):
    opm, tab, grid, fields, wvls = setup(name, num)
    c0, c1 = chunk_range(grid, which)
    summ, status, opd = launch(tab, grid, c0, c1)
    assert summ.shape == (grid.n_tiles, _abi.RT_WFE_DOUBLES)
    # 1. per-ray outputs equal trace_grid's on the same grid
    ref = E.trace_grid(tab, grid, c0, c1, outputs=('opd', 'status'), summary=False)
    assert status.tobytes() == ref.status.cpu().numpy().tobytes()
    assert opd.tobytes() == ref.opd.cpu().numpy().tobytes()
    # 2. the record against the restatement built from those per-ray values
    shape = WS.Shape.of(grid, c0, c1)
    x, y = WS.grid_pupil_xy(grid, shape)
    want = WS.ordered_summary(shape, status, opd, x, y)
    same_bits(summ, want, (name, num, which))
    exact, absum = WS.exact_summary(shape, status, opd, x, y)
    err = np.abs(summ[:, list(WS.SUM_COLS)] - exact[:, list(WS.SUM_COLS)])
    fin = np.isfinite(exact[:, list(WS.SUM_COLS)])
    assert (err[fin] <= WS.sum_bound(absum, WS.chain_depth(shape, 'items'))[fin]).all()
    if c1 == c0:
        assert np.array_equal(summ, WS.identity(grid.n_tiles))
    return opm, tab, grid, fields, wvls, summ, status, opd


SIZES = [1, 33, 64]


@pytest.mark.parametrize('which', ['full', 'mid', 'one', 'empty'])
@pytest.mark.parametrize('num', SIZES)
@pytest.mark.parametrize('name', list(FAMILY))
def test_record_equals_the_restatement(name, num, which):
    check_launch(name, num, which)


@pytest.mark.parametrize('name', ['dblgauss', 'exotic'])
def test_record_equals_the_restatement_512(name):
    check_launch(name, 512, 'full')
    check_launch(name, 512, 'mid')


@pytest.mark.parametrize('name', list(FAMILY))
def test_kernel_family(name):
    """the instance rt_trace_grid_wfe launches, by name (torch.profiler)"""
    opm, tab, grid, fields, wvls = setup(name, 33)
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        E.trace_grid_wfe(tab, grid)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    hit = [n for n in names if 'wfe' in n and 'k_trace_grid' in n]
    assert hit and all(FAMILY[name] in n for n in hit), (name, hit)
    assert any('k_reduce_wfe' in n for n in names)


@pytest.mark.parametrize('num', [33, 64, 512])
@pytest.mark.parametrize('name', list(FAMILY))
def test_statistics_equal_numpy_statistics_of_raygrids(name, num):
    """wavefront_error tile by tile against numpy statistics of the RayGrid map of that tile"""
    if num == 512 and name not in ('dblgauss', 'rc', 'exotic'):
        pytest.skip('512^2 on three fixtures')
    opm = load_model(name)
    wfe = A.wavefront_error(opm, num)
    fields, wvls = opm.optical_spec.field_of_view.fields, opm.seq_model.wvlns
    maps = [[A.RayGrid(opm, f=fi, wl=wl, num_rays=num).grid for wl in wvls] for fi in range(len(fields))]
    nan_tiles = np.isnan(wfe.summary[:, 7]).reshape(len(fields), len(wvls))
    for fi in range(len(fields)):
        for wi in range(len(wvls)):
            if nan_tiles[fi, wi]:                    # a status-0 ray with a NaN OPD: the map drops it
                assert np.isnan(wfe.rms[fi, wi]) and wfe.n_ok[fi, wi] > np.isfinite(maps[fi][wi][2]).sum()
                continue
            if wfe.n_ok[fi, wi] < 4:
                continue
            check_against_numpy(_Tile(wfe, fi, wi), opm, [None], [None], [[maps[fi][wi]]], depth=num*num)


class _Tile:
    """one tile of a WavefrontError as a 1 x 1 result (check_against_numpy's input)"""

    def __init__(self, wfe, fi, wi):
        for k in ('n_ok', 'rms', 'pv', 'rms_tilt', 'tilt_x', 'tilt_y', 'rms_focus', 'focus'):
            setattr(self, k, getattr(wfe, k)[fi:fi + 1, wi:wi + 1])


@pytest.mark.parametrize('name', ['dblgauss', 'exotic', 'diffractive_wild'])
def test_combine_over_ranges_that_split_tiles(name):
    opm, tab, grid, fields, wvls = setup(name, 33)
    n = grid.n_chunks
    cuts = [0, 3, grid.chunks_per_tile + 2, n - 1, n]
    parts, want = [], []
    for a, b in zip(cuts[:-1], cuts[1:]):
        summ, status, opd = launch(tab, grid, a, b)
        parts.append(summ)
        shape = WS.Shape.of(grid, a, b)
        x, y = WS.grid_pupil_xy(grid, shape)
        want.append(WS.ordered_summary(shape, status, opd, x, y))
    got = E.combine_summaries(torch.as_tensor(np.stack(parts), device='cuda')).cpu().numpy()
    same_bits(got, WS.combine(want), name)


@pytest.mark.parametrize('name', ['dblgauss', 'fisheye'])
def test_sharded_wavefront_error(name):
    opm = load_model(name)
    num = 40
    s0 = A.wavefront_error(opm, num, shard=(0, 2)).summary
    s1 = A.wavefront_error(opm, num, shard=(1, 2)).summary
    opm_, tab, grid, fields, wvls = setup(name, num)
    from rayoptics_b200.parallel import shard_chunks
    want = []
    for r in range(2):
        a, b = shard_chunks(grid.n_chunks, r, 2)
        summ, status, opd = launch(tab, grid, a, b)
        shape = WS.Shape.of(grid, a, b)
        x, y = WS.grid_pupil_xy(grid, shape)
        want.append(WS.ordered_summary(shape, status, opd, x, y))
    same_bits(s0, want[0], 'rank 0')
    same_bits(s1, want[1], 'rank 1')
    combined = E.combine_summaries(torch.as_tensor(np.stack([s0, s1]), device='cuda')).cpu().numpy()
    same_bits(combined, WS.combine(want), 'combined')
    whole = A.wavefront_error(opm, num)
    assert (whole.n_ok == combined[:, 0].reshape(whole.n_ok.shape)).all()


def test_one_grid_launch_and_one_small_copy():
    opm = load_model('dblgauss')
    A.wavefront_error(opm, 32)
    n0 = E.launch_count()
    A.wavefront_error(opm, 32)
    # chief rays (one grid launch), the WFE trace, its reduction
    assert E.launch_count() - n0 == 3


def test_abi_argument_checks():
    lib = _abi.load_library()
    opm, tab, grid, fields, wvls = setup('dblgauss', 8)
    dev = torch.device('cuda', 0)
    opts = _abi.make_opts(first_surf=1, last_surf=tab.n_ifc - 2, check_apertures=True)
    summ = torch.empty((grid.n_tiles, _abi.RT_WFE_DOUBLES), dtype=torch.float64, device=dev)
    scratch = torch.empty(lib.rt_grid_wfe_scratch_bytes(grid.handle, 0, grid.n_chunks)//8,
                          dtype=torch.float64, device=dev)
    plain = E.grid_for_model(opm, tab, 8, ref_img=None)          # no wave records
    full = torch.empty(10, dtype=torch.float64, device=dev)
    ok_out, bad_out = _abi.rt_out(), _abi.rt_out()
    bad_out.full = full.data_ptr()
    import ctypes as C
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())     # noqa: E731
    n0 = E.launch_count()
    for g, out, s, sc, msg in ((plain, ok_out, summ, scratch, 'wave'), (grid, bad_out, summ, scratch, 'full'),
                               (grid, ok_out, None, scratch, 'summary'), (grid, ok_out, summ, None, 'scratch')):
        rc = lib.rt_trace_grid_wfe(tab.handle, g.handle, 0, g.n_chunks, C.byref(opts), C.byref(out), P(s), P(sc), None)
        err = lib.rt_last_error().decode()
        assert rc == -1 and msg in err, (msg, rc, err)
    assert E.launch_count() == n0
    assert lib.rt_grid_wfe_scratch_bytes(grid.handle, 5, 4) == 0
    plain.close()


def test_decentered_image_gap_is_refused():
    """threemir decenters the last interface before the image: the OPD epilogue does not apply, as
    for rt_trace_grid's opd output (RT_ERR_UNSUPPORTED, before any device work)"""
    opm = load_model('threemir')
    tab = SurfaceTable.from_model(opm.seq_model, device=0)
    fields, wvls = list(opm.optical_spec.field_of_view.fields), list(opm.seq_model.wvlns)
    from test_analyses_vs_reference import OracleBackend
    args, kw = A.wavefront_grid_args(opm, None, 8, fields, wvls, 0.0, backend=OracleBackend(opm))
    args = (args[0], [tab.wvl_index(w) for w in wvls]) + args[2:]
    grid = E.PupilGrid(*args, device=0, **kw)
    n0 = E.launch_count()
    with pytest.raises(_abi.EngineError, match='-3'):
        E.trace_grid_wfe(tab, grid)
    with pytest.raises(_abi.EngineError, match='-3'):
        E.trace_grid(tab, grid, outputs=('opd',), summary=False)
    assert E.launch_count() == n0
    grid.close()
