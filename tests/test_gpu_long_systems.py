"""GPU: every trace entry point on the long systems of tests/long_models.py, whose
surface tables sit on the shared-memory budgets of rt_table_create (test_long_systems.py restates
the choice and places the fixtures):

  long640    lean plan exactly at the budget (a summary CTA asks for 204 800 B)
  long320    lean POLY plan exactly at the budget
  long256    general kernels, table staged, exactly at the budget
  long360    lean plan of 97 920 B: one summary CTA per SM, two of the other kernels
  <name>+1   the same model with one index row more: general kernels, table in global memory

Each launch is checked against the oracle (records bit for bit, opd within 1e-12 mm), its spot,
wavefront and Zernike sums against the restatements of tests/spot_sums.py, wfe_sums.py and
zernike_sums.py, and the kernel instance it ran against the one the table's regime implies
(torch.profiler).  The spot-sum regime of a launch (per-chunk records or work items) follows from its
CTA count; on these tables shared memory decides it, read from the table's own plan size and the
device's limits."""
import os

import numpy as np
import pytest
import torch

import aim_ref as AR
import spot_sums as S
import test_gpu_through_focus as TF
import test_gpu_wavefront_error as WF
import test_gpu_zernike as GZ
import long_models as LM
from conftest import seeded_bundle
from test_gpu_spot_sums import check_rays, check_summary, same_bits
from test_long_systems import plan, table_args
from rayoptics_b200 import _abi, engine as E, analyses as A, table as T

pytestmark = pytest.mark.gpu

DRY = os.environ.get('B200RT_DRYRUN') == '1'
device_only = pytest.mark.skipif(DRY, reason='the dry-run engine stands in for rt_trace_bundle and '
                                             'rt_trace_grid only')
SEEN = {}                    # kernel instance -> number of launches met by the checks
TABLES = ['long640', 'long640+1', 'long320', 'long320+1', 'long256', 'long256+1', 'long360']
_TABLES = {}


def table(key):
    """(model, table, plan) of ``key``: a fixture name, '+1' for one index row more"""
    if key not in _TABLES:
        name, _, extra = key.partition('+')
        opm, descs, n_by_wvl, wvls = table_args(name, int(extra or 0))
        tab = T.SurfaceTable.from_model(opm.seq_model, wvls=wvls, device=0)
        _TABLES[key] = (opm, tab, plan(descs, len(wvls)))
    return _TABLES[key]


def b(v):
    return 'true' if v else 'false'


def instance(p, entry, kind=0, summary=False, opd=False):
    """the kernel instance the entry point launches on a table of plan ``p``; ``kind``: output kind
    (0: p, d; 1: + normals / dst; 2: whole rays)"""
    lean, poly, stage = p['regime'] in ('lean', 'lean_poly'), p['regime'] == 'lean_poly', p['regime'] == 'staged'
    if entry == 'bundle':
        return f'k_trace_bundle_lean<{kind}, {b(poly)}>' if lean else f'k_trace_bundle<{b(kind == 2)}, {b(stage)}>'
    if entry == 'grid':
        if lean:
            return f'k_trace_grid_lean<{kind}, {b(summary)}, {b(opd)}, {b(poly)}>'
        return f'k_trace_grid<{b(kind == 2)}, {b(summary)}, {b(stage)}, {b(opd)}>'
    fam = {'focus': 'focus', 'wfe': 'wfe'}[entry]
    return f'k_trace_grid_lean_{fam}<{b(poly)}>' if lean else f'k_trace_grid_{fam}<{b(stage)}>'


def launched(want, fn):
    """run ``fn`` under torch.profiler and assert that the trace kernel it launches is ``want``"""
    if DRY:
        return fn()
    from torch.profiler import profile, ProfilerActivity
    for _ in range(3):        # a profiling session now and then reports no device events: run it again
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            r = fn()
            torch.cuda.synchronize()
        hit = [e.name for e in prof.events() if 'k_trace_' in e.name]
        if hit:
            break
    assert hit and all(want + '(' in n for n in hit), (want, hit)
    SEEN[want] = SEEN.get(want, 0) + len(hit)
    return r


def ctas_per_sm_bound(smem):
    """an upper bound of the 256-thread CTAs per SM of a launch with ``smem`` bytes of dynamic shared
    memory (threads and shared memory; registers can only lower it)"""
    prop = torch.cuda.get_device_properties(0)
    reserved = getattr(prop, 'reserved_shared_memory_per_block', 1024)
    return min(prop.max_threads_per_multi_processor//S.CHUNK,
               prop.shared_memory_per_multiprocessor//(smem + reserved))


def summary_smem(p):
    return p['plan_bytes'] + p['acc_bytes']


def regime(p, shape):
    """the spot-sum regime of a summary launch over ``shape`` on a table of plan ``p``, or None where
    registers could decide it"""
    if DRY:
        return S.regime(shape, 132, 1)
    return S.regime(shape, torch.cuda.get_device_properties(0).multi_processor_count,
                    ctas_per_sm_bound(summary_smem(p)))


def np_(t):
    return t.detach().cpu().numpy()


# ---------------------------------------------------------------- placement on the device
@device_only
def test_occupancy_of_the_tables():
    """the budget tables allow one summary CTA per SM; long360 one summary CTA and two of the kernels
    without accumulators"""
    for key in ('long640', 'long320', 'long256', 'long360'):
        p = table(key)[2]
        assert ctas_per_sm_bound(summary_smem(p)) == 1, key
    p = table('long360')[2]
    assert ctas_per_sm_bound(p['plan_bytes']) == 2


# ---------------------------------------------------------------- rt_trace_bundle
BUNDLE_OUTS = {0: ('p', 'd', 'op', 'status', 'fail_surf', 'n_seg'),
               1: ('p', 'd', 'nrml', 'dst', 'op', 'status', 'fail_surf', 'n_seg'),
               2: ('p', 'd', 'nrml', 'dst', 'op', 'status', 'fail_surf', 'n_seg')}


@pytest.mark.parametrize('key', TABLES)
def test_bundle_equals_the_oracle(oracle, key):
    """output kinds 0, 1, 2 against the oracle bit for bit (whole rays: 2 048 rays)"""
    opm, tab, p = table(key)
    p0, d0, wv = seeded_bundle(opm, 2048, np.random.default_rng(31))
    n_ifc = tab.n_ifc
    opts = dict(first_surf=1, last_surf=n_ifc - 2, check_apertures=True)
    ref = oracle.trace_bundle(tab.descs, tab.n_by_wvl, p0, d0, wv, _abi.make_opts(**opts), want_full=True,
                              n_threads=8, wvls=tab.wvls)
    assert {0, 3} <= set(np.unique(ref['status']).tolist())
    for kind in (0, 1, 2):
        r = launched(instance(p, 'bundle', kind),
                     lambda: E.trace_bundle(tab, p0, d0, wv, full=kind == 2, outputs=BUNDLE_OUTS[kind], **opts))
        torch.cuda.synchronize()
        assert (np_(r.status) == ref['status']).all()
        for k in ('fail_surf', 'n_seg', 'op'):
            assert same_bits(np_(getattr(r, k)), ref[k]), (key, kind, k)
        assert same_bits(np_(r.p), ref['last'][0:3]) and same_bits(np_(r.d), ref['last'][3:6]), (key, kind)
        if kind >= 1:
            assert same_bits(np_(r.dst), ref['last'][6]) and same_bits(np_(r.nrml), ref['last'][7:10]), (key, kind)
        if kind == 2:
            assert same_bits(np_(r.full), ref['full']), (key, kind)


# ---------------------------------------------------------------- rt_trace_grid
def grid_launch(oracle, key, grid, c0, c1, full, summary, want_regime=None, sample=None):
    """one rt_trace_grid launch: the instance, per-ray records against the oracle (whole rays too),
    the summary against the restatements; returns the regime the launch had"""
    opm, tab, p = table(key)
    outs = ('status', 'abr', 'op', 'p', 'd')
    r = launched(instance(p, 'grid', 2 if full else 0, summary),
                 lambda: E.trace_grid(tab, grid, c0, c1, outputs=outs, full=full, summary=summary))
    torch.cuda.synchronize()
    got = {k: np_(getattr(r, k)) for k in outs}
    chunks = None if sample is None else np.random.default_rng(c0 + 7*c1).integers(c0, c1, sample)
    check_rays(oracle, tab, grid, c0, c1, got, chunks)
    if full:
        base = grid.first_ray_of_chunk(c0)
        a, b_ = grid.first_ray_of_chunk(c0 + (c1 - c0)//2), grid.first_ray_of_chunk(c0 + (c1 - c0)//2 + 1)
        pr, dr, wv, _ = oracle.grid_start_rays(grid.c_spec(), a, b_)
        ref = oracle.trace_bundle(tab.descs, tab.n_by_wvl, pr, dr, wv,
                                  _abi.make_opts(first_surf=1, last_surf=tab.n_ifc - 2, check_apertures=True),
                                  want_full=True, n_threads=8, wvls=tab.wvls)
        assert same_bits(np_(r.full[:, :, a - base:b_ - base]), ref['full']), (key, 'full')
    if not summary:
        return None
    shape = S.Shape.of(grid, c0, c1)
    rg = regime(p, shape)
    if want_regime is not None:
        assert rg == want_regime, (key, c0, c1, rg)
    # (the dry-run engine's sums are exact: bound only)
    check_summary(np_(r.summary), shape, got['status'], got['abr'][0], got['abr'][1], got['op'],
                  None if DRY else rg, what=(key, c0, c1))
    return rg


@pytest.mark.parametrize('key', TABLES)
def test_grid_instances(oracle, key):
    """(full, summary) x {no, yes} at 24^2 rays per tile (3 chunks): every instance of the table's
    regime, over the whole grid and over a range that cuts tiles"""
    opm, tab, p = table(key)
    grid = E.grid_for_model(opm, tab, 24)
    n = grid.n_chunks
    for full in (False, True):
        for summary in (False, True):
            for c0, c1 in ((0, n), (4, n - 2)):
                grid_launch(oracle, key, grid, c0, c1, full, summary)
    grid.close()


@pytest.mark.parametrize('num,want', [(180, 'records'), (192, 'items')])
@pytest.mark.parametrize('key', ['long640', 'long320', 'long256', 'long360'])
def test_grid_regime_set_by_shared_memory(oracle, key, num, want):
    """one summary CTA per SM: 180^2 rays per tile (127 chunks) keep per-chunk records, 192^2
    (144 chunks) take work items, over the whole grid and over ranges that cut tiles"""
    opm, tab, p = table(key)
    grid = E.grid_for_model(opm, tab, num)
    n, cpt = grid.n_chunks, grid.chunks_per_tile
    for c0, c1 in ((0, n), (cpt//2, n - cpt//3)):
        grid_launch(oracle, key, grid, c0, c1, False, True, want_regime=want, sample=6)
    grid.close()


def wave_grid(key, num):
    opm, tab, p = table(key)
    fields, wvls = list(opm.optical_spec.field_of_view.fields), list(opm.seq_model.wvlns)
    args, kw = A.wavefront_grid_args(opm, tab, num, fields, wvls, opm.optical_spec.defocus.focus_shift)
    return E.PupilGrid(*args, device=0, **kw)


@pytest.mark.parametrize('key', ['long640+1', 'long640', 'long320'])
def test_opd_against_the_oracle(oracle, key):
    """opd of the unstaged general and the lean-at-budget instances (with and without summary):
    within 1e-12 mm of the oracle and >= 95 % bit-equal"""
    opm, tab, p = table(key)
    grid = wave_grid(key, 16)
    opts = _abi.make_opts(first_surf=1, last_surf=tab.n_ifc - 2, check_apertures=True)
    ref = oracle.trace_grid(grid.c_spec(), tab.descs, tab.n_by_wvl, 0, grid.n_rays, opts, n_threads=8,
                            wvls=tab.wvls)
    for summary in (False, True):
        r = launched(instance(p, 'grid', 0, summary, opd=True),
                     lambda: E.trace_grid(tab, grid, outputs=('status', 'opd'), summary=summary))
        torch.cuda.synchronize()
        st, opd = np_(r.status), np_(r.opd)
        assert (st == ref['status']).all()
        ok = (st == 0) & np.isfinite(ref['opd'])
        assert ok.sum() > grid.n_rays//4
        np.testing.assert_allclose(opd[ok], ref['opd'][ok], rtol=0, atol=1e-12)
        assert (opd[ok] == ref['opd'][ok]).mean() >= 0.95
    grid.close()


@pytest.mark.parametrize('key', ['long640+1', 'long256+1'])
def test_trace_grid_to_host_in_two_pieces(oracle, key):
    """rt_trace_grid_to_host, 2 pieces on an unstaged table: the aberrations equal rt_trace_grid's,
    the summary is the combine of the two pieces' restatements"""
    opm, tab, p = table(key)
    grid = E.grid_for_model(opm, tab, 16)               # one chunk per tile: per-chunk records
    n = grid.n_rays
    ref = E.trace_grid(tab, grid, outputs=('status', 'abr', 'op'), summary=False)
    h = torch.empty((2, n), dtype=torch.float64).pin_memory()
    summ, _ = E.trace_grid_to_host(tab, grid, h, pieces=2)
    torch.cuda.synchronize()
    st, abr, op = np_(ref.status), np_(ref.abr), np_(ref.op)
    hs, _ = E.decode_nan_status(h.numpy())
    assert (hs == st).all() and same_bits(h.numpy()[:, st == 0], abr[:, st == 0])
    check_rays(oracle, tab, grid, 0, grid.n_chunks, {'status': st, 'abr': abr, 'op': op})
    parts = []
    for a, b_ in ((0, grid.n_chunks//2), (grid.n_chunks//2, grid.n_chunks)):
        sh = S.Shape.of(grid, a, b_)
        assert regime(p, sh) == 'records'
        sl = slice(grid.first_ray_of_chunk(a), grid.first_ray_of_chunk(b_))
        parts.append(S.ordered_summary(sh, st[sl], abr[0, sl], abr[1, sl], op[sl], 'records'))
    if not DRY:                                      # (the dry-run engine's sums are exact)
        assert same_bits(np_(summ), S.combine(parts))
    grid.close()


# ---------------------------------------------------------------- rt_trace_grid_focus
def focus_planes(key, num, c0c1):
    """test_gpu_through_focus.check_planes on the table ``key``"""
    opm, tab, p = table(key)
    grid = E.grid_for_model(opm, tab, num, ref_img=None)
    wi = tab.wvl_index(opm.seq_model.central_wavelength())
    foc = TF.planes(opm)
    c0, c1 = c0c1(grid.n_chunks, grid.chunks_per_tile)
    ref = grid.chief_ref_focus(tab, wi, foc)
    summ = np_(launched(instance(p, 'focus'), lambda: E.trace_grid_focus(tab, grid, foc, c0, c1, ref_img=ref)))
    ref_h = np_(ref)
    for k, f in enumerate(foc):
        want = TF.single_focus_summary(opm, tab, num, f, ref_h[k], grid.n_wvls, c0, c1)
        TF.assert_same_summary(summ[k], want, (key, num, k, f))
    assert summ[:, :, 0].sum() > 0
    cpt = grid.chunks_per_tile
    grid.close()
    return cpt


@device_only
@pytest.mark.parametrize('key,num', [('long640+1', 16), ('long640+1', 48), ('long256+1', 48), ('long640', 48),
                                     ('long320', 48)])
def test_focus_planes_equal_single_focus_traces(key, num):
    focus_planes(key, num, lambda n, cpt: (0, n))
    focus_planes(key, num, lambda n, cpt: (3, n - 5))


@device_only
def test_focus_between_the_cta_counts_of_summary_and_focus_launch():
    """long360: the summary launch keeps one CTA per SM, the focus kernel two.  At 192^2 rays per
    tile (144 chunks) the single-focus trace takes work items; the focus trace must take them too,
    which only a range that cuts tiles shows"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cpt = focus_planes('long360', 192, lambda n, cpt: (cpt//2 + 3, n - cpt//3))
    assert sms*1 < cpt <= sms*2, (sms, cpt)


# ---------------------------------------------------------------- wavefront error, Zernike
def register(module, key, num):
    """put the table ``key`` into ``module``'s setup cache, so that its check_launch runs on it"""
    if (key, num) not in module._SETUP:
        opm, tab, p = table(key)
        fields, wvls = list(opm.optical_spec.field_of_view.fields), list(opm.seq_model.wvlns)
        module._SETUP[(key, num)] = (opm, tab, wave_grid(key, num), fields, wvls)


@device_only
@pytest.mark.parametrize('which', ['full', 'mid'])
@pytest.mark.parametrize('key', ['long640+1', 'long256+1', 'long640', 'long320', 'long256', 'long360'])
def test_wfe_records(key, which):
    register(WF, key, 33)
    p = table(key)[2]
    tab, grid = WF._SETUP[(key, 33)][1:3]
    c0, c1 = WF.chunk_range(grid, which)
    launched(instance(p, 'wfe'), lambda: E.trace_grid_wfe(tab, grid, c0, c1))
    WF.check_launch(key, 33, which)


@device_only
@pytest.mark.parametrize('key', ['long640+1', 'long320'])
def test_zernike_records(key):
    register(GZ, key, 33)
    for which in ('full', 'mid'):
        GZ.check_launch(key, 33, which, 16)


# ---------------------------------------------------------------- chief rays and aiming
@pytest.mark.parametrize('key', ['long640', 'long640+1'])
def test_chief_ref_against_the_oracle(oracle, key):
    """rt_grid_chief_ref through 640 interfaces: the image intercepts of the chief rays"""
    opm, tab, p = table(key)
    grid = E.grid_for_model(opm, tab, 4, ref_img=None)
    wi = tab.wvl_index(opm.seq_model.central_wavelength())
    out = torch.empty((grid.n_fields, 2), dtype=torch.float64, device='cuda')
    grid.chief_ref(tab, wi, out=out)
    torch.cuda.synchronize()
    recs, eprad, z_pupil = opm.optical_spec.grid_fields(opm.optical_spec.field_of_view.fields)
    g0 = E.PupilGridSpec(recs, [wi], [0.0], [0.0], eprad, z_pupil, apply_vignetting=False,
                         flip_z_dir=opm.seq_model.z_dir[0])
    ref = oracle.trace_grid(g0.c_spec(), tab.descs, tab.n_by_wvl, 0, g0.n_rays,
                            _abi.make_opts(first_surf=1, last_surf=tab.n_ifc - 2, check_apertures=False),
                            wvls=tab.wvls)
    assert (ref['status'] == 0).all()
    assert same_bits(np_(out), ref['last'][0:2].T)
    grid.close()


@device_only
def test_aim_through_hundreds_of_interfaces():
    """rt_grid_aim_chief on long640 (318 interfaces before the stop): the fixture's fields and a 7 x 7
    field grid against the restatement tests/aim_ref.py, bit for bit"""
    from test_gpu_field_map import device_aims
    from test_field_map import field_grid
    opm = LM.load('long640')
    assert opm.seq_model.stop_surface > 300
    for fields in (list(opm.optical_spec.field_of_view.fields), field_grid(opm, 7)):
        aim, term = device_aims(opm, fields)
        want, wterm, _ = AR.aim_fields(AR.oracle_stop_xy(opm, fields), len(fields), AR.aim_step(opm))
        assert np.array_equal(term, wterm)
        assert same_bits(aim, want)


# ---------------------------------------------------------------- what ran
REQUIRED = ['k_trace_bundle<false, false>', 'k_trace_bundle<true, false>',
            'k_trace_grid<false, false, false, false>', 'k_trace_grid<false, true, false, false>',
            'k_trace_grid<true, false, false, false>', 'k_trace_grid<true, true, false, false>',
            'k_trace_grid<false, false, false, true>', 'k_trace_grid<false, true, false, true>',
            'k_trace_grid_focus<false>', 'k_trace_grid_wfe<false>',
            'k_trace_grid_lean<0, true, false, false>', 'k_trace_grid_lean<0, true, false, true>',
            'k_trace_bundle_lean<2, false>', 'k_trace_bundle_lean<2, true>']


@device_only
def test_zz_every_instance_ran():
    """the ten instances only an unstaged table reaches, and the lean / lean POLY instances at the
    budget, were each launched and checked above"""
    if not SEEN:
        pytest.skip('no launch checked in this session')
    print('\nkernel instances launched on the long systems:')
    for name in sorted(SEEN):
        print(f'  {SEEN[name]:4d}  {name}')
    missing = [k for k in REQUIRED if k not in SEEN]
    assert not missing, missing
