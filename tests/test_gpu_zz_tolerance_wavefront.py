"""Wavefront tolerancing on the device: rt_variants_wave's records, reference points and statuses against
waveabr.setup_tiles on a table of each variant alone; rt_trace_grid_variants_wfe's records against
rt_trace_grid_wfe's summary for that variant alone (bit for bit); variant ranges and batches; argument
checks; the analysis merit against wavefront_error of the perturbed model; launch counts."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_model
from rayoptics_b200 import _abi, analyses as A, engine as E, tolerance as TOL, waveabr as WA
from rayoptics_b200.table import SurfaceTable, describe_model
from test_tolerance_wavefront import every_kind

pytestmark = pytest.mark.gpu
T = TOL.Tolerance


def _sets(sm, k):
    sets = [[]]
    tols = every_kind(sm)
    i = 0
    while len(sets) < k:
        t = tols[i % len(tols)]
        sg = 1.0 if (i//len(tols)) % 2 == 0 else -1.0
        scale = 1.0 + 0.5*(i//(2*len(tols)))
        sets += [[(t, sg*scale*t.delta)], [(t, -sg*scale*t.delta)]]
        i += 1
    return sets[:k]


def _setup(name, num_rays, k):
    opm = load_model(name)
    sm, osp = opm.seq_model, opm.optical_spec
    fields, wvls = list(osp.field_of_view.fields), list(sm.wvlns)
    foc = osp.defocus.focus_shift
    d0, n0, all_w = describe_model(sm)
    sets = _sets(sm, k)
    var = [TOL.perturbed_descriptors(d0, n0, ch, sm) for ch in sets]
    tab0 = SurfaceTable(d0, n0, all_w)
    args, kw = A._wavefront_grid_args(opm, tab0, num_rays, fields, wvls, foc, None, None)
    grid = E.PupilGrid(*args, **kw)
    vs = E.VariantSet([v[0] for v in var], np.stack([v[1] for v in var]), all_w)
    fod = opm['analysis_results']['parax_data'].fod
    parax = (fod.exp_dist, abs(fod.n_obj), abs(fod.n_img))
    return opm, sets, var, all_w, (fields, wvls, foc), args, kw, grid, vs, parax


def _check(name, num_rays, k, per_variant=None):
    opm, sets, var, all_w, (fields, wvls, foc), args, kw, grid, vs, parax = _setup(name, num_rays, k)
    wave, ref, st = vs.wave(grid, parax)
    rec = E.trace_grid_variants_wfe(vs, grid, wave).cpu().numpy()
    wave, ref, st = wave.cpu().numpy(), ref.cpu().numpy(), st.cpu().numpy()
    assert (st == 0).all(), name
    for v in (range(len(sets)) if per_variant is None else per_variant):
        d, nb = var[v]
        pm = TOL.perturbed_model(opm, sets[v])
        tab = SurfaceTable(d, nb, all_w)
        w_h, r_h, _ = WA.setup_tiles(pm, tab, fields, wvls, foc)
        assert np.array_equal(wave[v], w_h.reshape(-1, _abi.RT_WAVE_DOUBLES)), (name, v)
        assert np.array_equal(ref[v], r_h.reshape(-1, 2)), (name, v)
        g = E.PupilGrid(*args, **dict(kw, wave=w_h, ref_img=r_h))
        summ = E.trace_grid_wfe(tab, g).cpu().numpy()
        assert np.array_equal(rec[v], summ, equal_nan=True), (name, v)
        g.close()
        tab.close()
    return vs, grid, wave, rec, parax


@pytest.mark.parametrize('name', ['dblgauss', 'cellphone', 'relay_na', 'fisheye', 'diffractive', 'telecentric'])
def test_records_every_model(name):
    _check(name, 32, 2*len(every_kind(load_model(name).seq_model)) + 1)


@pytest.mark.parametrize('num_rays,k', [(8, 1), (8, 41), (64, 41), (256, 1), (256, 41)])
def test_records_sizes(num_rays, k):
    _check('dblgauss', num_rays, k, None if num_rays < 256 or k == 1 else (0, 1, 17, 40))


def test_variant_ranges_and_batches_give_the_same_records():
    vs, grid, wave, rec, parax = _check('dblgauss', 64, 41, per_variant=(0,))
    lib = _abi.load_library()
    opts = _abi.make_opts(check_apertures=True, first_surf=1, last_surf=vs.n_ifc - 2)
    dev = torch.device('cuda', 0)
    wv = torch.as_tensor(wave, device=dev)
    out = torch.empty((41, grid.n_tiles, _abi.RT_WFE_DOUBLES), dtype=torch.float64, device=dev)
    scratch = torch.empty(lib.rt_grid_variants_wfe_scratch_bytes(grid.handle, 41)//8 + 1, dtype=torch.float64,
                          device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for a, b in ((0, 1), (1, 17), (17, 17), (17, 41)):
        _abi.check(lib.rt_trace_grid_variants_wfe(vs.handle, grid.handle, a, b, C.byref(opts),
                                                  C.c_void_p(wv[a].data_ptr()) if b > a else None,
                                                  C.c_void_p(out[a].data_ptr()) if b > a else None,
                                                  C.c_void_p(scratch.data_ptr()), stream))
    assert np.array_equal(out.cpu().numpy(), rec, equal_nan=True)
    cap = int(lib.rt_grid_variants_wfe_scratch_bytes(grid.handle, 3))
    batched = E.trace_grid_variants_wfe(vs, grid, wv, cap=cap)
    assert np.array_equal(batched.cpu().numpy(), rec, equal_nan=True)
    part = E.trace_grid_variants_wfe(vs, grid, wv[5:30].contiguous(), var_begin=5, var_end=30, cap=cap)
    assert np.array_equal(part.cpu().numpy(), rec[5:30], equal_nan=True)
    w3, r3, s3 = vs.wave(grid, parax, var_begin=12, var_end=20)
    full = vs.wave(grid, parax)
    assert torch.equal(w3, full[0][12:20]) and torch.equal(r3, full[1][12:20]) and torch.equal(s3, full[2][12:20])
    # argument checks: errors before any device work
    p3 = np.zeros(3)
    pp = p3.ctypes.data_as(_abi.c_double_p)
    ptr = C.c_void_p(out.data_ptr())
    for a, b in ((-1, 3), (5, 42), (7, 6)):
        assert lib.rt_trace_grid_variants_wfe(vs.handle, grid.handle, a, b, C.byref(opts), C.c_void_p(wv.data_ptr()),
                                              ptr, C.c_void_p(scratch.data_ptr()), stream) != 0
        assert lib.rt_variants_wave(vs.handle, grid.handle, a, b, pp, ptr, ptr, ptr, stream) != 0
    assert lib.rt_trace_grid_variants_wfe(vs.handle, grid.handle, 0, 1, C.byref(opts), None, ptr,
                                          C.c_void_p(scratch.data_ptr()), stream) == _abi_err('INVALID')
    assert lib.rt_trace_grid_variants_wfe(vs.handle, grid.handle, 0, 1, C.byref(opts), C.c_void_p(wv.data_ptr()),
                                          None, C.c_void_p(scratch.data_ptr()), stream) == _abi_err('INVALID')
    assert lib.rt_variants_wave(vs.handle, grid.handle, 0, 1, None, ptr, ptr, ptr, stream) == _abi_err('INVALID')
    assert lib.rt_variants_wave(vs.handle, grid.handle, 0, 1, pp, None, ptr, ptr, stream) == _abi_err('INVALID')


def _abi_err(name):
    return {'INVALID': -1, 'UNSUPPORTED': -3}[name]      # enum rt_error, include/b200rt.h


def test_decentered_image_gap_is_refused():
    opm = load_model('dblgauss')
    sm = opm.seq_model
    n = len(sm.ifcs)
    d0, n0, all_w = describe_model(sm)
    sets = [[], [(T('decenter_y', n - 2, 0.01), 0.01)], []]
    var = [TOL.perturbed_descriptors(d0, n0, ch, sm) for ch in sets]
    tab0 = SurfaceTable(d0, n0, all_w)
    args, kw = A._wavefront_grid_args(opm, tab0, 8, list(opm.optical_spec.field_of_view.fields), list(sm.wvlns),
                                      0.0, None, None)
    grid = E.PupilGrid(*args, **kw)
    vs = E.VariantSet([v[0] for v in var], np.stack([v[1] for v in var]), all_w)
    c0 = E.launch_count()
    with pytest.raises(_abi.EngineError):
        vs.wave(grid, (0.0, 1.0, 1.0))
    wave = torch.zeros((3, grid.n_tiles, _abi.RT_WAVE_DOUBLES), dtype=torch.float64, device='cuda')
    with pytest.raises(_abi.EngineError):
        E.trace_grid_variants_wfe(vs, grid, wave)
    lib = _abi.load_library()
    p3 = np.zeros(3)
    ptr = C.c_void_p(wave.data_ptr())
    assert lib.rt_variants_wave(vs.handle, grid.handle, 1, 2, p3.ctypes.data_as(_abi.c_double_p), ptr, ptr, ptr,
                                None) == _abi_err('UNSUPPORTED')
    assert E.launch_count() == c0
    w, _, st = vs.wave(grid, (0.0, 1.0, 1.0), var_begin=2, var_end=3)       # the others are fine
    assert (st.cpu().numpy() == 0).all()
    E.trace_grid_variants_wfe(vs, grid, w, var_begin=2, var_end=3)
    three = load_model('threemir')
    d3, n3, w3 = describe_model(three.seq_model)
    tab3 = SurfaceTable(d3, n3, w3)
    a3, k3 = A._wavefront_grid_args(three, tab3, 8, list(three.optical_spec.field_of_view.fields),
                                    list(three.seq_model.wvlns), 0.0, None, None)
    g3 = E.PupilGrid(*a3, **k3)
    vs3 = E.VariantSet([d3], n3[None], w3)
    with pytest.raises(_abi.EngineError):
        vs3.wave(g3, (0.0, 1.0, 1.0))


@pytest.mark.parametrize('compensate_focus', (True, False))
def test_sensitivity_merit_equals_wavefront_error_of_the_perturbed_models(compensate_focus):
    opm = load_model('dblgauss')
    sm, osp = opm.seq_model, opm.optical_spec
    n = len(sm.ifcs)
    tols = [T('radius', 2, 1.0), T('thickness', len(sm.gaps) - 1, 0.05), T('tilt_x', 6, 0.05), T('index', 3, 2e-3),
            T('decenter_y', n - 3, 0.02)]
    s = A.tolerance_sensitivity(opm, tols, criterion='wavefront', compensate_focus=compensate_focus)
    region = osp.spectral_region
    ww = [region.spectral_wts[list(region.wavelengths).index(w)] for w in sm.wvlns]
    fw = [f.wt for f in osp.field_of_view.fields]
    sets = [[]] + [[(t, sg*t.delta)] for t in tols for sg in (1.0, -1.0)]
    key = 'rms_focus' if compensate_focus else 'rms_tilt'
    for v, ch in enumerate(sets):
        we = A.wavefront_error(TOL.perturbed_model(opm, ch), num_rays=32)
        rms = getattr(we, key)
        assert np.array_equal(s.result.rms[v], rms), (v, ch)
        m, sig = A.wave_merit_of(rms[None], ww, fw)
        assert s.result.merit[v] == m[0], (v, s.result.merit[v], m[0])
        assert np.array_equal(s.result.sigma[v], sig[0])
    mc = A.tolerance_monte_carlo(opm, tols, num_trials=50, num_rays=16, criterion='wavefront')
    assert np.isfinite(mc.merit).all() and mc.percentiles[98] >= mc.percentiles[50]


def test_launches_do_not_grow_with_tolerances():
    opm = load_model('dblgauss')
    tols = every_kind(opm.seq_model)
    A.tolerance_sensitivity(opm, tols[:2], num_rays=16, criterion='wavefront')
    counts = []
    for k in (2, len(tols)):
        torch.cuda.synchronize()
        c0 = E.launch_count()
        A.tolerance_sensitivity(opm, tols[:k], num_rays=16, criterion='wavefront')
        counts.append(E.launch_count() - c0)
    assert counts[0] == counts[1] == 3
