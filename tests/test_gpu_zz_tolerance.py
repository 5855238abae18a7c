"""rt_trace_grid_variants on the device: every variant's record against rt_trace_grid's summary on a
table of that variant alone and against tests/tol_sums.py fed that trace's rays (bit for bit); batch
ranges; the closed-form focus compensator against a real trace at the refocused plane; launch counts."""
import ctypes as C

import numpy as np
import pytest
import torch

import tol_sums as TS
from conftest import load_model
from rayoptics_b200 import _abi, analyses as A, engine as E, tolerance as TOL
from rayoptics_b200.table import SurfaceTable, describe_model

pytestmark = pytest.mark.gpu
T = TOL.Tolerance


def _tolerances(sm, n):
    """n tolerances of mixed kinds on the interfaces / gaps of sm"""
    n_ifc = len(sm.ifcs)
    kinds = ['radius', 'thickness', 'tilt_x', 'decenter_y', 'index', 'conic', 'tilt_y', 'decenter_x']
    out, i = [], 0
    while len(out) < n:
        k = kinds[i % len(kinds)]
        s = 1 + (i*5) % (n_ifc - 2)
        i += 1
        if k == 'thickness' and s > len(sm.gaps) - 1:
            continue
        if k == 'radius' and sm.ifcs[s].profile.cv == 0.0:
            continue
        if sm._tfrms_given is not None and k in ('thickness', 'tilt_x', 'tilt_y', 'decenter_x', 'decenter_y'):
            continue
        d = {'radius': 0.2, 'thickness': 0.02, 'index': 5e-4, 'conic': 0.02}.get(k, 0.01)
        out.append(T(k, s, d))
    return out


def _variant_sets(opm, k):
    sm = opm.seq_model
    tols = _tolerances(sm, max(1, (k - 1)//2))
    sets = [[]]
    for t in tols:
        sets += [[(t, t.delta)], [(t, -t.delta)]]
    return sets[:k]


def _check(name, num_rays, k):
    opm = load_model(name)
    sm = opm.seq_model
    d0, n0, wvls = describe_model(sm)
    var = [TOL.perturbed_descriptors(d0, n0, ch, sm) for ch in _variant_sets(opm, k)]
    tab0 = SurfaceTable(d0, n0, wvls)
    grid = E.grid_for_model(opm, tab0, num_rays)
    vs = E.VariantSet([v[0] for v in var], np.stack([v[1] for v in var]), wvls)
    rec = E.trace_grid_variants(vs, grid).cpu().numpy()
    shape = TS.Shape.of(grid)
    for v, (d, nb) in enumerate(var):
        tab = SurfaceTable(d, nb, wvls)
        r = E.trace_grid(tab, grid, outputs=('p', 'd', 'op', 'status', 'abr'))
        summ = r.summary.cpu().numpy()
        assert np.array_equal(rec[v, :, :16], summ, equal_nan=True), (name, v)
        st = r.status.cpu().numpy()
        ab, dd = r.abr.cpu().numpy(), r.d.cpu().numpy()
        ref = TS.record(shape, st, ab[0], ab[1], r.op.cpu().numpy(), dd[0], dd[1], dd[2])
        assert np.array_equal(rec[v, :, 16:], ref[:, 16:], equal_nan=True), (name, v)
        tab.close()
    return vs, grid, rec


@pytest.mark.parametrize('name', ['dblgauss', 'cellphone', 'threemir', 'relay_na', 'fisheye', 'diffractive'])
def test_records_every_model(name):
    _check(name, 32, 5)


@pytest.mark.parametrize('num_rays,k', [(8, 1), (8, 41), (64, 41), (256, 5)])
def test_records_sizes(num_rays, k):
    _check('dblgauss', num_rays, k)


def test_variant_ranges_give_the_same_records():
    vs, grid, rec = _check('dblgauss', 64, 41)
    lib = _abi.load_library()
    opts = _abi.make_opts(check_apertures=True, first_surf=1, last_surf=vs.n_ifc - 2)
    dev = torch.device('cuda', 0)
    out = torch.empty((41, grid.n_tiles, _abi.RT_TOL_DOUBLES), dtype=torch.float64, device=dev)
    scratch = torch.empty(lib.rt_grid_variants_scratch_bytes(grid.handle, 41)//8 + 1, dtype=torch.float64,
                          device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for a, b in ((0, 1), (1, 17), (17, 17), (17, 41)):
        _abi.check(lib.rt_trace_grid_variants(vs.handle, grid.handle, a, b, C.byref(opts),
                                              C.c_void_p(out[a].data_ptr()) if b > a else None,
                                              C.c_void_p(scratch.data_ptr()), stream))
    assert np.array_equal(out.cpu().numpy(), rec)
    batched = E.trace_grid_variants(vs, grid, cap=int(lib.rt_grid_variants_scratch_bytes(grid.handle, 3)))
    assert np.array_equal(batched.cpu().numpy(), rec)
    for a, b in ((-1, 3), (5, 42), (7, 6)):
        assert lib.rt_trace_grid_variants(vs.handle, grid.handle, a, b, C.byref(opts),
                                          C.c_void_p(out.data_ptr()), C.c_void_p(scratch.data_ptr()), stream) != 0
    assert lib.rt_trace_grid_variants(vs.handle, grid.handle, 0, 1, C.byref(opts), None,
                                      C.c_void_p(scratch.data_ptr()), stream) != 0


def test_focus_compensator_against_refocused_trace():
    opm = load_model('dblgauss')
    sm, osp = opm.seq_model, opm.optical_spec
    tols = [T('thickness', 4, 0.1), T('radius', 2, 1.0), T('tilt_x', 6, 0.1), T('index', 3, 2e-3)]
    s = A.tolerance_sensitivity(opm, tols, num_rays=32)
    res = s.result
    fields, wvls = list(osp.field_of_view.fields), list(sm.wvlns)
    region = osp.spectral_region
    ww = np.array([region.spectral_wts[list(region.wavelengths).index(w)] for w in wvls])
    fw = np.array([f.wt for f in fields])
    sets = [[]] + [[(t, sg*t.delta)] for t in tols for sg in (1.0, -1.0)]
    tab0 = SurfaceTable.from_model(sm)
    args, kw = E._grid_args(opm, sm.index_for_wavelength, 32, fields, wvls, None, (-1.0, 1.0), True)
    grid = E.PupilGrid(*args, **kw)
    ref = torch.empty((len(fields), 2), dtype=torch.float64, device='cuda')
    grid.chief_ref(tab0, sm.index_for_wavelength(sm.central_wavelength()), out=ref)
    nf, nw = len(fields), len(wvls)
    for v, ch in enumerate(sets):
        tab = SurfaceTable.from_model(TOL.perturbed_model(opm, ch).seq_model)
        summ = E.trace_grid_focus(tab, grid, [grid.foc + res.focus[v]], ref_img=ref[None].contiguous())
        sm_ = summ.cpu().numpy().reshape(nf, nw, 16)
        n = (sm_[..., 0]*ww).sum(1)
        x1, y1 = (sm_[..., 5]*ww).sum(1), (sm_[..., 6]*ww).sum(1)
        x2 = ((sm_[..., 7] + sm_[..., 8])*ww).sum(1)
        s2 = x2/n - (x1*x1 + y1*y1)/(n*n)
        m = np.sqrt((s2*fw).sum()/fw.sum())
        assert abs(m - res.merit[v]) <= 1e-9*m, (v, m, res.merit[v])


def test_launches_do_not_grow_with_tolerances():
    opm = load_model('dblgauss')
    tols = _tolerances(opm.seq_model, 12)
    A.tolerance_sensitivity(opm, tols[:2], num_rays=16)
    counts = []
    for k in (2, 12):
        torch.cuda.synchronize()
        c0 = E.launch_count()
        A.tolerance_sensitivity(opm, tols[:k], num_rays=16)
        counts.append(E.launch_count() - c0)
    assert counts[0] == counts[1]
