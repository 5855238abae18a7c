"""Chief-ray aiming on the H100 (k_aim_chief, rt_grid_aim_chief) and analyses.field_map.

- Device aim points and termination codes equal the restatement tests/aim_ref.py (oracle traces) bit
  for bit: every 'epd' fixture's own fields, 1, 7 x 7 and 33 x 33 field grids, points beyond the
  field where rays fail.  hybrid (phase elements) gets a stated bound instead.
- On-meridian fields equal vigcalc.aim_all_fields_batched (CUDA bundles) bit for bit, off-meridian
  fields meet the quality bound of DESIGN.md section 4.
- One launch per call, grid records unchanged, argument errors before any device work.
- CODE V's listing from device aims; field_map against zernike_fit and the CPU backend run.
"""
import numpy as np
import pytest

import aim_ref as AR
from conftest import load_model
from test_field_map import (AimingBackend, EPD_FIXTURES, bits, central_index, check_codev, codev_chief_rays,
                            field_grid, residual)
from rayoptics_b200 import _abi, analyses as A, engine as E, vigcalc as V
from rayoptics_b200.opticalspec import grid_fields_of

pytestmark = pytest.mark.gpu

# phase elements: the device's phase arithmetic is held to the pow() tolerance of DESIGN.md section 2a
BOUNDED = {'hybrid'}


@pytest.fixture(scope='module', autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')


def aim_grid(opm, fields, tab):
    sm = opm.seq_model
    recs, eprad, z_pupil = grid_fields_of(opm, fields)
    return E.PupilGrid(recs, [central_index(opm)], [0.0], [0.0], eprad, z_pupil, apply_vignetting=False,
                       flip_z_dir=sm.z_dir[0], device=tab.device)


def device_aims(opm, fields, h=None, max_iter=30):
    tab = A._table_for(opm)
    grid = aim_grid(opm, fields, tab)
    n0 = E.launch_count()
    aim, term = E.aim_chief_rays(tab, grid, opm.seq_model.stop_surface, central_index(opm),
                                 AR.aim_step(opm) if h is None else h, 1e-13, max_iter)
    assert E.launch_count() - n0 == 1
    out = aim.cpu().numpy(), term.cpu().numpy()
    grid.close()
    return out


def device_cases():
    out = [(name, name, lambda opm: list(opm.optical_spec.field_of_view.fields), {}) for name in EPD_FIXTURES]
    out += [(f'dblgauss {n}x{n}', 'dblgauss', lambda opm, n=n: field_grid(opm, n), {}) for n in (1, 7, 33)]
    out += [('zoom52 33x33', 'zoom52', lambda opm: field_grid(opm, 33), {}),
            ('dblgauss 4x', 'dblgauss', lambda opm: field_grid(opm, 7, 4.0), {}),
            ('triplet 2x', 'triplet', lambda opm: field_grid(opm, 7, 2.0), {}),
            ('dblgauss max_iter 1', 'dblgauss', lambda opm: field_grid(opm, 3), dict(max_iter=1)),
            ('dblgauss h 1e-300', 'dblgauss', lambda opm: field_grid(opm, 3), dict(h=1e-300)),
            ('dblgauss h 100', 'dblgauss', lambda opm: field_grid(opm, 3), dict(h=100.0))]
    return out


@pytest.mark.parametrize('case', device_cases(), ids=lambda c: c[0])
def test_device_aims_equal_the_restatement(case):
    label, name, make, kw = case
    opm = load_model(name)
    fields = make(opm)
    aim, term = device_aims(opm, fields, kw.get('h'), kw.get('max_iter', 30))
    want, wterm, _ = AR.aim_fields(AR.oracle_stop_xy(opm, fields), len(fields), kw.get('h', AR.aim_step(opm)),
                                   max_iter=kw.get('max_iter', 30))
    assert np.array_equal(term, wterm)
    if name in BOUNDED:
        assert np.abs(aim - want).max() <= 1e-12
    else:
        assert np.array_equal(bits(aim), bits(want))
    print(f'{label}: {len(fields)} fields, codes {np.bincount(term, minlength=6).tolist()}')


@pytest.mark.parametrize('name,grid', [(n, None) for n in EPD_FIXTURES] + [('dblgauss', 9), ('threemir', 5)])
def test_device_aims_against_the_host_aiming(name, grid):
    opm = load_model(name)
    fov = opm.optical_spec.field_of_view
    if grid is not None:
        fov.fields = field_grid(opm, grid)
    fields = list(fov.fields)
    host = np.array(V.aim_all_fields_batched(opm), dtype=np.float64)
    dev = np.array(V.aim_fields_on_device(opm, fields), dtype=np.float64)
    on = np.array([f.x == 0.0 for f in fields])
    if name in BOUNDED:
        assert np.abs(dev[on] - host[on]).max() <= 1e-12
    else:
        assert np.array_equal(bits(dev[on]), bits(host[on]))
    off = ~on
    if off.any():
        sub = [fields[i] for i in np.nonzero(off)[0]]
        assert (residual(opm, sub, dev[off]) <= 2*residual(opm, sub, host[off]) + 1e-9).all()
        assert np.abs(dev[off] - host[off]).max() <= 1e-4


def test_grid_records_unchanged_and_errors_before_any_device_work():
    import torch
    lib = _abi.load_library()
    opm = load_model('dblgauss')
    fields = list(opm.optical_spec.field_of_view.fields)
    tab = A._table_for(opm)
    grid = aim_grid(opm, fields, tab)
    before = E.trace_grid(tab, grid, outputs=('p', 'd'), summary=False).p.cpu().numpy()
    E.aim_chief_rays(tab, grid, opm.seq_model.stop_surface, central_index(opm), AR.aim_step(opm))
    after = E.trace_grid(tab, grid, outputs=('p', 'd'), summary=False).p.cpu().numpy()
    assert np.array_equal(bits(before), bits(after))
    aim = torch.full((len(fields), 2), float('nan'), dtype=torch.float64, device='cuda')
    term = torch.full((len(fields),), -7, dtype=torch.int32, device='cuda')
    stop, wi, h = opm.seq_model.stop_surface, central_index(opm), AR.aim_step(opm)

    def call(t=tab.handle, g=grid.handle, s=stop, w=wi, hh=h, tol=1e-13, it=30, a=aim):
        return lib.rt_grid_aim_chief(t, g, s, w, hh, tol, it, E._ptr(a), E._ptr(term), None)
    others = []
    for name in ('fisheye', 'relay_na'):                       # wide-angle fields, an angular pupil
        m = load_model(name)
        t2 = A._table_for(m)
        others.append((m, t2, aim_grid(m, list(m.optical_spec.field_of_view.fields), t2)))
    torch.cuda.synchronize()
    n0 = E.launch_count()
    for kw in (dict(s=0), dict(s=tab.n_ifc - 1), dict(s=-1), dict(w=-1), dict(w=len(opm.seq_model.wvlns)),
               dict(hh=0.0), dict(hh=float('nan')), dict(tol=0.0), dict(tol=float('inf')), dict(it=-1),
               dict(a=None), dict(t=None), dict(g=None)):
        assert call(**kw) == -1, kw                            # RT_ERR_INVALID
    for m, t2, g2 in others:
        assert g2.pupil_kind != _abi.PUPIL_EPD
        assert lib.rt_grid_aim_chief(t2.handle, g2.handle, m.seq_model.stop_surface, 0, 1e-4, 1e-13, 30,
                                     E._ptr(aim), E._ptr(term), None) == -3       # RT_ERR_UNSUPPORTED
        assert 'epd' in lib.rt_last_error().decode()
        with pytest.raises(NotImplementedError):
            V.aim_fields_on_device(m, list(m.optical_spec.field_of_view.fields))
        g2.close()
    torch.cuda.synchronize()
    assert E.launch_count() == n0
    assert torch.isnan(aim).all() and (term == -7).all()
    assert call(it=0) == 0 and E.launch_count() == n0 + 1          # max_iter 0: the first ray only
    assert (term.cpu().numpy() == AR.MAX_ITER).all() and (aim.cpu().numpy() == 0.0).all()
    grid.close()


def test_device_aims_reproduce_the_codev_listing():
    opm = load_model('dblgauss')

    def aims_of(opm, fields):
        return np.array(V.aim_fields_on_device(opm, fields))
    kat, rays = codev_chief_rays(opm, aims_of)
    check_codev(kat, rays)


def test_field_map_equals_zernike_fit_and_the_cpu_run():
    opm = load_model('dblgauss')
    n, nr, terms = 9, 32, 37
    fm = A.field_map(opm, n, nr, terms)
    assert fm.valid.sum() == fm.traced.sum() == 49
    vi, vj = np.nonzero(fm.valid)
    fov = opm.optical_spec.field_of_view
    from rayoptics_b200.model import Field
    kept = [Field(x=float(fm.field_x[i, j]), y=float(fm.field_y[i, j]), fov=fov) for i, j in zip(vi, vj)]
    V.aim_fields_on_device(opm, kept)
    assert np.array_equal(bits(np.array([f.aim_info for f in kept])), bits(fm.aim[vi, vj]))
    zf = A.zernike_fit(opm, nr, terms, fields=kept)
    for k in ('coef', 'rms', 'rms_residual', 'pv', 'ref_img'):
        assert np.array_equal(bits(getattr(fm.zernike, k)), bits(getattr(zf, k))), k
    assert np.array_equal(bits(fm.coef[vi, vj]), bits(zf.coef))
    cpu = A.field_map(opm, n, nr, terms, backend=AimingBackend(opm))
    assert np.array_equal(cpu.valid, fm.valid)
    assert np.array_equal(bits(cpu.aim[vi, vj]), bits(fm.aim[vi, vj]))
    assert np.array_equal(bits(cpu.img[vi, vj]), bits(fm.img[vi, vj]))
    scale = np.abs(cpu.coef[vi, vj]).max(axis=-1, keepdims=True)
    assert (np.abs(cpu.coef[vi, vj] - fm.coef[vi, vj]) <= 1e-8*scale).all()
    np.testing.assert_allclose(fm.rms[vi, vj], cpu.rms[vi, vj], rtol=1e-9)
    np.testing.assert_array_equal(fm.distortion[vi, vj], cpu.distortion[vi, vj])
