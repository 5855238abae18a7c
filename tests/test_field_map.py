"""Chief-ray aiming on the device (csrc/rt_aim.cuh, rt_grid_aim_chief) and analyses.field_map, on CPU.

- rt_aim.cuh compiled for the host (tests/hostsim/aim.cpp) equals the numpy restatement
  tests/aim_ref.py driven by oracle traces, bit for bit: aim points, termination codes and Newton
  steps, on the own fields of every 'epd' fixture, 9 x 9 field grids and points beyond the field.
- The restatement against vigcalc.aim_all_fields_batched (np.linalg.solve) on the oracle: bit for bit
  on the meridian, within the quality bound of DESIGN.md section 4 elsewhere.
- The aimed chief rays of the double Gauss against CODE V's own listing
  (tests/golden/codev_dblgauss_chief.json).
- field_map through its backend= seam, and the ABI argument checks that need no device.
"""
import collections
import ctypes as C
import json
import os

import numpy as np
import pytest

import aim_ref as AR
from conftest import GOLDEN, load_model
from rayoptics_b200 import _abi, analyses as A, engine as E, table as T, vigcalc as V
from rayoptics_b200.model import Field
from rayoptics_b200.opticalspec import grid_fields_of

EPD_FIXTURES = ['dblgauss', 'triplet', 'rc', 'evenasph', 'cellphone', 'cellphone_even', 'zoom52', 'telecentric',
                'threemir', 'hybrid']


def central_index(opm):
    return opm.seq_model.index_for_wavelength(opm.optical_spec.spectral_region.central_wvl)


def aim_spec(opm, fields):
    """the rt_grid_spec aim_fields_on_device builds (kept alive by the returned PupilGridSpec)"""
    sm = opm.seq_model
    recs, eprad, z_pupil = grid_fields_of(opm, fields)
    return E.PupilGridSpec(recs, [central_index(opm)], [0.0], [0.0], eprad, z_pupil, apply_vignetting=False,
                           flip_z_dir=sm.z_dir[0])


def hostsim_aims(opm, fields, h=None, tol=1e-13, max_iter=30):
    from hostsim import aim_build as AB
    descs, n_by_wvl, wvls = T.describe_model(opm.seq_model)
    spec = aim_spec(opm, fields)
    return AB.aim_chief(descs, n_by_wvl, wvls, spec.c_spec(), opm.seq_model.stop_surface, central_index(opm),
                        AR.aim_step(opm) if h is None else h, tol, max_iter)


def field_grid(opm, n, factor=1.0):
    """n x n Field objects over [-factor, factor]^2 of the maximum field (x outer, y inner)"""
    fov = opm.optical_spec.field_of_view
    s = factor*fov.max_field()[0]/(fov.value if fov.is_relative and fov.value else 1.0)
    u = np.linspace(-1.0, 1.0, n)
    return [Field(x=float(s*a), y=float(s*b), fov=fov) for a in u for b in u]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def assert_same(got, want):
    (a, t, i), (b, u, j) = got, want
    assert np.array_equal(bits(a), bits(b))
    assert np.array_equal(t, u) and np.array_equal(i, j)


def with_x_rule(aims, fields):
    x = np.array(aims, dtype=np.float64, copy=True)
    for k, f in enumerate(fields):
        if f.x == 0.0:
            x[k, 0] = 0.0
    return x


# --- the device source on the host against the restatement ---------------------------------------
def cases():
    """(label, model name, fields factory, keyword arguments) of the bit-for-bit comparison"""
    out = [(name, name, lambda opm: list(opm.optical_spec.field_of_view.fields), {}) for name in EPD_FIXTURES]
    out += [(f'{name} 9x9', name, lambda opm: field_grid(opm, 9), {}) for name in ('dblgauss', 'zoom52')]
    out += [(f'{name} 1.5x', name, lambda opm: field_grid(opm, 7, 1.5), {}) for name in ('dblgauss', 'zoom52',
                                                                                          'triplet', 'cellphone')]
    # beyond the field the first rays and difference rays miss surfaces (apertures are not checked,
    # so 1.5x the field still traces): triplet from 2x, the double Gauss at 4x has both
    out += [('triplet 2x', 'triplet', lambda opm: field_grid(opm, 7, 2.0), {}),
            ('dblgauss 4x', 'dblgauss', lambda opm: field_grid(opm, 7, 4.0), {})]
    # constructed: one Newton step allowed (max_iter); h = 1e-300, so small that every difference
    # ray is the base ray again: J = 0, a zero pivot (singular); h = 100 mm: every difference ray
    # misses a surface
    out += [('dblgauss max_iter 1', 'dblgauss', lambda opm: field_grid(opm, 3), dict(max_iter=1)),
            ('dblgauss h 1e-300', 'dblgauss', lambda opm: field_grid(opm, 3), dict(h=1e-300)),
            ('dblgauss h 100', 'dblgauss', lambda opm: field_grid(opm, 3), dict(h=100.0))]
    return out


def test_device_source_equals_the_restatement_bit_for_bit():
    seen = collections.Counter()
    for label, name, make, kw in cases():
        opm = load_model(name)
        fields = make(opm)
        got = hostsim_aims(opm, fields, h=kw.get('h'), max_iter=kw.get('max_iter', 30))
        want = AR.aim_fields(AR.oracle_stop_xy(opm, fields), len(fields), kw.get('h', AR.aim_step(opm)),
                             max_iter=kw.get('max_iter', 30))
        assert_same(got, want)
        dist = collections.Counter(AR.TERM_NAMES[t] for t in got[1])
        seen.update(dist)
        print(f'{label}: {len(fields)} fields, {dict(dist)}, Newton steps {got[2].min()}-{got[2].max()}')
    assert set(seen) == set(AR.TERM_NAMES), seen


def test_first_and_difference_ray_failures_leave_the_aim_where_it_was():
    opm = load_model('dblgauss')
    fields = field_grid(opm, 7, 4.0)
    aim, term, iters = hostsim_aims(opm, fields)
    first = term == AR.FIRST_FAILED
    assert first.any() and (term == AR.DIFF_FAILED).any()
    assert np.array_equal(bits(aim[first]), np.zeros((first.sum(), 2), np.float64).view(np.uint64))
    assert (iters[first] == 0).all()


# --- the restatement against the host aiming ------------------------------------------------------
def residual(opm, fields, aims):
    return np.abs(AR.oracle_stop_xy(opm, fields)(list(range(len(fields))), aims)).max(axis=1)


@pytest.mark.parametrize('name,grid', [(n, None) for n in EPD_FIXTURES] + [('dblgauss', 9), ('zoom52', 9),
                                                                          ('threemir', 5)])
def test_restatement_against_the_host_aiming(name, grid):
    from test_trace_drivers import oracle_bundle_fn
    opm = load_model(name)
    fov = opm.optical_spec.field_of_view
    if grid is not None:
        fov.fields = field_grid(opm, grid)
    fields = list(fov.fields)
    x, term, _ = AR.restate(opm, fields)
    mine = with_x_rule(x, fields)
    host = np.array(V.aim_all_fields_batched(opm, oracle_bundle_fn(opm)), dtype=np.float64)
    on = np.array([f.x == 0.0 for f in fields])
    assert np.array_equal(bits(mine[on]), bits(host[on])), name
    off = ~on & (term != AR.FIRST_FAILED)
    if off.any():
        r_mine, r_host = residual(opm, [fields[i] for i in np.nonzero(off)[0]], mine[off]), \
            residual(opm, [fields[i] for i in np.nonzero(off)[0]], host[off])
        assert (r_mine <= 2*r_host + 1e-9).all()
        assert np.abs(mine[off] - host[off]).max() <= 1e-4
    print(f'{name}{"" if grid is None else f" {grid}x{grid}"}: on-meridian {on.sum()} identical, '
          f'off-meridian {off.sum()} (identical {int((bits(mine[off]) == bits(host[off])).all(axis=1).sum())}); '
          f'{dict(collections.Counter(AR.TERM_NAMES[t] for t in term))}')
    if name in ('dblgauss', 'zoom52'):          # objects at 1e10-1e11 mm: the noise floor ends the iteration
        assert (term[np.array([f.x != 0.0 or f.y != 0.0 for f in fields])] == AR.NO_STEP).all()


def test_restatement_reproduces_the_stored_aim_points():
    """the .roa aim points of the double Gauss (the reference's own iteration) to 8 digits"""
    opm = load_model('dblgauss')
    fields = list(opm.optical_spec.field_of_view.fields)
    stored = np.array([np.asarray(f.aim_info, dtype=float) for f in fields])
    x, term, iters = AR.restate(opm, fields)
    np.testing.assert_allclose(with_x_rule(x, fields), stored, rtol=0, atol=1e-8)
    assert list(term) == [AR.CONVERGED, AR.NO_STEP, AR.NO_STEP] and iters[2] == 4


# --- against CODE V's listing ---------------------------------------------------------------------
def codev_chief_rays(opm, aims_of):
    """(listing ray, traced whole ray [n_ifc, 10]) of the double Gauss at 10 and 14 degrees, aimed by
    ``aims_of(opm, fields) -> [n, 2]``"""
    from oracle import rt_oracle
    kat = json.load(open(os.path.join(GOLDEN, 'codev_dblgauss_chief.json')))
    fov = opm.optical_spec.field_of_view
    fields = [Field(x=0.0, y=r['field_deg'], fov=fov) for r in kat['rays']]
    aims = aims_of(opm, fields)
    for f, a in zip(fields, aims):
        f.aim_info = np.array(a, dtype=float)
    sm = opm.seq_model
    descs, n_by_wvl, wvls = T.describe_model(sm)
    recs, eprad, z_pupil = grid_fields_of(opm, fields)
    spec = E.PupilGridSpec(recs, [central_index(opm)], [0.0], [0.0], eprad, z_pupil, apply_vignetting=False,
                           flip_z_dir=sm.z_dir[0])
    p, d, wv, _ = rt_oracle.grid_start_rays(spec.c_spec(), 0, spec.n_rays)
    r = rt_oracle.trace_bundle(descs, n_by_wvl, p, d, wv, _abi.make_opts(first_surf=1, last_surf=len(descs) - 2),
                               want_full=True, wvls=wvls)
    assert (r['status'] == 0).all()
    return kat, [(ray, r['full'][:, :, k]) for k, ray in enumerate(kat['rays'])]


def check_codev(kat, rays):
    for ray, full in rays:
        lis = np.array(ray['xyz'])
        got = full[1:12, 0:3]
        gap = np.abs(got - lis).max(axis=0)
        assert gap.max() < kat['abs_tol'], gap
        img = full[-1, 1]
        assert abs(img - ray['img_y']) < kat['img_abs_tol'], img
        print(f"{ray['field_deg']} deg: |gap| x {gap[0]:.2g}  y {gap[1]:.2g}  z {gap[2]:.2g}, image {img:.7f}")


def test_aimed_chief_rays_reproduce_the_codev_listing():
    opm = load_model('dblgauss')
    kat, rays = codev_chief_rays(opm, lambda opm, fields: with_x_rule(AR.restate(opm, fields)[0], fields))
    check_codev(kat, rays)


# --- field_map through the backend seam ------------------------------------------------------------
class AimingBackend:
    """the zernike_fit seam of test_analyses_vs_reference plus the restatement's aim points"""

    def __init__(self, opm, drop=()):
        from test_analyses_vs_reference import OracleBackend
        self.be, self.drop, self.aimed = OracleBackend(opm), set(drop), None

    def aim_fields(self, opm, fields, wvl):
        x, _, _ = AR.restate(opm, fields, wvl)
        x = with_x_rule(x, fields)
        for k, f in enumerate(fields):
            f.aim_info = x[k].copy()
        self.aimed = list(fields)
        return [f.aim_info for f in fields]

    def chief_rays(self, opm, fields, wvls):
        full, op, status = self.be.chief_rays(opm, fields, wvls)
        status = np.array(status).reshape(len(fields), len(wvls))
        for k, f in enumerate(fields):       # a point whose chief ray is made to miss at one wavelength
            if (f.x, f.y) in self.drop:
                status[k, -1] = _abi.RAY_MISSED
        return full, op, status.ravel()

    def trace_tile(self, *args):
        return self.be.trace_tile(*args)


def test_field_map_layout_and_results():
    opm = load_model('dblgauss')
    n, nw, terms = 7, len(opm.seq_model.wvlns), 9
    fmax = opm.optical_spec.field_of_view.max_field()[0]
    u = np.linspace(-1.0, 1.0, n)
    dropped = (float(fmax*u[2]), float(fmax*u[4]))
    be = AimingBackend(opm, drop={dropped})
    fm = A.field_map(opm, n, 16, terms, backend=be)
    assert np.array_equal(fm.field_x, np.repeat(fmax*u[:, None], n, axis=1))
    assert np.array_equal(fm.field_y, np.repeat(fmax*u[None, :], n, axis=0))
    traced = np.hypot(*np.meshgrid(u, u, indexing='ij')) <= 1.0
    assert np.array_equal(fm.traced, traced) and len(be.aimed) == traced.sum()
    want_valid = traced.copy()
    want_valid[2, 4] = False
    assert np.array_equal(fm.valid, want_valid)
    assert all(f.vux == f.vlx == f.vuy == f.vly == 0.0 for f in be.aimed)
    assert np.isnan(fm.aim[~traced]).all() and np.isfinite(fm.aim[traced]).all()
    for a in (fm.img, fm.coef, fm.rms, fm.rms_residual, fm.pv, fm.distortion):
        assert np.isnan(a[~fm.valid]).all()
    assert fm.coef.shape == (n, n, nw, terms) and fm.img.shape == (n, n, nw, 2)
    # the result is zernike_fit's on the kept, aimed fields
    kept = [f for f in be.aimed if (f.x, f.y) != dropped]
    zf = A.zernike_fit(opm, 16, terms, fields=kept, backend=be)
    vi, vj = np.nonzero(fm.valid)
    assert np.array_equal(bits(fm.coef[vi, vj]), bits(zf.coef))
    assert np.array_equal(bits(fm.img[vi, vj]), bits(zf.ref_img))
    for k in ('rms', 'rms_residual', 'pv'):
        assert np.array_equal(bits(getattr(fm, k)[vi, vj]), bits(getattr(zf, k)))
    assert np.array_equal(bits(fm.zernike.coef), bits(zf.coef))
    # distortion: the formula in numpy on the oracle's chief rays
    fod = opm.optical_spec.fod
    from rayoptics_b200.firstorder import HT
    for i, j in zip(vi, vj):
        ax, ay = np.deg2rad(fm.field_x[i, j]), np.deg2rad(fm.field_y[i, j])
        slope = np.array([np.tan(ax), np.tan(ay)/np.cos(ax)])
        par = fod.pr_ray[-1][HT]*slope/fod.pr_slp0
        np.testing.assert_allclose(fm.parax_img[i, j], par, rtol=1e-14, atol=1e-14)
        for w in range(nw):
            if fm.field_x[i, j] == fm.field_y[i, j] == 0.0:
                assert np.isnan(fm.distortion[i, j, w])
                continue
            want = 100*(np.hypot(*fm.img[i, j, w]) - np.hypot(*par))/np.hypot(*par)
            np.testing.assert_allclose(fm.distortion[i, j, w], want, rtol=1e-12)


def test_double_gauss_distortion_is_barrel_growing_to_the_edge():
    opm = load_model('dblgauss')
    n = 9
    fm = A.field_map(opm, n, 12, 4, backend=AimingBackend(opm))
    c = n//2
    wc = opm.optical_spec.spectral_region.reference_wvl
    assert np.isnan(fm.distortion[c, c]).all()
    r = np.hypot(fm.field_x, fm.field_y)
    d = fm.distortion[..., wc]
    ok = fm.valid & (r > 0)
    assert (d[ok] < 0).all()
    order = np.argsort(r[ok], kind='stable')
    rs, ds = r[ok][order], d[ok][order]
    assert (np.diff(np.abs(ds))[np.diff(rs) > 1e-9] > 0).all()
    assert abs(d[c, -1] - (-1.038)) < 1e-3           # 14 degrees: 24.588738 against 24.846681
    assert fm.valid.sum() == 49 and np.isnan(fm.distortion[0, 0]).all()


def test_field_map_without_points_and_the_host_fallback_errors():
    opm = load_model('fisheye')
    with pytest.raises(NotImplementedError, match='aim_all_fields_batched'):
        V.aim_fields_on_device(opm, list(opm.optical_spec.field_of_view.fields))
    opm = load_model('relay_na')
    with pytest.raises(NotImplementedError, match='aim_all_fields_batched'):
        V.aim_fields_on_device(opm, list(opm.optical_spec.field_of_view.fields))
    opm = load_model('dblgauss')
    opm.seq_model.stop_surface = None              # floating stop: zeros, no table, no launch
    fields = field_grid(opm, 3)
    aims = V.aim_fields_on_device(opm, fields, table=object())
    assert all(np.array_equal(a, [0.0, 0.0]) for a in aims) and fields[4].aim_info is aims[4]


def test_paraxial_image_points_of_other_field_specifications_are_nan():
    for name in ('rc', 'cellphone', 'fisheye'):
        opm = load_model(name)
        assert np.isnan(A.paraxial_image_points(opm, [0.0, 0.1], [0.2, 0.3])).all()
    opm = load_model('exotic')                         # object heights: linear in the height
    p = A.paraxial_image_points(opm, [0.0, 3.0], [6.0, 0.0])
    from rayoptics_b200.firstorder import HT
    h = opm.optical_spec.fod.pr_ray[-1][HT]
    np.testing.assert_allclose(p, [[0.0, h], [h/2, 0.0]], rtol=1e-15)


# --- ABI ---------------------------------------------------------------------------------------------
def test_abi_arguments_checked_without_a_device():
    """the checks that need no handle contents; stop, wvl_idx and the pupil kind are checked in
    tests/test_gpu_field_map.py on real handles"""
    import re
    from conftest import ROOT
    hdr = open(os.path.join(ROOT, 'include', 'b200rt.h')).read()
    assert 'rt_grid_aim_chief' in re.findall(r'\b(rt_[a-z0-9_]+)\s*\(', hdr) and 'rt_grid_aim_chief' in _abi.EXPORTS
    names = re.findall(r'(RT_AIM_[A-Z_]+) = (\d)', hdr)
    assert [int(v) for _, v in names] == list(range(6)) and len(AR.TERM_NAMES) == 6
    lib = _abi.load_library()
    fake = C.c_void_p(1)
    aim = (C.c_double*8)()
    term = (C.c_int32*4)()
    call = lambda t, g, h=1e-4, tol=1e-13, it=30, a=aim: lib.rt_grid_aim_chief(t, g, 6, 0, h, tol, it, a, term,  # noqa: E731
                                                                               None)
    assert call(None, fake) == -1 and call(fake, None) == -1
    assert call(fake, fake, a=None) == -1 and 'aim_out' in lib.rt_last_error().decode()
    for h in (0.0, -1e-4, float('inf'), float('nan')):
        assert call(fake, fake, h=h) == -1 and ' h ' in lib.rt_last_error().decode()
    for tol in (0.0, -1.0, float('inf'), float('nan')):
        assert call(fake, fake, tol=tol) == -1 and 'tol' in lib.rt_last_error().decode()
    assert call(fake, fake, it=-1) == -1 and 'max_iter' in lib.rt_last_error().decode()
