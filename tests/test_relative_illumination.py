"""CPU: the sums of rt_grid_illumination (csrc/rt_illum.cuh through tests/hostsim) against the numpy
restatement engine.illumination_sums_host, the restatement against the closed-form projected solid
angle of a disk, and analyses.relative_illumination through the backend= seam with the oracle."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import aim_ref as AR
from conftest import ROOT, load_model
from rayoptics_b200 import _abi, analyses as A, engine as E
from rayoptics_b200.model import Field


def bits(v):
    return np.ascontiguousarray(v, dtype=np.float64).view(np.uint64).tolist()


class IllumBackend:
    """the backend= seam of relative_illumination: chief rays and grid directions traced by the oracle,
    aim points by the restatement of the device aiming (as test_field_map.py's AimingBackend)"""

    def __init__(self, opm):
        from test_analyses_vs_reference import OracleBackend
        self.be = OracleBackend(opm)
        self.aimed = []

    def chief_rays(self, opm, fields, wvls):
        return self.be.chief_rays(opm, fields, wvls)

    def aim_fields(self, opm, fields, wvl):
        x, _, _ = AR.restate(opm, fields, wvl)
        for k, f in enumerate(fields):
            f.aim_info = np.array([0.0 if f.x == 0.0 else x[k, 0], x[k, 1]])
        self.aimed += list(fields)
        return [f.aim_info for f in fields]

    def trace_directions(self, opm, spec, check_apertures):
        r = self.be.o.trace_grid(spec.c_spec(), self.be.descs, self.be.n_by_wvl, 0, spec.n_rays,
                                 self.be._opts(check_apertures), wvls=self.be.wvls)
        return {'status': r['status'], 'd': r['last'][3:6]}


# --- the integrator against the closed form ----------------------------------------------------------
def disk_rays(n, H, R):
    """rays from the point (H, 0, 0) through the point (R x, R y, 1) of a disk at unit distance, every
    grid point traced (status 0): the direction cosines L, M of each"""
    x = E.accumulated_steps(-1.0, 1.0, n)
    gx, gy = np.meshgrid(x, x, indexing='ij')
    vx, vy = R*gx - H, R*gy
    norm = np.sqrt(vx*vx + vy*vy + 1.0)
    return np.zeros((n, n), dtype=np.int32), vx/norm, vy/norm, x


def omega_exact(H, R):
    """the differential-to-parallel-disk view factor times pi"""
    return np.pi/2*(1 - (1 + H*H - R*R)/np.sqrt((1 + H*H + R*R)**2 - 4*R*R*H*H))


def test_closed_form_against_quadrature():
    from scipy import integrate
    for H, R in ((0.0, 0.3), (1.0, 1.0), (2.0, 0.05)):
        def f(v, u):
            vx, vy = R*u - H, R*v
            return R*R/(vx*vx + vy*vy + 1.0)**2           # |d(L, M)/d(u, v)| of disk_rays
        q, _ = integrate.dblquad(f, -1, 1, lambda u: -np.sqrt(1 - u*u), lambda u: np.sqrt(1 - u*u),
                                 epsabs=1e-14, epsrel=1e-13)
        assert abs(q/omega_exact(H, R) - 1) <= 1e-11, (H, R)


@pytest.mark.parametrize('n, tol_omega, tol_ri', [(32, 1e-2, 2e-2), (64, 4e-3, 7e-3), (128, 1e-3, 2e-3),
                                                  (256, 4e-4, 8e-4)])
def test_integrator_against_the_closed_form(n, tol_omega, tol_ri):
    worst_o = worst_ri = 0.0
    for R in (0.05, 0.3, 1.0):
        st, L, M, x = disk_rays(n, 0.0, R)
        rec0 = E.illumination_sums_host(st, L, M, x, x)
        om0 = np.pi*rec0[8]/rec0[6]
        for H in (0.0, 0.5, 1.0, 2.0):
            st, L, M, x = disk_rays(n, H, R)
            rec = E.illumination_sums_host(st, L, M, x, x)
            assert rec[5] == rec[6] and rec[7] == 0 and rec[8] == abs(rec[9])     # no fold, none isolated
            om = np.pi*rec[8]/rec[6]
            worst_o = max(worst_o, abs(om/omega_exact(H, R) - 1))
            worst_ri = max(worst_ri, abs((om/om0)/(omega_exact(H, R)/omega_exact(0.0, R)) - 1))
    print(f'n = {n}: largest |Omega/Omega_exact - 1| = {worst_o:.3g}, RI error {worst_ri:.3g}')
    assert worst_o <= tol_omega and worst_ri <= tol_ri


# --- the header compiled for the host, on oracle-traced grids ----------------------------------------
HEADER_MODELS = ['dblgauss', 'cellphone', 'rc', 'threemir', 'fisheye', 'relay_na', 'edge_stops']


def oracle_grid(opm, n):
    """(spec, status, d) of the start rays of grid_for_model(..., pupil_range=(-1, 1),
    apply_vignetting=False), apertures checked, traced by the oracle"""
    be = IllumBackend(opm)
    spec = E.grid_spec_for_model(opm, n, pupil_range=(-1.0, 1.0), apply_vignetting=False)
    r = be.trace_directions(opm, spec, True)
    return spec, r['status'], r['d']


def synthetic_tiles():
    """status patterns that take every branch: lone rays, pairs and full runs, and a tile with no
    ray at status 0"""
    rng = np.random.default_rng(7)
    out = []
    for n, p in ((2, 0.5), (3, 0.4), (9, 0.5), (33, 0.3), (33, 0.8)):
        st = np.where(rng.random((n, n)) < p, 0, rng.integers(1, 6, (n, n))).astype(np.int32)
        out.append((st, rng.standard_normal((n, n)), rng.standard_normal((n, n)), E.accumulated_steps(-1, 1, n)))
    out.append((np.full((4, 4), 3, dtype=np.int32), np.zeros((4, 4)), np.zeros((4, 4)), E.accumulated_steps(-1, 1, 4)))
    return out


def test_header_equals_the_restatement_bit_for_bit():
    from hostsim import illum_build as IB
    kinds = np.zeros(4, dtype=np.int64)
    isolated = tiles = 0
    for name in HEADER_MODELS:
        opm = load_model(name)
        for n in (2, 3, 33, 64):
            spec, status, d = oracle_grid(opm, n)
            per = n*n
            for t in range(spec.n_tiles):
                f = t//spec.n_wvls
                sl = slice(t*per, (t + 1)*per)
                args = (status[sl].reshape(n, n), d[0, sl].reshape(n, n), d[1, sl].reshape(n, n),
                        spec.pupil_x[f], spec.pupil_y[f])
                got, k = IB.illum_tile(*args)
                want = E.illumination_sums_host(*args)
                assert bits(got) == bits(want), (name, n, t)
                kinds += k
                isolated += int(got[7])
                tiles += 1
    print(f'{tiles} fixture tiles: central / forward / backward / none = {kinds.tolist()}, isolated {isolated}')
    for st, L, M, x in synthetic_tiles():
        got, k = IB.illum_tile(st, L, M, x, x)
        assert bits(got) == bits(E.illumination_sums_host(st, L, M, x, x))
        kinds += k
        isolated += int(got[7])
    assert (kinds > 0).all() and isolated > 0


def test_counts_of_the_record():
    rng = np.random.default_rng(3)
    n = 17
    st = rng.integers(-2, 7, (n, n)).astype(np.int32)
    st[rng.random((n, n)) < 0.5] = 0
    x = E.accumulated_steps(-1.0, 1.0, n)
    rec = E.illumination_sums_host(st, rng.standard_normal((n, n)), rng.standard_normal((n, n)), x, x)
    cls = np.where((st >= 0) & (st <= 3), st, 4).ravel()
    disk = x[:, None]**2 + x[None, :]**2 <= 1.0
    assert (rec[:5] == np.bincount(cls, minlength=5)[:5]).all()
    assert rec[5] == ((st == 0) & disk).sum() and rec[6] == disk.sum() and rec[:5].sum() == n*n


# --- analyses.relative_illumination through the backend seam -------------------------------------------
@pytest.mark.parametrize('name', ['dblgauss', 'cellphone'])
def test_reference_field_axis_and_polychromatic_ratio(name):
    opm = load_model(name)
    r = A.relative_illumination(opm, 32, backend=IllumBackend(opm))
    nf, nw = len(opm.optical_spec.field_of_view.fields), len(opm.seq_model.wvlns)
    assert r.ri.shape == (nf, nw) and r.chief_img.shape == (nf, nw, 2) and r.chief_dir.shape == (nf, nw, 3)
    assert r.ref_index == 0 and len(r.fields) == nf
    assert (r.ri[r.ref_index] == 1.0).all() and r.ri_poly[r.ref_index] == 1.0
    assert (r.cra[r.ref_index] == 0.0).all()                 # rotationally symmetric: the axis is the axis
    assert (r.cra[1:] > 0).all() and (r.ri[1:] < 1).all()
    want = (r.omega @ r.wts)/(r.omega[r.ref_index] @ r.wts)
    assert bits(r.ri_poly) == bits(want)
    np.testing.assert_allclose(r.omega, np.pi*r.record[:, 8].reshape(nf, nw)/r.n_disk, rtol=0, atol=0)
    np.testing.assert_allclose(r.f_number, 1/(2*r.n_img*np.sqrt(r.omega/np.pi)), rtol=1e-15)
    assert (np.abs(r.fold) < 1e-12).all() and (r.n_isolated == 0).all()
    assert (r.n_ok + r.n_missed + r.n_tir + r.n_blocked + r.n_other == 32*32).all()
    # the chief rays: the oracle's image segment
    full, _, _ = IllumBackend(opm).chief_rays(opm, r.fields, opm.seq_model.wvlns)
    assert bits(r.chief_img.reshape(-1, 2)) == bits(full[-1, 0:2].T)
    # on axis the effective F-number is the paraxial working F-number, to the grid's accuracy
    fod = opm['analysis_results']['parax_data'].fod
    ci = opm.seq_model.wvlns.index(opm.seq_model.central_wavelength())
    assert abs(r.f_number[0, ci]*2*abs(fod.img_na) - 1) <= 0.03


def test_num_fields_layout_and_the_added_axial_field():
    opm = load_model('cellphone')
    fov = opm.optical_spec.field_of_view
    be = IllumBackend(opm)
    r = A.relative_illumination(opm, 16, num_fields=5, backend=be)
    scale = fov.max_field()[0]/(fov.value if fov.is_relative and fov.value else 1.0)
    assert [f.x for f in r.fields] == [0.0]*5
    assert np.array_equal([f.y for f in r.fields], scale*np.linspace(0.0, 1.0, 5))
    assert be.aimed == r.fields and r.ref_index == 0 and r.ri.shape == (5, len(opm.seq_model.wvlns))
    assert (np.diff(r.ri_poly) < 0).all()                    # falls off towards the corner
    # fields without an axial one: an axial field is appended, aimed, and is the reference
    be = IllumBackend(opm)
    off = [Field(x=0.0, y=float(scale*0.5), fov=fov), Field(x=float(scale*0.3), y=float(scale*0.4), fov=fov)]
    be.aim_fields(opm, off, opm.optical_spec.spectral_region.central_wvl)
    r2 = A.relative_illumination(opm, 16, fields=off, backend=be)
    assert len(r2.fields) == 3 and r2.ref_index == 2 and r2.fields[2].x == 0 and r2.fields[2].y == 0
    assert be.aimed[-1] is r2.fields[2] and (r2.ri[2] == 1).all()
    np.testing.assert_array_equal(r2.ri[0], r.ri[2])         # the same point as num_fields' third


def test_argument_errors():
    opm = load_model('dblgauss')
    for n in (0, 1, 1025):
        with pytest.raises(ValueError, match='num_rays'):
            A.relative_illumination(opm, n, backend=IllumBackend(opm))
    with pytest.raises(ValueError, match='not both'):
        A.relative_illumination(opm, 8, fields=list(opm.optical_spec.field_of_view.fields), num_fields=3,
                                backend=IllumBackend(opm))
    # no axial field, and one cannot be aimed on the device (wide-angle fields, angular pupils)
    for name in ('fisheye', 'relay_na'):
        opm = load_model(name)
        off = [f for f in opm.optical_spec.field_of_view.fields if f.x != 0 or f.y != 0]
        with pytest.raises(ValueError, match='axial field'):
            A.relative_illumination(opm, 8, fields=off, table=object())
        with pytest.raises(NotImplementedError):
            A.relative_illumination(opm, 8, num_fields=3, table=object())


def test_angular_and_wide_models_with_their_own_fields():
    for name in ('fisheye', 'relay_na'):
        opm = load_model(name)
        r = A.relative_illumination(opm, 24, backend=IllumBackend(opm))
        assert r.ref_index == 0 and (r.ri[0] == 1).all() and np.isfinite(r.ri).all()


# --- ABI -----------------------------------------------------------------------------------------
def test_abi_export_and_constants():
    hdr = open(os.path.join(ROOT, 'include', 'b200rt.h')).read()
    declared = set(re.findall(r'\b(rt_[a-z0-9_]+)\s*\(', hdr))
    assert 'rt_grid_illumination' in declared and 'rt_grid_illumination' in _abi.EXPORTS
    assert re.search(r'#define RT_ILLUM_DOUBLES (\d+)', hdr).group(1) == str(_abi.RT_ILLUM_DOUBLES) == '10'
    assert re.search(r'#define RT_ILLUM_MAX_RAYS (\d+)', hdr).group(1) == str(_abi.RT_ILLUM_MAX_RAYS) == '1024'
    assert len(E.ILLUM_RECORD) == _abi.RT_ILLUM_DOUBLES
    assert _abi.RT_ABI_VERSION == 6


def test_abi_null_grid_without_a_device():
    lib = _abi.load_library()
    buf = (C.c_double*64)()
    st = (C.c_int32*64)()
    assert lib.rt_grid_illumination(None, st, buf, buf, buf, None) == -1
    assert 'grid' in lib.rt_last_error().decode()
