"""CPU: the sums of rt_grid_mtf (csrc/rt_mtf.cuh through tests/hostsim) against the restatement in
tests/mtf_sums.py, the restatement against exactly rounded sums, the physics of the OTF on synthetic
pupils, and analyses.mtf through the backend= seam with the oracle."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import mtf_sums as MS
from conftest import ROOT, load_model
from rayoptics_b200 import _abi, analyses as A, engine as E


def bits(v):
    return np.ascontiguousarray(v).view(np.uint64).tolist()


def random_pupil(n, seed, holes=True, scale=0.4):
    rng = np.random.default_rng(seed)
    m, x, y = MS.disk_mask(n, holes=holes, rng=rng)
    w = scale*rng.standard_normal((n, n)) + 0.7*x*x*y
    return MS.phasors(w, m), m


# --- the header compiled for the host ----------------------------------------------------------------
@pytest.mark.parametrize('holes', [False, True])
@pytest.mark.parametrize('n', [1, 2, 33, 64, 256])
def test_header_sums_equal_the_restatement_bit_for_bit(n, holes):
    from hostsim import mtf_build as MB
    P, _ = random_pupil(n, n + holes, holes)
    cx, cy, s = MB.mtf_sums(P)
    want = MS.sums(P)
    assert bits(cx) == bits(want[0]) and bits(cy) == bits(want[1])
    assert bits(np.array([s])) == bits(np.array([want[2]]))
    # the package's backend= sums are a third statement of the same order
    got = E.mtf_sums_host(P)
    assert bits(got[0]) == bits(want[0]) and bits(got[1]) == bits(want[1]) and got[2] == want[2]


def test_header_phasor_and_used_rule():
    from hostsim import mtf_build as MB
    rng = np.random.default_rng(3)
    n = 4000
    x, y = rng.uniform(-1.2, 1.2, (2, n))
    x[:4], y[:4] = [1.0, np.nextafter(1.0, 2), 0.6, -0.0], [0.0, 0.0, 0.8, -1.0]
    status = np.where(rng.random(n) < 0.8, 0, rng.integers(-2, 7, n)).astype(np.int32)
    opd = rng.standard_normal(n)*10.0**rng.integers(-6, 1, n)
    lam = 5.5e-4
    got = MB.pupil(status, opd, x, y, lam)
    used = (status == 0) & (x*x + y*y <= 1.0)
    assert used[0] == (status[0] == 0) and not used[1]
    assert (got[~used] == 0).all() and not np.signbit(got[~used].real).any()
    want = MS.phasors(opd/lam, used)
    assert np.abs(got - want).max() <= 1e-15


# --- the restatement -----------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 5, 33, 64])
def test_restatement_within_bound_of_exact_sums(n):
    P, _ = random_pupil(n, 10 + n)
    for axis in (0, 1):
        got = MS.autocorr(P, axis)
        ex, ab = MS.exact_autocorr(P, axis)
        for k in range(n):
            g = MS.gamma(MS.depth(n, k))
            assert abs(got[k].real - ex[k].real) <= g*ab[k, 0]
            assert abs(got[k].imag - ex[k].imag) <= g*ab[k, 1]


def test_plausible_mistakes_change_the_bits():
    n = 12
    P, _ = random_pupil(n, 5, holes=True, scale=0.8)
    good = [MS.autocorr(P, a) for a in (0, 1)]
    for kw in ({'reverse_lines': True}, {'fma': True}, {'conj_first': True}):
        for a in (0, 1):
            assert bits(MS.autocorr(P, a, **kw)) != bits(good[a]), (kw, a)
    assert bits(good[0]) != bits(good[1])                      # the axes are not interchangeable


def test_chain_is_sequential_from_positive_zero():
    rng = np.random.default_rng(4)
    v = rng.standard_normal((300, 3))*10.0**rng.integers(-8, 8, (300, 3))
    loop = np.zeros(3)
    for r in v:
        loop = loop + r
    assert bits(MS.chain(v)) == bits(loop)
    assert not np.signbit(MS.chain(np.full((3, 1), -0.0))).any()


# --- physics on synthetic pupils -----------------------------------------------------------------
@pytest.mark.parametrize('n', [2, 33, 64])
def test_zero_wavefront_gives_the_overlap_count(n):
    m, _, _ = MS.disk_mask(n, holes=True, rng=np.random.default_rng(n))
    P = np.where(m, 1.0 + 0.0j, 0.0j)
    cx, cy, s = E.mtf_sums_host(P)
    mi = m.astype(np.int64)
    for k in range(n):
        assert cx[k] == (mi[k:]*mi[:n - k]).sum() and cy[k] == (mi[:, k:]*mi[:, :n - k]).sum()
    assert s == m.sum()


def test_disk_mtf_against_the_analytic_curve():
    """The used rays of a 256-point grid over [-1, 1] sample the disk; the overlap of two sampled
    disks differs from that of the disks by the samples the two rims cross, about 2 x 2 pi/delta
    against the area pi/delta^2: a bound of 4 delta (delta = 2/255) on the MTF"""
    n = 256
    m, _, _ = MS.disk_mask(n)
    cx, cy, _ = E.mtf_sums_host(np.where(m, 1.0 + 0.0j, 0.0j))
    delta = 2.0/(n - 1)
    v = np.clip(np.arange(n)*delta/2.0, 0, 1)
    ideal = 2/np.pi*(np.arccos(v) - v*np.sqrt(1 - v*v))
    err = max(np.abs(cx.real/cx[0].real - ideal).max(), np.abs(cy.real/cy[0].real - ideal).max())
    print(f'disk at {n}^2: max |MTF - analytic| = {err:.3g} (bound {4*delta:.3g})')
    assert err <= 4*delta


def test_tilt_leaves_the_mtf_unchanged():
    n = 64
    m, x, y = MS.disk_mask(n, holes=True, rng=np.random.default_rng(1))
    w = 0.1*np.sin(3*x) + 0.05*y*y
    base = E.mtf_sums_host(MS.phasors(w, m))
    tilted = E.mtf_sums_host(MS.phasors(w + 2.3*x - 1.7*y, m))
    for a in (0, 1):
        np.testing.assert_allclose(np.abs(tilted[a]/tilted[a][0].real), np.abs(base[a]/base[a][0].real),
                                   rtol=0, atol=1e-12)


@pytest.mark.parametrize('seed', [1, 2, 3])
def test_aberrations_never_raise_the_mtf(seed):
    n = 48
    P, m = random_pupil(n, seed, holes=True, scale=0.3)
    cx, cy, _ = E.mtf_sums_host(P)
    fx, fy, _ = E.mtf_sums_host(np.where(m, 1.0 + 0.0j, 0.0j))
    assert (np.abs(cx/cx[0].real) <= fx.real/fx[0].real + 1e-12).all()
    assert (np.abs(cy/cy[0].real) <= fy.real/fy[0].real + 1e-12).all()


@pytest.mark.parametrize('n', [1, 17, 64])
def test_autocorrelation_equals_the_fft_route(n):
    """independent of the sum order: the axis slices of ifft2(|fft2(P padded to 2n)|^2)"""
    P, m = random_pupil(n, 40 + n)
    cx, cy, _ = E.mtf_sums_host(P)
    F = np.fft.fft2(P, s=(2*n, 2*n))
    ac = np.fft.ifft2(np.abs(F)**2)
    tol = 1e-12*max(m.sum(), 1)
    assert np.abs(cx - ac[:n, 0]).max() <= tol and np.abs(cy - ac[0, :n]).max() <= tol


# --- analyses.mtf through the backend seam -----------------------------------------------------------
def _oracle(name):
    from test_analyses_vs_reference import OracleBackend
    opm = load_model(name)
    return opm, OracleBackend(opm)


@pytest.mark.parametrize('name', ['dblgauss', 'cellphone'])
def test_n_used_and_counts_equal_zernike_fit(name):
    opm, be = _oracle(name)
    r = A.mtf(opm, 24, backend=be)
    z = A.zernike_fit(opm, 24, 4, backend=be)
    for k in ('n_used', 'n_ok', 'n_missed', 'n_tir', 'n_blocked', 'n_other'):
        assert (getattr(r, k) == getattr(z, k)).all(), k
    assert r.otf_x.shape == (len(opm.optical_spec.field_of_view.fields), len(opm.seq_model.wvlns), 24)
    assert (r.otf_x[..., 0] == 1).all() and (r.otf_y[..., 0] == 1).all()
    np.testing.assert_array_equal(r.mtf_x, np.abs(r.otf_x))


def test_axial_strehl_against_marechal():
    """On axis, where the piston-removed RMS over the used rays is below 0.07 waves: the Strehl ratio
    |<exp(i phi)>|^2 against exp(-sigma^2), sigma = 2 pi rms.  Their series differ first at fourth
    order, by sigma^4 (kappa/12 - 1/4) with kappa the kurtosis of phi; the test allows sigma^4/2
    (kappa up to 9).  The double Gauss's axial wavefront is above 0.7 waves RMS at every focus, so
    no tile of it qualifies; the Ritchey-Chretien is perfect on axis and is defocused to 0.006 ...
    0.065 waves."""
    checked = 0
    for name, focs in (('dblgauss', (0.0, 0.05)), ('rc', (0.0, -0.01, 0.03, -0.1, 0.1))):
        opm, be = _oracle(name)
        fld = [opm.optical_spec.field_of_view.fields[0]]
        for foc in focs:
            r = A.mtf(opm, 48, fields=fld, foc=foc, backend=be)
            z = A.zernike_fit(opm, 48, 4, fields=fld, foc=foc, backend=be)
            for wi in range(r.n_wvls):
                rms = z.rms[0, wi]
                if rms < 0.07:
                    s2 = (2*np.pi*rms)**2
                    assert abs(r.strehl[0, wi] - np.exp(-s2)) <= s2*s2/2 + 1e-12, (name, foc, wi, rms)
                    checked += 1
    assert checked >= 5


def test_axial_cutoff_is_two_na_over_lambda():
    opm, be = _oracle('dblgauss')
    fod = opm['analysis_results']['parax_data'].fod
    r = A.mtf(opm, 16, fields=[opm.optical_spec.field_of_view.fields[0]], backend=be)
    for wi, wl in enumerate(opm.seq_model.wvlns):
        want = 2*abs(fod.img_na)/opm.nm_to_sys_units(wl)
        assert abs(r.cutoff[0, wi]/want - 1) <= 0.02
        np.testing.assert_allclose(r.freq_x[0, wi, -1], r.cutoff[0, wi], rtol=1e-12)     # bbox [-1, 1]


def test_interpolated_otf_and_polychromatic_combine():
    opm, be = _oracle('dblgauss')
    freqs = np.array([0.0, 25.0, 80.0, 400.0, 2000.0])
    r = A.mtf(opm, 24, freqs=freqs, polychromatic=True, backend=be)
    assert r.otf_x_at.shape == (r.n_fields, r.n_wvls, len(freqs)) and r.poly_x.shape == (r.n_fields, len(freqs))
    assert (r.otf_x_at[..., 0] == 1).all()
    assert (r.otf_x_at[..., -1] == 0).all()                     # past every cutoff
    t = (0, 1)
    want = np.interp(25.0, r.freq_y[t], r.otf_y[t].real) + 1j*np.interp(25.0, r.freq_y[t], r.otf_y[t].imag)
    assert r.otf_y_at[t][1] == want
    # every wavelength is referred to the central wavelength's chief-ray image point
    ci = opm.seq_model.wvlns.index(opm.seq_model.central_wavelength())
    assert (r.ref_img == r.ref_img[:, ci:ci + 1]).all()
    np.testing.assert_allclose(r.poly_x, A.polychromatic_mtf(r.otf_x_at, r.wts), rtol=0, atol=0)


def test_polychromatic_combine_on_synthetic_otfs():
    k = np.linspace(0, 1, 7)
    o1 = np.exp(-k)*np.exp(1j*k)
    o2 = np.exp(-2*k)*np.exp(-1j*k)
    otf = np.stack([o1, o2, o1])[None]                         # [1, 3, 7]
    got = A.polychromatic_mtf(otf, [1.0, 2.0, 1.0])
    np.testing.assert_allclose(got[0], np.abs(2*o1 + 2*o2)/4, rtol=1e-15)
    np.testing.assert_allclose(A.polychromatic_mtf(otf[:, :1], [3.0])[0], np.abs(o1), rtol=1e-15)


def test_frequencies_and_the_infinite_reference():
    wave = np.zeros((2, 1, _abi.RT_WAVE_DOUBLES))
    wave[:, 0, 20], wave[:, 0, 21] = [-50.0, 7.0], [1.0, 0.0]
    pupil = np.array([np.linspace(-1, 1, 5), np.linspace(-0.5, 1, 5)])
    freq, cutoff = A.mtf_frequencies(pupil, wave, np.array([1e-3, 1e-3]), 10.0)
    np.testing.assert_allclose(freq[0], np.arange(5)*0.5*10/(1e-3*50), rtol=1e-15)
    np.testing.assert_allclose(cutoff[0], 2*10/(1e-3*50), rtol=1e-15)
    assert np.isnan(freq[1]).all() and np.isnan(cutoff[1])
    at = A.otf_at([0.0, 1.0], freq, np.ones((2, 5), complex), cutoff)
    assert (at[0] == 1).all() and np.isnan(at[1]).all()


def test_mtf_argument_checks():
    opm = load_model('singlet')
    for kw in ({'num_rays': 0}, {'num_rays': 1025}, {'polychromatic': True}, {'freqs': [-1.0]},
               {'freqs': [np.nan]}):
        with pytest.raises(ValueError):
            A.mtf(opm, **kw)
    wl = [w for w in opm.seq_model.wvlns if w != opm.seq_model.central_wavelength()]
    if wl:
        with pytest.raises(ValueError, match='central'):
            A.mtf(opm, 8, wvls=wl, freqs=[0.0], polychromatic=True)


def test_wavefront_grid_args_default_is_unchanged():
    opm, be = _oracle('dblgauss')
    fields, wvls = opm.optical_spec.field_of_view.fields, opm.seq_model.wvlns
    a0, k0 = A.wavefront_grid_args(opm, None, 8, fields, wvls, 0.0, backend=be)
    a1, k1 = A.wavefront_grid_args(opm, None, 8, fields, wvls, 0.0, backend=be, ref_wvl_for_image_pt=None)
    assert bits(k0['wave']) == bits(k1['wave']) and bits(k0['ref_img']) == bits(k1['ref_img'])


# --- ABI -----------------------------------------------------------------------------------------
def test_abi_exports_are_declared():
    hdr = open(os.path.join(ROOT, 'include', 'b200rt.h')).read()
    declared = set(re.findall(r'\b(rt_[a-z0-9_]+)\s*\(', hdr))
    for name in ('rt_grid_pupil_function', 'rt_grid_mtf'):
        assert name in declared and name in _abi.EXPORTS
    assert re.search(r'#define RT_MTF_MAX_RAYS (\d+)', hdr).group(1) == str(_abi.RT_MTF_MAX_RAYS) == '1024'
    assert re.search(r'#define RT_MTF_DOUBLES (\d+)', hdr).group(1) == str(_abi.RT_MTF_DOUBLES)
    assert len(E.MTF_RECORD) == _abi.RT_MTF_DOUBLES


def test_abi_null_grid_without_a_device():
    lib = _abi.load_library()
    buf = (C.c_double*64)()
    st = (C.c_int32*64)()
    assert lib.rt_grid_pupil_function(None, st, buf, buf, buf, buf, None) == -1
    assert 'grid' in lib.rt_last_error().decode()
    assert lib.rt_grid_mtf(None, st, buf, buf, buf, buf, buf, None) == -1
    assert 'grid' in lib.rt_last_error().decode()
