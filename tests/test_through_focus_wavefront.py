"""CPU: the OPD at many reference spheres (csrc/rt_refocus.cuh through tests/hostsim) against the
reference's rapid-refocus split (waveabr.wave_abr_pre_calc / wave_abr_calc) on the golden OPD fixtures,
the per-plane sphere records against setup_tiles, the shift subset of the MTF interpolation, and
analyses.through_focus_wavefront through its backend= seam against per-plane zernike_fit / mtf."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, load_model
from test_analyses_vs_reference import OracleBackend
from rayoptics_b200 import _abi, analyses as A, engine as E, table as T, waveabr as W

FOCS = [0.0, 0.02, -0.02, 0.1, -0.1, 1.0, -1.0]


def bits(v):
    return np.ascontiguousarray(v, dtype=np.float64).view(np.uint64).tolist()


class RefocusBackend(OracleBackend):
    """OracleBackend with the whole rays the host refocus route needs"""

    def trace_rays(self, opt_model, spec, check_apertures):
        p, d, wv, _ = self.o.grid_start_rays(spec.c_spec(), 0, spec.n_rays)
        r = self.o.trace_bundle(self.descs, self.n_by_wvl, p, d, wv, self._opts(check_apertures), want_full=True,
                                wvls=self.wvls)
        return r['full'], r['op'], r['status']


def load_opd(name):
    z = np.load(os.path.join(GOLDEN, 'vectors', name + '_opd.npz'))
    return {k: z[k] for k in z.files}


# --- the split, compiled for the host, on the golden fixtures -------------------------------------
@pytest.mark.parametrize('name', ['dblgauss', 'triplet', 'rc', 'cellphone', 'telecentric'])
def test_header_split_equals_the_reference_refocus(oracle, name):
    from hostsim import refocus_build as RB, build as HS
    opm = load_model(name)
    osp, sm = opm.optical_spec, opm.seq_model
    fields, wvls = list(osp.fov.fields), list(sm.wvlns)
    v = load_opd(name)
    be = RefocusBackend(opm)
    wave, _, spheres, pkgs = W.setup_tiles_focus(opm, None, fields, wvls, FOCS, chief_tracer=be.chief_rays)
    nw = len(wvls)
    # plane 0 is foc = 0: the fixture's own records
    assert bits(wave[0].reshape(-1, _abi.RT_WAVE_DOUBLES)) == bits(v['wave'])
    descs, n_by_wvl, _ = T.describe_model(sm)
    n_ifc = len(descs)
    opts = _abi.make_opts(first_surf=1, last_surf=n_ifc - 2, check_apertures=True)
    r = oracle.trace_bundle(descs, n_by_wvl, v['p0'], v['d0'], v['wvl_idx'], opts, want_full=True)
    assert (r['status'] == v['status']).all()
    fod = opm['analysis_results']['parax_data'].fod
    n_bits = n_all = n_inf = 0
    for k in np.nonzero(v['status'] == 0)[0]:
        t = int(v['tile'][k])
        fi, wi = divmod(t, nw)
        full = r['full'][:, :, k]
        got = RB.refocus(v['wave'][t], full, r['op'][k], spheres[:, fi, wi])
        ray = [[full[i, 0:3], full[i, 3:6], float(full[i, 6]), full[i, 7:10]] for i in range(n_ifc)]
        ray_pkg = (ray, float(r['op'][k]), wvls[wi])
        crp = pkgs[0][fi][wi][0]
        pre = W.wave_abr_pre_calc(fod, fields[fi], wvls[wi], 0.0, ray_pkg, crp, pkgs[0][fi][wi][1])
        inf = v['wave'][t, 21] == 0.0
        for p, foc in enumerate(FOCS):
            rs = pkgs[p][fi][wi][1]
            want = W.wave_abr_calc(fod, fields[fi], wvls[wi], foc, ray_pkg, crp, pre, rs)
            exact = inf
            if not inf:
                F = rs[1].dot(pre[3]) - pre[3].dot(pre[1])/rs[2]
                exact = F**2 == F*F
            if exact:
                assert got[p] == want, (k, foc)
            assert abs(got[p] - want) <= 1e-12, (k, foc)
            n_bits += got[p] == want
            n_all += 1
        n_inf += inf
        if not inf:
            # the tile's own sphere: the single-focus epilogue wave_opd, bit for bit
            own = HS.wave_opd(v['wave'][t], full[1, 0:3], full[0, 3:6], full[n_ifc - 2, 0:3],
                              full[n_ifc - 2, 3:6], full[n_ifc - 1, 0:3], full[n_ifc - 1, 3:6], r['op'][k])
            assert got[0] == own, k
    assert n_bits >= 0.95*n_all
    if name == 'telecentric':
        assert n_inf > 100


# --- the sphere records -----------------------------------------------------------------------------
@pytest.mark.parametrize('name, kw', [
    ('dblgauss', {}),
    ('dblgauss', {'image_pt_2d': np.array([0.01, -0.02]), 'image_delta': np.array([0.003, 0.001])}),
    ('dblgauss', {'image_delta': np.array([0.0, 0.004])}),
    ('cellphone', {'ref_wvl_for_image_pt': 'central'}),
    ('telecentric', {}),
])
def test_sphere_records_equal_setup_tiles(name, kw):
    opm = load_model(name)
    osp, sm = opm.optical_spec, opm.seq_model
    fields, wvls = list(osp.fov.fields), list(sm.wvlns)
    kw = dict(kw)
    if kw.get('ref_wvl_for_image_pt') == 'central':
        kw['ref_wvl_for_image_pt'] = sm.central_wavelength()
    be = RefocusBackend(opm)
    wave, ref_img, spheres, _ = W.setup_tiles_focus(opm, None, fields, wvls, FOCS, chief_tracer=be.chief_rays, **kw)
    for p, foc in enumerate(FOCS):
        w1, r1, pk1 = W.setup_tiles(opm, None, fields, wvls, foc, chief_tracer=be.chief_rays, **kw)
        assert bits(wave[p]) == bits(w1) and bits(ref_img[p]) == bits(r1)
        for fi in range(len(fields)):
            for wi in range(len(wvls)):
                image_pt, ref_dir, radius, _ = pk1[fi][wi][1]
                S = spheres[p, fi, wi]
                assert bits(S[0:3]) == bits(ref_dir) and bits(S[5:8]) == bits(image_pt)
                assert bits(S[3:4]) == bits([radius]) and S[4] == w1[fi, wi, 21]
                if w1[fi, wi, 21] != 0.0:                          # finite: the wave record's own sphere
                    assert bits(S[0:5]) == bits(w1[fi, wi, 17:22])
    # the focus-independent columns do not move
    fin = wave[0, ..., 21] != 0.0
    cols = list(range(17)) + [22, 23]
    assert bits(wave[:, fin][..., cols]) == bits(np.broadcast_to(wave[0, fin][..., cols], wave[:, fin][..., cols].shape))


def test_mixed_variants_are_refused(monkeypatch):
    """a tile whose sphere is finite at one focus and infinite at another cannot share one pre-calc"""
    opm = load_model('dblgauss')
    fields, wvls = list(opm.optical_spec.fov.fields), list(opm.seq_model.wvlns)
    be = RefocusBackend(opm)
    real = W.wave_record
    calls = {'n': 0}

    def flip(opt_model, crp, rs):
        calls['n'] += 1
        w = real(opt_model, crp, rs)
        if rs[0][2] > 0.5:                                # the plane at foc = 1
            w[21] = 0.0
        return w
    monkeypatch.setattr(W, 'wave_record', flip)
    with pytest.raises(ValueError, match='finite'):
        W.setup_tiles_focus(opm, None, fields, wvls, [0.0, 1.0], chief_tracer=be.chief_rays)
    assert calls['n'] > 0


# --- the shift subset of the MTF interpolation ------------------------------------------------------
def test_shift_subset_gives_the_same_interpolation_bits():
    rng = np.random.default_rng(7)
    n, nt = 64, 4
    scale = np.array([37.3, 12.9, np.nan, 251.0])
    delta = np.array([2/63, 1.7/63, 2/63, 0.9/63])
    freq = np.arange(n)[None, :]*delta[:, None]*scale[:, None]
    cutoff = 2*scale
    acf = rng.standard_normal((nt, n)) + 1j*rng.standard_normal((nt, n))
    acf[:, 0] = np.abs(acf[:, 0]) + 5
    otf = acf/acf[:, :1].real
    nodes = [freq[0, 5], freq[1, 17], freq[3, 40], freq[0, -1], freq[1, -1]]
    past = [freq[0, -1]*1.001, freq[3, -1] + 1.0, cutoff[1]*0.999, cutoff[0]*1.5, 1e9]
    mids = list(rng.uniform(0, freq[3, -1], 40)) + [0.0, np.nextafter(freq[0, 5], 0), np.nextafter(freq[0, 5], 1e9)]
    freqs = np.array(nodes + past + mids)
    S = A.otf_shift_set(freqs, freq)
    assert S[0] == 0 and (np.diff(S) > 0).all() and len(S) < n
    sub = acf[:, S]/acf[:, S][:, :1].real
    got = A.otf_at(freqs, freq[:, S], sub, cutoff)
    want = A.otf_at(freqs, freq, otf, cutoff)
    assert bits(got.view(np.float64)) == bits(want.view(np.float64))
    assert np.isnan(got[2]).all()
    # one frequency alone keeps its bracket and the shift 0 that normalises
    for f in (freqs[1], freqs[7], 0.0):
        S1 = A.otf_shift_set([f], freq)
        g1 = A.otf_at([f], freq[:, S1], acf[:, S1]/acf[:, S1][:, :1].real, cutoff)
        assert bits(g1.view(np.float64)) == bits(A.otf_at([f], freq, otf, cutoff).view(np.float64))


# --- the analysis through the backend seam ------------------------------------------------------------
@pytest.mark.parametrize('name', ['dblgauss', 'rc'])
def test_seam_equals_per_plane_zernike_fit_and_mtf(name):
    opm = load_model(name)
    be = RefocusBackend(opm)
    fields = list(opm.optical_spec.fov.fields)[:2]
    focs = [-0.05, 0.0, 0.03]
    freqs = [0.0, 25.0, 50.0, 100.0, 5000.0]
    n = 12
    tf = A.through_focus_wavefront(opm, n, foc=focs, num_terms=9, freqs=freqs, fields=fields, backend=be)
    assert tf.coef.shape == (3, len(fields), tf.n_wvls, 9) and tf.n_used.shape == (len(fields), tf.n_wvls)
    for k, f in enumerate(focs):
        z = A.zernike_fit(opm, n, 9, fields=fields, foc=f, backend=be)
        z3 = A.zernike_fit(opm, n, 3, fields=fields, foc=f, backend=be)
        m = A.mtf(opm, n, fields=fields, foc=f, freqs=freqs, backend=be)
        assert bits(tf.zernike_record[k]) == bits(z.summary)
        assert bits(tf.coef[k]) == bits(z.coef) and bits(tf.rms[k]) == bits(z.rms) and bits(tf.pv[k]) == bits(z.pv)
        assert bits(tf.rms_wfe[k]) == bits(z3.rms_residual)
        assert bits(tf.strehl[k]) == bits(m.strehl)
        assert bits(tf.cutoff[k]) == bits(m.cutoff)
        for key in ('otf_x_at', 'otf_y_at', 'mtf_x_at', 'mtf_y_at'):
            assert bits(np.asarray(getattr(tf, key)[k]).view(np.float64)) == \
                bits(np.asarray(getattr(m, key)).view(np.float64)), key
        assert bits(tf.ref_img[k]) == bits(z.ref_img)
    assert (tf.n_used == z.n_used).all()
    assert len(tf.shifts) < n and tf.shifts[0] == 0
    bi = tf.best_index_strehl
    assert ((bi >= 0) & (bi < 3)).all()
    np.testing.assert_array_equal(tf.best_foc_strehl, np.asarray(focs)[bi])
    np.testing.assert_array_equal(tf.best_index_rms, np.argmin(tf.rms_wfe, axis=0))


def test_seam_polychromatic_equals_mtf():
    opm = load_model('dblgauss')
    be = RefocusBackend(opm)
    fields = list(opm.optical_spec.fov.fields)[:1]
    freqs = [10.0, 40.0]
    tf = A.through_focus_wavefront(opm, 10, foc=[0.0, 0.02], freqs=freqs, polychromatic=True, fields=fields,
                                   backend=be)
    for k, f in enumerate([0.0, 0.02]):
        m = A.mtf(opm, 10, fields=fields, foc=f, freqs=freqs, polychromatic=True, backend=be)
        assert bits(tf.poly_x[k]) == bits(m.poly_x) and bits(tf.poly_y[k]) == bits(m.poly_y)
    assert bits(tf.wts) == bits(m.wts)


def test_seam_without_freqs_has_strehl_only():
    opm = load_model('rc')
    be = RefocusBackend(opm)
    fields = list(opm.optical_spec.fov.fields)[:1]
    tf = A.through_focus_wavefront(opm, 8, foc=[-0.01, 0.01], num_terms=3, fields=fields, backend=be)
    assert len(tf.shifts) == 0 and tf.acf_x.shape == (2, tf.n_wvls, 0)
    assert not hasattr(tf, 'otf_x_at') and np.isfinite(tf.strehl).all()


# --- arguments and the ABI ------------------------------------------------------------------------------
def test_argument_checks():
    opm = load_model('singlet')
    for kw in ({'num_rays': 0}, {'num_rays': 1025}, {'num_terms': 2}, {'num_terms': 38}, {'foc': []},
               {'foc': np.zeros(65)}, {'foc': [np.nan]}, {'foc': [0.0], 'freqs': [-1.0]},
               {'foc': [0.0], 'freqs': [np.inf]}, {'foc': [0.0], 'polychromatic': True}):
        with pytest.raises(ValueError):
            A.through_focus_wavefront(opm, **kw)
    with pytest.raises(ValueError, match='defocus_range'):       # foc=None on a model without a range
        A.through_focus_wavefront(opm)
    sm = opm.seq_model
    wl = [w for w in sm.wvlns if w != sm.central_wavelength()]
    if wl:
        with pytest.raises(ValueError, match='central'):
            A.through_focus_wavefront(opm, 8, foc=[0.0], wvls=wl, freqs=[0.0], polychromatic=True)


def test_abi_exports_are_declared():
    hdr = open(os.path.join(ROOT, 'include', 'b200rt.h')).read()
    declared = set(re.findall(r'\b(rt_[a-z0-9_]+)\s*\(', hdr))
    for name in ('rt_trace_grid_opd_focus', 'rt_grid_mtf_shifts'):
        assert name in declared and name in _abi.EXPORTS
    assert re.search(r'#define RT_SPHERE_DOUBLES (\d+)', hdr).group(1) == str(_abi.RT_SPHERE_DOUBLES) == '8'
    assert _abi.RT_ABI_VERSION == 6


def test_abi_refusals_without_a_device():
    lib = _abi.load_library()
    buf = (C.c_double*64)()
    st = (C.c_int32*64)()
    opts = _abi.make_opts()
    out = _abi.rt_out()
    for n_foc in (0, 65):
        assert lib.rt_trace_grid_opd_focus(None, None, 0, 1, C.byref(opts), buf, n_foc, C.byref(out), buf, None) == -1
        assert 'n_foc' in lib.rt_last_error().decode()
    assert lib.rt_trace_grid_opd_focus(None, None, 0, 1, C.byref(opts), buf, 1, C.byref(out), buf, None) == -1
    assert 'required' in lib.rt_last_error().decode()
    assert lib.rt_grid_mtf_shifts(None, st, buf, buf, st, 1, buf, buf, buf, None) == -1
    assert 'grid' in lib.rt_last_error().decode()
    assert lib.rt_grid_mtf_shifts(None, st, buf, buf, st, -1, buf, buf, buf, None) == -1
    assert 'n_shifts' in lib.rt_last_error().decode()
