"""Wavefront tolerancing on the CPU: the wave records of csrc/rt_tolwave.cuh, compiled for the host and fed
the oracle's chief rays of perturbed systems, against waveabr's host path on the perturbed model (bit for
bit); the merit algebra against brute force (oracle OPDs per perturbed model -> _wfe_sums_host ->
wavefront_statistics -> weights); the refusals; the spot criterion unchanged."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, load_model
from rayoptics_b200 import _abi, analyses as A, engine as E, tolerance as TOL, waveabr as WA
from rayoptics_b200.table import describe_model
from test_analyses_vs_reference import OracleBackend as ModelBackend
from test_tolerance import OracleBackend as SpotBackend

sys.path.insert(0, os.path.join(ROOT, 'tests', 'hostsim'))
import tolwave_build as HW  # noqa: E402

T = TOL.Tolerance
MODELS = ['dblgauss', 'cellphone', 'relay_na', 'fisheye', 'diffractive', 'telecentric']


def _parax(opm):
    fod = opm['analysis_results']['parax_data'].fod
    return (fod.exp_dist, abs(fod.n_obj), abs(fod.n_img))


def every_kind(sm):
    """one tolerance of every kind on the interfaces / gaps of sm (decenters and tilts short of interface
    n_ifc - 2), plus the thickness of the last gap, which moves the image plane"""
    n_ifc = len(sm.ifcs)
    prof = [i for i in range(1, n_ifc - 2) if getattr(sm.ifcs[i], 'profile', None) is not None
            and type(sm.ifcs[i]).__name__ != 'ThinLens' and sm.ifcs[i].profile.cv != 0.0]
    s = prof[len(prof)//2] if prof else 1
    out = [T('radius', s, 0.01/abs(sm.ifcs[s].profile.cv)) if prof else None, T('conic', s, 0.05),
           T('thickness', max(1, (len(sm.gaps) - 1)//2), 0.03), T('index', s, 1e-3),
           T('thickness', len(sm.gaps) - 1, 0.05)]
    if sm._tfrms_given is None:
        out += [T('decenter_x', s, 0.01), T('decenter_y', s, 0.01), T('tilt_x', s, 0.05), T('tilt_y', s, 0.05)]
    return [t for t in out if t is not None]


def _change_sets(sm):
    sets = [[]]
    for t in every_kind(sm):
        sets += [[(t, t.delta)], [(t, -t.delta)]]
    return sets


class WaveBackend:
    """``variant_waves`` / ``trace_variants_wfe`` of the wavefront criterion on the C oracle and the host
    build of csrc/rt_tolwave.cuh"""

    def __init__(self, oracle, opm):
        self.o, self.opm = oracle, opm
        self.wide = bool(opm.optical_spec.field_of_view.is_wide_angle)
        self.wvls = list(opm.seq_model.wvlns)

    def _opts(self, n_ifc, check_apertures):
        return _abi.make_opts(first_surf=1, last_surf=n_ifc - 2, check_apertures=check_apertures,
                              intersect_obj=not self.wide)

    def chief_rays(self, descs, n_by_wvl, spec):
        g = E.PupilGridSpec(spec.fields, spec.wvl_idx, [0.0], [0.0], spec.eprad, spec.z_pupil,
                            apply_vignetting=False, flip_z_dir=spec.flip_z_dir, pupil_kind=spec.pupil_kind)
        p, d, wv, _ = self.o.grid_start_rays(g.c_spec(), 0, g.n_rays)
        r = self.o.trace_bundle(descs, n_by_wvl, p, d, wv, self._opts(len(descs), False), want_full=True,
                                wvls=self.wvls)
        return r['full'], r['op'], r['status']

    def variant_waves(self, descs, n_by_wvl, spec, parax):
        waves, refs, status = [], [], []
        for d, nb in zip(descs, n_by_wvl):
            full, op, st = self.chief_rays(d, nb, spec)
            W, ref, _ = HW.records(full, op, st, d[len(d) - 2], spec.foc, parax)
            waves.append(W)
            refs.append(ref)
            status.append(st)
        return np.stack(waves), np.stack(refs), np.stack(status)

    def trace_variants_wfe(self, descs, n_by_wvl, spec, wave):
        recs = []
        for d, nb, w in zip(descs, n_by_wvl, wave):
            sv = E.PupilGridSpec(spec.fields, spec.wvl_idx, spec.pupil_x, spec.pupil_y, spec.eprad, spec.z_pupil,
                                 apply_vignetting=False, flip_z_dir=spec.flip_z_dir, foc=spec.foc, wave=w,
                                 pupil_kind=spec.pupil_kind)
            r = self.o.trace_grid(sv.c_spec(), d, nb, 0, sv.n_rays, self._opts(len(d), True), wvls=self.wvls)
            recs.append(A._wfe_sums_host(sv, r['status'], r['opd']))
        return np.stack(recs)


@pytest.mark.parametrize('name', MODELS)
def test_header_records_equal_the_host_path(oracle, name):
    """rt_tolwave.cuh on the oracle's chief rays of every perturbed system == waveabr._tiles_at on
    perturbed_model, bit for bit; the image gap of descriptor n_ifc - 2 == gaps[-1].thi"""
    opm = load_model(name)
    sm, osp = opm.seq_model, opm.optical_spec
    fields, wvls = list(osp.field_of_view.fields), list(sm.wvlns)
    foc = osp.defocus.focus_shift
    be = WaveBackend(oracle, opm)
    args, kw = A._wavefront_grid_args(opm, None, 4, fields, wvls, foc, None, None)
    spec = E.PupilGridSpec(*args, **kw)
    d0, n0, _ = describe_model(sm)
    branches = set()
    for ch in _change_sets(sm):
        d, nb = TOL.perturbed_descriptors(d0, n0, ch, sm)
        pm = TOL.perturbed_model(opm, ch)
        assert d[len(d) - 2].t[2] == pm.seq_model.gaps[-1].thi, ch
        full, op, st = be.chief_rays(d, nb, spec)
        assert (st == 0).all(), ch
        W, ref, br = HW.records(full, op, st, d[len(d) - 2], foc, _parax(opm))
        wave, ref_img, _ = WA._tiles_at(pm, full, op, fields, wvls, foc, None, None, None)
        assert np.array_equal(W, wave.reshape(-1, _abi.RT_WAVE_DOUBLES)), (name, ch)
        assert np.array_equal(ref, ref_img.reshape(-1, 2)), (name, ch)
        branches |= set(br.tolist())
    if name == 'telecentric':
        assert 1 in branches                        # the infinite-reference record
    if name == 'dblgauss':
        assert 2 in branches                        # the on-axis chief ray: |u| < 1e-14


def test_failed_chief_ray_gives_nan_record():
    last = describe_model(load_model('dblgauss').seq_model)[0][-2]
    full = np.ones((6, 10, 2))
    W, ref, br = HW.records(full, np.zeros(2), np.array([0, 3]), last, 0.0, (1.0, 1.0, 1.0))
    assert np.isfinite(W[0]).all() and np.isnan(W[1]).all() and np.isnan(ref[1]).all()


def _weights(opm):
    osp, sm = opm.optical_spec, opm.seq_model
    region = osp.spectral_region
    ww = [region.spectral_wts[list(region.wavelengths).index(w)] for w in sm.wvlns]
    return ww, [f.wt for f in osp.field_of_view.fields]


@pytest.mark.parametrize('compensate_focus', (True, False))
def test_merit_algebra_against_brute_force(oracle, compensate_focus):
    """the sensitivity merit through the backend seam == wavefront_error of each perturbed model
    (oracle-traced, its own host reference spheres) combined with the weights by hand"""
    opm = load_model('dblgauss')
    tols = [T('radius', 3, 1.0), T('thickness', len(opm.seq_model.gaps) - 1, 0.05), T('tilt_y', 4, 0.05)]
    s = A.tolerance_sensitivity(opm, tols, num_rays=12, backend=WaveBackend(oracle, opm), criterion='wavefront',
                                compensate_focus=compensate_focus)
    res = s.result
    ww, fw = _weights(opm)
    sets = [[]] + [[(t, sg*t.delta)] for t in tols for sg in (1.0, -1.0)]
    key = 'rms_focus' if compensate_focus else 'rms_tilt'
    for v, ch in enumerate(sets):
        pm = TOL.perturbed_model(opm, ch)
        we = A.wavefront_error(pm, num_rays=12, backend=ModelBackend(pm))
        rms = getattr(we, key)
        assert np.array_equal(res.rms[v], rms), (v, ch)
        assert np.array_equal(res.n_ok[v], we.n_ok.sum(axis=1))
        s2 = [sum(ww[w]*rms[f, w]**2 for w in range(len(ww)))/sum(ww) for f in range(len(fw))]
        m = np.sqrt(sum(fw[f]*s2[f] for f in range(len(fw)))/sum(fw))
        assert abs(res.merit[v] - m) <= 1e-13*m, (v, res.merit[v], m)
        assert np.allclose(res.strehl[v], np.exp(-(2*np.pi*np.sqrt(s2))**2), rtol=1e-13, atol=0)
    m0 = res.merit[0]
    worst = [max(res.merit[1 + 2*i]**2 - m0**2, res.merit[2 + 2*i]**2 - m0**2, 0.0) for i in range(len(tols))]
    assert abs(s.estimated - np.sqrt(m0**2 + sum(worst))) <= 1e-13*s.estimated
    assert s.estimated >= s.nominal and s.nominal_focus.shape == (3, 3)


def test_monte_carlo_through_backend(oracle):
    opm = load_model('dblgauss')
    tols = [T('radius', 2, 0.5), T('index', 5, 1e-3)]
    be = WaveBackend(oracle, opm)
    a = A.tolerance_monte_carlo(opm, tols, num_trials=3, seed=2, num_rays=8, backend=be, criterion='wavefront')
    b = A.tolerance_monte_carlo(opm, tols, num_trials=3, seed=2, num_rays=8, backend=be, criterion='wavefront')
    assert np.array_equal(a.merit, b.merit) and np.isfinite(a.merit).all()
    assert a.focus.shape == (3, 3, 3) and a.result.strehl.shape == (4, 3)
    assert (a.result.chief_status == 0).all()


def test_refusals(oracle):
    opm = load_model('dblgauss')
    sm, n = opm.seq_model, len(opm.seq_model.ifcs)
    for kind in ('decenter_x', 'decenter_y', 'tilt_x', 'tilt_y'):
        TOL.check(sm, T(kind, n - 2, 0.01))                 # the spot criterion takes them
        with pytest.raises(ValueError):
            TOL.check(sm, T(kind, n - 2, 0.01), 'wavefront')
        with pytest.raises(ValueError):
            A.tolerance_sensitivity(opm, [T(kind, n - 2, 0.01)], num_rays=4, criterion='wavefront',
                                    backend=WaveBackend(oracle, opm))
    TOL.check(sm, T('tilt_x', n - 3, 0.01), 'wavefront')
    TOL.check(sm, T('thickness', len(sm.gaps) - 1, 0.01), 'wavefront')
    with pytest.raises(ValueError):
        TOL.check(sm, T('radius', 2, 0.1), 'bogus')
    three = load_model('threemir')                         # wavefront_error refuses its OPD
    with pytest.raises(ValueError):
        TOL.check_wavefront_model(three.seq_model)
    with pytest.raises(ValueError):
        TOL.check(three.seq_model, T('radius', 2, 0.1), 'wavefront')
    with pytest.raises(ValueError):
        A.tolerance_monte_carlo(three, [T('radius', 2, 0.1)], num_trials=2, num_rays=4, criterion='wavefront',
                                backend=WaveBackend(oracle, three))


def test_spot_criterion_unchanged(oracle):
    opm = load_model('dblgauss')
    be = SpotBackend(oracle, opm)
    tols = [T('radius', 2, 0.5), T('tilt_x', 6, 0.05)]
    a = A.tolerance_sensitivity(opm, tols, num_rays=8, backend=be)
    b = A.tolerance_sensitivity(opm, tols, num_rays=8, backend=be, criterion='spot')
    assert isinstance(a.result, A.TolMerit)
    for k in ('merit_plus', 'merit_minus', 'focus_plus', 'focus_minus'):
        assert np.array_equal(getattr(a, k), getattr(b, k))
    assert (a.nominal, a.nominal_focus, a.estimated) == (b.nominal, b.nominal_focus, b.estimated)
    c = A.tolerance_monte_carlo(opm, tols, num_trials=3, num_rays=8, backend=be)
    d = A.tolerance_monte_carlo(opm, tols, num_trials=3, num_rays=8, backend=be, criterion='spot')
    assert np.array_equal(c.merit, d.merit) and np.array_equal(c.focus, d.focus)


def test_abi_declares_variant_waves():
    src = open(os.path.join(ROOT, 'include', 'b200rt.h')).read()
    for name in ('rt_variants_wave', 'rt_grid_variants_wfe_scratch_bytes', 'rt_trace_grid_variants_wfe'):
        assert name in _abi.EXPORTS and name + '(' in src
