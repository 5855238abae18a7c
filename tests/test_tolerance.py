"""Tolerance analysis on the CPU: the fast descriptor path against the perturbed model, the summands
of csrc/rt_tol.cuh compiled for the host against tests/tol_sums.py, the merit algebra against brute
force on oracle-traced rays, and the analyses through the oracle-backed ``backend=`` seam."""
import os
import sys

import numpy as np
import pytest

import tol_sums as TS
from conftest import ROOT, load_model
from rayoptics_b200 import _abi, analyses as A, engine as E, model as M, tolerance as TOL
from rayoptics_b200.table import describe_model

sys.path.insert(0, os.path.join(ROOT, 'tests', 'hostsim'))
import tolerance_build as HB  # noqa: E402

T = TOL.Tolerance


def _same(opm, changes):
    sm = opm.seq_model
    d0, n0, _ = describe_model(sm)
    d1, n1 = TOL.perturbed_descriptors(d0, n0, changes, sm)
    d2, n2, _ = describe_model(TOL.perturbed_model(opm, changes).seq_model)
    changed = bytes(d1) != bytes(d0) or n1.tobytes() != n0.tobytes()
    return changed and bytes(d1) == bytes(d2) and n1.tobytes() == n2.tobytes()


@pytest.mark.parametrize('kind', TOL.KINDS)
@pytest.mark.parametrize('sign', (1.0, -1.0))
def test_fast_path_equals_perturbed_model_dblgauss(kind, sign):
    opm = load_model('dblgauss')
    n = len(opm.seq_model.ifcs)
    for i in (1, 3, 6, n - 2):
        if kind == 'radius' and opm.seq_model.ifcs[i].profile.cv == 0.0:
            continue
        assert _same(opm, [(T(kind, i, 0.03), sign*0.03)]), (kind, i)


def test_fast_path_other_models():
    cell = load_model('cellphone')
    for i in (2, 5, 9):                       # RadialPolynomial aspheres
        for k in ('radius', 'conic'):
            assert _same(cell, [(T(k, i, 0.01), 0.01)]) and _same(cell, [(T(k, i, 0.01), -0.01)])
    three = load_model('threemir')            # decenters and tilts added to the existing ones
    for i in (2, 3, 4, 5):
        for k in ('decenter_x', 'decenter_y', 'tilt_x', 'tilt_y', 'thickness'):
            if k == 'thickness' and i > len(three.seq_model.gaps) - 1:
                continue
            assert _same(three, [(T(k, i, 0.02), -0.02)]), (k, i)
    diff = load_model('diffractive')          # phase elements
    for k in TOL.KINDS:
        assert _same(diff, [(T(k, 3, 0.01), 0.01)]), k
    dg = load_model('dblgauss')
    combo = [(T('radius', 2, 0.1), 0.05), (T('conic', 3, 0.1), -0.02), (T('thickness', 4, 0.1), 0.07),
             (T('index', 5, 1e-3), 4e-4), (T('tilt_x', 6, 0.1), 0.03)]
    assert _same(dg, combo)


def test_refusals():
    opm = load_model('dblgauss')
    sm, n = opm.seq_model, len(opm.seq_model.ifcs)
    bad = [T('radius', 0, 0.1), T('radius', n - 1, 0.1), T('thickness', 0, 0.1), T('bogus', 2, 0.1),
           T('tilt_x', n - 1, 0.1)]
    plane = [i for i in range(1, n - 1) if sm.ifcs[i].profile.cv == 0.0]
    bad += [T('radius', plane[0], 0.1)]
    for t in bad:
        with pytest.raises(ValueError):
            TOL.check(sm, t)
        with pytest.raises(ValueError):
            TOL.perturbed_model(opm, [(t, 0.05)])
    thin = load_model('thin_triplet')
    k = [i for i, f in enumerate(thin.seq_model.ifcs) if type(f).__name__ == 'ThinLens'][0]
    for kind in ('radius', 'conic'):
        with pytest.raises(ValueError):
            TOL.check(thin.seq_model, T(kind, k, 0.1))
    sm._tfrms_given = [t for t in sm.lcl_tfrms]
    for kind in ('thickness', 'decenter_x', 'tilt_y'):
        with pytest.raises(ValueError):
            TOL.check(sm, T(kind, 2, 0.1))
    TOL.check(sm, T('radius', 2, 0.1))


# ---- oracle-traced rays
def _oracle_rays(oracle, opm, descs, n_by_wvl, spec):
    opts = _abi.make_opts(check_apertures=True, first_surf=1, last_surf=len(descs) - 2)
    r = oracle.trace_grid(spec.c_spec(), descs, n_by_wvl, 0, spec.n_rays, opts, wvls=list(opm.seq_model.wvlns))
    return r['status'], r['abr'][0], r['abr'][1], r['op'], r['last'][3], r['last'][4], r['last'][5]


class OracleBackend:
    """``trace_variants`` / ``chief_ref`` of tolerance_sensitivity on the C oracle and tol_sums"""

    def __init__(self, oracle, opm):
        self.oracle, self.opm = oracle, opm

    def chief_ref(self, descs, n_by_wvl, spec, wvl_idx):
        g = E.PupilGridSpec(spec.fields, [wvl_idx], [0.0], [0.0], spec.eprad, spec.z_pupil, apply_vignetting=False,
                            flip_z_dir=spec.flip_z_dir, foc=0.0)
        opts = _abi.make_opts(check_apertures=False, first_surf=1, last_surf=len(descs) - 2)
        r = self.oracle.trace_grid(g.c_spec(), descs, n_by_wvl, 0, g.n_rays, opts, wvls=list(self.opm.seq_model.wvlns))
        return np.ascontiguousarray(r['last'][0:2].T)

    def trace_variants(self, descs, n_by_wvl, spec):
        shape = TS.Shape.of(spec)
        return np.stack([TS.record(shape, *_oracle_rays(self.oracle, self.opm, d, nb, spec))
                         for d, nb in zip(descs, n_by_wvl)])


def _nominal_spec(opm, num_rays, backend):
    sm = opm.seq_model
    args, kw = E._grid_args(opm, sm.index_for_wavelength, num_rays, None, None, None, (-1.0, 1.0), True)
    spec = E.PupilGridSpec(*args, **kw)
    d0, n0, _ = describe_model(sm)
    ref = backend.chief_ref(d0, n0, spec, sm.index_for_wavelength(sm.central_wavelength()))
    return E.PupilGridSpec(*args, ref_img=np.repeat(ref[:, None, :], spec.n_wvls, axis=1), **kw)


def test_header_summands_equal_restatement(oracle):
    opm = load_model('dblgauss')
    be = OracleBackend(oracle, opm)
    spec = _nominal_spec(opm, 12, be)
    d0, n0, _ = describe_model(opm.seq_model)
    d1, n1 = TOL.perturbed_descriptors(d0, n0, [(T('tilt_y', 3, 0.1), 0.08)], opm.seq_model)
    st, ax, ay, op, dx, dy, dz = _oracle_rays(oracle, opm, d1, n1, spec)
    ok = st == 0
    h = HB.summands(ax, ay, op, dx, dy, dz)
    assert np.array_equal(h[ok][:, list(TS.SLOPE_COLS)], TS.slope_summands(ax, ay, dx, dy, dz, ok)[ok])
    assert np.array_equal(h[ok][:, [5, 6, 7, 8, 9, 14]],
                          np.stack([ax, ay, ax*ax, ay*ay, ax*ay, op], axis=1)[ok])


def test_merit_algebra_against_brute_force(oracle):
    opm = load_model('dblgauss')
    be = OracleBackend(oracle, opm)
    spec = _nominal_spec(opm, 16, be)
    sm = opm.seq_model
    d0, n0, _ = describe_model(sm)
    sets = [[], [(T('thickness', 5, 0.1), 0.08)], [(T('radius', 3, 1.0), -0.6), (T('decenter_y', 4, 0.05), 0.03)]]
    var = [TOL.perturbed_descriptors(d0, n0, ch, sm) for ch in sets]
    rec = be.trace_variants([v[0] for v in var], np.stack([v[1] for v in var]), spec)
    nf, nw = spec.n_fields, spec.n_wvls
    rec = rec.reshape(len(sets), nf, nw, -1)
    ww, fw = [1.0, 2.0, 1.0], [1.0, 0.5, 2.0]
    m = A._tol_moments(rec, ww)
    res = A.tol_merit(rec, ww, fw)
    deltas = np.array([-0.2, -0.05, -0.01, 0.0, 0.013, 0.07, 0.3])
    for v, (d, nb) in enumerate(var):
        st, ax, ay, op, dx, dy, dz = _oracle_rays(oracle, opm, d, nb, spec)
        per = spec.rays_per_tile

        def brute(delta):
            s2 = np.zeros(nf)
            for f in range(nf):
                N = X1 = Y1 = X2 = 0.0
                for w in range(nw):
                    sl = slice((f*nw + w)*per, (f*nw + w + 1)*per)
                    ok = st[sl] == 0
                    x = ax[sl][ok] + delta*(dx[sl][ok]/dz[sl][ok])
                    y = ay[sl][ok] + delta*(dy[sl][ok]/dz[sl][ok])
                    N += ww[w]*ok.sum()
                    X1 += ww[w]*x.sum()
                    Y1 += ww[w]*y.sum()
                    X2 += ww[w]*(x*x + y*y).sum()
                s2[f] = X2/N - (X1*X1 + Y1*Y1)/(N*N)
            return s2

        for delta in deltas:
            assert np.allclose(A.tol_sigma2(m, delta)[v], brute(delta), rtol=1e-12, atol=0)
        scan = np.linspace(res.focus[v] - 0.05, res.focus[v] + 0.05, 2001)
        mm = [np.sqrt((brute(x)*fw).sum()/sum(fw)) for x in scan]
        assert abs(scan[int(np.argmin(mm))] - res.focus[v]) <= 1e-4
        assert res.merit[v] <= min(mm)*(1 + 1e-12)
    # a change of 0 gives exactly the nominal record and merit
    z = TOL.perturbed_descriptors(d0, n0, [(T('thickness', 5, 0.1), 0.0)], sm)
    rz = be.trace_variants([z[0]], z[1][None], spec).reshape(1, nf, nw, -1)
    assert np.array_equal(A.tol_merit(rz, ww, fw).merit, res.merit[:1])


def test_analyses_through_backend(oracle):
    opm = load_model('dblgauss')
    be = OracleBackend(oracle, opm)
    tols = [T('radius', 2, 0.5), T('thickness', 4, 0.05), T('tilt_x', 6, 0.05)]
    s = A.tolerance_sensitivity(opm, tols, num_rays=8, backend=be)
    assert len(s.merit_plus) == 3 and np.isfinite(s.merit_plus).all()
    assert s.estimated >= s.nominal
    nom = be.trace_variants([describe_model(opm.seq_model)[0]], describe_model(opm.seq_model)[1][None],
                            _nominal_spec(opm, 8, be))
    region = opm.optical_spec.spectral_region
    ww = [region.spectral_wts[list(region.wavelengths).index(w)] for w in opm.seq_model.wvlns]
    fw = [f.wt for f in opm.optical_spec.field_of_view.fields]
    r0 = A.tol_merit(nom.reshape(1, len(fw), len(ww), -1), ww, fw)
    assert s.nominal == r0.merit[0] and s.nominal_focus == r0.focus[0]
    mc1 = A.tolerance_monte_carlo(opm, tols, num_trials=6, seed=3, num_rays=8, backend=be)
    mc2 = A.tolerance_monte_carlo(opm, tols, num_trials=6, seed=3, num_rays=8, backend=be)
    assert np.array_equal(mc1.merit, mc2.merit) and np.array_equal(mc1.values, mc2.values)
    assert mc1.nominal == s.nominal
    assert (np.abs(mc1.values) <= np.array([t.delta for t in tols])).all()
    u = A.draw_tolerances(tols, 50, seed=1, distribution='uniform')
    assert (np.abs(u) <= np.array([t.delta for t in tols])).all()
    with pytest.raises(ValueError):
        A.draw_tolerances(tols, 2, distribution='cauchy')


def test_abi_declares_variants():
    src = open(os.path.join(ROOT, 'include', 'b200rt.h')).read()
    for name in ('rt_variants_create', 'rt_variants_destroy', 'rt_grid_variants_scratch_bytes',
                 'rt_trace_grid_variants'):
        assert name in _abi.EXPORTS and name + '(' in src
    assert '#define RT_TOL_DOUBLES 24' in src and _abi.RT_TOL_DOUBLES == 24
