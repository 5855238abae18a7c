"""CPU: the wavefront-error sums (restated in tests/wfe_sums.py), engine.wavefront_statistics, the
host logic of analyses.wavefront_error through the backend= seam with the oracle, and the ABI v6
surface of rt_trace_grid_wfe.

Bounds.  ``rms`` is the one-pass sqrt(sum W^2/n - mean^2): with sums of depth d its square is off
by at most (3d + 10)·u·kappa relative, kappa = (sum W^2/n)/var (DESIGN.md section 3 item 5d).  A fit
with p basis functions solves the normal equations G c = b and forms RSS = sum W^2 - c.b.  The
sums carry a relative error of at most gamma_d each; the solve, done on the Gram matrix scaled to
unit diagonal, adds at most about p·u·cond of the scaled matrix to c.  So the error of RSS is at
most ((3d + 10) + p·cond)·u·(sum W^2 + |c|.|b|), and RSS/n = rms_fit^2 may be off by that over n.
The tests check every tile against this bound and report the worst kappa = (sum W^2 + |c|.|b|)/RSS
of the fixtures."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import wfe_sums as WS
from conftest import ROOT, load_model
from rayoptics_b200 import _abi, analyses as A, engine as E

U = 2.0**-53


# --- the restatement of the 13 sums ------------------------------------------------------------
def adversarial(rng, n):
    """OPDs and pupil coordinates with magnitudes 1e-9 to 1e3, cancellation and signed zeros"""
    w = rng.standard_normal(n)*10.0**rng.integers(-9, 4, n)
    w[rng.random(n) < 0.1] *= -1e6
    w[rng.random(n) < 0.05] = -0.0
    x = rng.uniform(-1, 1, n)
    y = rng.uniform(-1, 1, n)
    x[rng.random(n) < 0.05] = -0.0
    status = np.where(rng.random(n) < 0.8, 0, rng.integers(1, 6, n))
    return status, w, x, y


@pytest.mark.parametrize('rays_per_tile, n_tiles, rng_range', [
    (1, 3, None), (33*33, 2, None), (64*64, 3, (5, 27)), (512*512, 1, (100, 101)), (64*64, 2, (9, 9))])
def test_ordered_sums_within_bound_of_exact(rays_per_tile, n_tiles, rng_range):
    rng = np.random.default_rng(rays_per_tile + n_tiles)
    shape = WS.Shape(rays_per_tile, n_tiles, *(rng_range or (0, None)))
    status, w, x, y = adversarial(rng, shape.n_rays)
    got = WS.ordered_summary(shape, status, w, x, y)
    want, absum = WS.exact_summary(shape, status, w, x, y)
    assert (got[:, :5] == want[:, :5]).all()
    assert (got[:, 5:7] == want[:, 5:7]).all()
    bound = WS.sum_bound(absum, WS.chain_depth(shape, 'items'))
    err = np.abs(got[:, list(WS.SUM_COLS)] - want[:, list(WS.SUM_COLS)])
    assert (err <= bound).all()
    if shape.chunk_end == shape.chunk_begin:
        assert np.array_equal(got, WS.identity(n_tiles))


def test_item_tree_equals_the_shuffle_tree_lane_by_lane():
    rng = np.random.default_rng(7)
    for _ in range(50):
        status, w, x, y = adversarial(rng, 32)
        v = WS.summands(w, x, y, status == 0)
        tree = WS.item_tree(v)
        lanes = WS.shuffle_tree_lanes(v)
        assert tree.view(np.uint64).tolist() == lanes.view(np.uint64).tolist()


def fused(a, b, c):
    """fma(a, b, c) rounded once (exact rational arithmetic)"""
    from fractions import Fraction
    return float(Fraction(a)*Fraction(b) + Fraction(c))


def test_plausible_mistakes_change_the_bits():
    rng = np.random.default_rng(11)
    shape = WS.Shape(64*64, 2)
    status, w, x, y = adversarial(rng, shape.n_rays)
    x, y = rng.uniform(-1, 1, (2, shape.n_rays))        # no signed zeros: every mistake must show
    good = WS.ordered_summary(shape, status, w, x, y)
    bits = lambda s: s.view(np.uint64).tolist()         # noqa: E731

    swapped = good.copy()
    swapped[:, [9, 10]] = swapped[:, [10, 9]]
    assert bits(swapped) != bits(good)                                 # two columns swapped
    assert bits(WS.ordered_summary(shape, status, w, y, x)) != bits(good)   # x and y swapped

    def with_summands(fn):
        # the tile's work-item sums: one ulp per ray can cancel out of a whole tile's sum
        return WS.tile_items(shape, 0, fn(w, x, y, status == 0)[:shape.rays_per_tile])[0]

    def r2_fused(w_, x_, y_, ok=None):
        v = orig_summands(w_, x_, y_, ok)
        r2 = np.array([fused(a, a, b*b) for a, b in zip(x_, y_)])
        v[:, 4], v[:, 10], v[:, 11], v[:, 12] = r2*w_, x_*r2, y_*r2, r2*r2
        if ok is not None:
            v[~np.asarray(ok, bool)] = 0.0
        return v

    def r2w_reordered(w_, x_, y_, ok=None):
        v = orig_summands(w_, x_, y_, ok)
        v[:, 4] = x_*x_*w_ + y_*y_*w_
        if ok is not None:
            v[~np.asarray(ok, bool)] = 0.0
        return v
    orig_summands = WS.summands
    items0 = bits(with_summands(orig_summands))
    assert bits(with_summands(r2_fused)) != items0                     # r2 fused
    assert bits(with_summands(r2w_reordered)) != items0                # r2*W reordered

    v = WS.summands(w, x, y, status == 0)[:shape.rays_per_tile]
    items, inr = WS.tile_items(shape, 0, v)
    keep = np.ones(int(inr.sum()), bool)
    assert bits(WS.reduce_entries(items[inr], keep)) == bits(good[0, 7:20])
    keep[37] = False                                                   # an item dropped
    assert bits(WS.reduce_entries(items[inr], keep)) != bits(good[0, 7:20])

    n = shape.n_chunks
    parts = [WS.ordered_summary(shape.sub(a, b), *sl) for a, b, sl in
             [(a, b, _slice(shape, a, b, status, w, x, y)) for a, b in ((0, 3), (3, 7), (7, n))]]
    whole = WS.combine(parts)
    assert bits(WS.combine(parts[::-1])) != bits(whole)                # parts combined out of order


def _slice(shape, a, b, *arrays):
    i, j = shape.first_ray(a), shape.first_ray(b)
    return tuple(np.asarray(v)[i:j] for v in arrays)


# --- wavefront_statistics ----------------------------------------------------------------------
def record(w, x, y, status=None):
    status = np.zeros(len(w), int) if status is None else status
    s, _ = WS.exact_summary(WS.Shape(len(w), 1), status, w, x, y)
    return s


def test_statistics_recover_known_coefficients():
    rng = np.random.default_rng(3)
    g = np.linspace(-1, 1, 41)
    x, y = (v.ravel() for v in np.meshgrid(g, g, indexing='ij'))
    keep = x*x + y*y <= 1.0
    x, y = x[keep], y[keep]
    lam = 5.5e-4
    a, b, c, d = 0.3, -1.2, 0.7, 2.5                     # waves
    res = rng.standard_normal(len(x))*0.01
    res -= res.mean()
    w = (a + b*x + c*y + d*(x*x + y*y) + res)*lam
    st = E.wavefront_statistics(record(w, x, y), lam)
    A4 = np.stack([np.ones_like(x), x, y, x*x + y*y], axis=1)
    coef, *_ = np.linalg.lstsq(A4, w/lam, rcond=None)
    assert abs(st['focus'][0] - coef[3]) < 1e-9
    assert abs(st['focus'][0] - d) < 0.01
    r = w/lam - A4 @ coef
    np.testing.assert_allclose(st['rms_focus'][0], np.sqrt(np.mean(r*r)), rtol=1e-7)
    A3 = A4[:, :3]
    c3, *_ = np.linalg.lstsq(A3, w/lam, rcond=None)
    np.testing.assert_allclose([st['tilt_x'][0], st['tilt_y'][0]], c3[1:], rtol=1e-9)
    np.testing.assert_allclose(st['rms'][0], np.std(w/lam), rtol=1e-9)
    np.testing.assert_allclose(st['pv'][0], (w.max() - w.min())/lam, rtol=1e-12)


def test_pure_tilt_has_no_residual_and_units_convert():
    g = np.linspace(-1, 1, 21)
    x, y = (v.ravel() for v in np.meshgrid(g, g, indexing='ij'))
    w = 0.002*x - 0.0005*y + 1e-4
    s = record(w, x, y)
    for lam in (5.0e-4, 1.0e-3):
        st = E.wavefront_statistics(s, lam)
        assert st['rms_tilt'][0] < 1e-6*st['rms'][0]
        assert st['rms_focus'][0] < 1e-6*st['rms'][0]
        np.testing.assert_allclose(st['tilt_x'][0], 0.002/lam, rtol=1e-10)
        np.testing.assert_allclose(st['tilt_y'][0], -0.0005/lam, rtol=1e-10)
        assert abs(st['focus'][0]) < 1e-8/lam
        np.testing.assert_allclose(st['pv'][0], (w.max() - w.min())/lam, rtol=0)
    st2 = E.wavefront_statistics(np.concatenate([s, s]), np.array([5.0e-4, 1.0e-3]))
    np.testing.assert_allclose(st2['rms'][0], 2*st2['rms'][1], rtol=1e-15)


def test_undetermined_fits_and_nan():
    s_one = record(np.array([0.1]), np.array([0.0]), np.array([0.0]))          # one ray
    g = np.linspace(-1, 1, 9)
    s_line = record(0.01*g, g, np.zeros_like(g))                               # all rays on y = 0
    s_none = record(np.array([0.1, 0.2]), np.zeros(2), np.zeros(2), status=np.array([1, 3]))
    w_nan = 0.01*g
    w_nan[3] = np.nan
    s_nan = record(w_nan, g, g*g)
    st = E.wavefront_statistics(np.concatenate([s_one, s_line, s_none, s_nan]), 1e-3)
    assert st['rms'][0] == 0.0 and st['pv'][0] == 0.0
    for k in ('rms_tilt', 'tilt_x', 'tilt_y', 'rms_focus', 'focus'):
        assert np.isnan(st[k][0]) and np.isnan(st[k][1]) and np.isnan(st[k][2]) and np.isnan(st[k][3]), k
    assert np.isfinite(st['rms'][1])
    for k in ('rms', 'pv'):
        assert np.isnan(st[k][2]), k
    assert st['n_ok'][2] == 0 and st['n_missed'][2] == 1 and st['n_blocked'][2] == 1
    assert np.isnan(st['rms'][3]) and np.isfinite(st['pv'][3])                 # NaN W: sums NaN, fmin / fmax skip it


def test_statistics_accept_torch_tensors():
    import torch
    g = np.linspace(-1, 1, 7)
    x, y = (v.ravel() for v in np.meshgrid(g, g, indexing='ij'))
    s = record(0.01*x*y + 0.02*(x*x + y*y), x, y)
    a = E.wavefront_statistics(s, 1e-3)
    b = E.wavefront_statistics(torch.as_tensor(s), 1e-3)
    for k in a:
        assert torch.is_tensor(b[k])
        np.testing.assert_array_equal(b[k].numpy(), a[k])


# --- wavefront_error through the backend seam ------------------------------------------------
def numpy_statistics(grid):
    """statistics of a RayGrid map (waves) by two-pass / least-squares numpy"""
    gx, gy, opd = grid
    m = np.isfinite(opd)
    w, x, y = opd[m], gx[m], gy[m]
    n = len(w)
    out = {'n': n, 'rms': np.sqrt(math.fsum((w - math.fsum(w)/n)**2)/n), 'pv': w.max() - w.min()}
    for key, cols in (('tilt', [np.ones(n), x, y]), ('focus', [np.ones(n), x, y, x*x + y*y])):
        Am = np.stack(cols, axis=1)
        c, *_ = np.linalg.lstsq(Am, w, rcond=None)
        r = w - Am @ c
        out['rms_' + key] = np.sqrt(math.fsum(r*r)/n)
        out['c_' + key] = c
        out['kappa_' + key] = math.fsum(w*w)/max(math.fsum(r*r), 1e-300)
        out['cond_' + key] = np.linalg.cond(Am.T @ Am/np.sqrt(np.outer(np.diag(Am.T @ Am), np.diag(Am.T @ Am))))
    out['kappa'] = (math.fsum(w*w)/n)/max(out['rms']**2, 1e-300)
    return out


def check_against_numpy(wfe, opm, fields, wvls, maps, depth):
    """every tile of ``wfe`` against numpy statistics of its RayGrid map; returns the worst kappa"""
    worst = 0.0
    for fi in range(len(fields)):
        for wi in range(len(wvls)):
            ref = numpy_statistics(maps[fi][wi])
            assert wfe.n_ok[fi, wi] == ref['n']
            tol = (3*depth + 10)*U*ref['kappa']
            assert abs(wfe.rms[fi, wi]**2 - ref['rms']**2) <= tol*ref['rms']**2 + 1e-300
            # (max - min)/lambda against max*(1/lambda) - min*(1/lambda): four roundings of max |W|
            assert abs(wfe.pv[fi, wi] - ref['pv']) <= 8*U*np.abs(maps[fi][wi][2][np.isfinite(maps[fi][wi][2])]).max()
            for key, p in (('tilt', 3), ('focus', 4)):
                got = getattr(wfe, 'rms_' + key)[fi, wi]
                want = ref['rms_' + key]
                kappa = ref['kappa_' + key]
                tol = ((3*depth + 10) + p*ref['cond_' + key])*U*kappa*2
                assert abs(got**2 - want**2) <= tol*want**2 + 1e-300, (key, fi, wi, got, want)
                worst = max(worst, kappa)
            np.testing.assert_allclose([wfe.tilt_x[fi, wi], wfe.tilt_y[fi, wi]], ref['c_tilt'][1:], rtol=1e-8,
                                       atol=1e-9*max(1.0, np.abs(ref['c_tilt']).max()))
            np.testing.assert_allclose(wfe.focus[fi, wi], ref['c_focus'][3], rtol=1e-8,
                                       atol=1e-9*max(1.0, np.abs(ref['c_focus']).max()))
    return worst


WORST_KAPPA = {}


@pytest.mark.parametrize('name', ['dblgauss', 'rc', 'cellphone', 'fisheye'])
def test_wavefront_error_equals_numpy_statistics_of_raygrids(name):
    from test_analyses_vs_reference import OracleBackend
    opm = load_model(name)
    be = OracleBackend(opm)
    num = 24
    fields = opm.optical_spec.field_of_view.fields
    wvls = opm.seq_model.wvlns
    wfe = A.wavefront_error(opm, num, backend=be)
    assert wfe.rms.shape == (len(fields), len(wvls)) and wfe.num_rays == num
    maps = [[A.RayGrid(opm, f=fi, wl=wl, num_rays=num, backend=be).grid for wl in wvls]
            for fi in range(len(fields))]
    WORST_KAPPA[name] = check_against_numpy(wfe, opm, fields, wvls, maps, depth=num*num)
    print(f'{name}: worst kappa of the fits {WORST_KAPPA[name]:.3g}')


def test_wavefront_error_sanity_values():
    """the double Gauss at 64^2, field 0 / 2 at the central wavelength (order of magnitude)"""
    from test_analyses_vs_reference import OracleBackend
    opm = load_model('dblgauss')
    be = OracleBackend(opm)
    wl = opm.seq_model.central_wavelength()
    wfe = A.wavefront_error(opm, 64, wvls=[wl], backend=be)
    np.testing.assert_allclose(wfe.rms[[0, 2], 0], [0.935, 2.13], rtol=0.01)
    np.testing.assert_allclose(wfe.pv[[0, 2], 0], [4.16, 7.07], rtol=0.01)
    np.testing.assert_allclose(wfe.rms_tilt[[0, 2], 0], [0.935, 2.10], rtol=0.01)
    np.testing.assert_allclose(wfe.rms_focus[[0, 2], 0], [0.848, 0.836], rtol=0.01)


# --- ABI ---------------------------------------------------------------------------------------
def test_abi_v6_exports_are_declared():
    hdr = open(os.path.join(ROOT, 'include', 'b200rt.h')).read()
    declared = set(re.findall(r'\b(rt_[a-z0-9_]+)\s*\(', hdr))
    for name in ('rt_grid_wfe_scratch_bytes', 'rt_trace_grid_wfe', 'rt_combine_wfe'):
        assert name in declared and name in _abi.EXPORTS
    assert re.search(r'#define RT_WFE_DOUBLES (\d+)', hdr).group(1) == str(_abi.RT_WFE_DOUBLES)
    assert _abi.RT_ABI_VERSION == 6 == _abi.load_library().rt_abi_version()


def test_abi_bad_arguments_without_a_device():
    lib = _abi.load_library()
    opts = _abi.make_opts()
    out = _abi.rt_out()
    buf = (C.c_double*64)()
    assert lib.rt_trace_grid_wfe(None, None, 0, 0, C.byref(opts), C.byref(out), buf, buf, None) == -1
    assert lib.rt_trace_grid_wfe(C.c_void_p(1), C.c_void_p(1), 0, 0, C.byref(opts), C.byref(out),
                                 None, buf, None) == -1
    assert 'summary' in lib.rt_last_error().decode()
    assert lib.rt_trace_grid_wfe(C.c_void_p(1), C.c_void_p(1), 0, 0, C.byref(opts), C.byref(out),
                                 buf, None, None) == -1
    full = _abi.rt_out()
    full.full = C.cast(buf, C.c_void_p)
    assert lib.rt_trace_grid_wfe(C.c_void_p(1), C.c_void_p(1), 0, 0, C.byref(opts), C.byref(full),
                                 buf, buf, None) == -1
    assert 'full' in lib.rt_last_error().decode()
    assert lib.rt_grid_wfe_scratch_bytes(None, 0, 10) == 0
    assert lib.rt_combine_wfe(None, 1, 1, buf, None) == -1
    assert lib.rt_combine_wfe(buf, 0, 1, buf, None) == -1


def test_combine_summaries_chooses_the_layout_by_width():
    import torch
    rng = np.random.default_rng(5)
    parts = []
    for k in range(3):
        status, w, x, y = adversarial(rng, 300)
        parts.append(WS.ordered_summary(WS.Shape(100, 3), status, w, x, y))
    got = E.combine_summaries(torch.as_tensor(np.stack(parts))).numpy()
    want = WS.combine(parts)
    assert np.array_equal(got[:, :7], want[:, :7])
    np.testing.assert_allclose(got[:, 7:], want[:, 7:], rtol=1e-12, atol=0)
    with pytest.raises(ValueError):
        E.combine_summaries(torch.zeros((2, 3, 17), dtype=torch.float64))
