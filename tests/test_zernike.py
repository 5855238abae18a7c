"""CPU: the Fringe Zernike polynomials (engine.zernike_terms and csrc/rt_zernike.cuh through
tests/hostsim), the Zernike moments restated in tests/zernike_sums.py, engine.zernike_statistics,
the host logic of analyses.zernike_fit through the backend= seam with the oracle, and the ABI
surface of rt_grid_zernike.

Bound of the fit against lstsq.  The normal equations are solved on the Gram matrix scaled to unit
diagonal; with sums accurate to gamma_d relative to sum |a_i a_j| the coefficients of that solve are
off by about (d + p)·u·cond relative, cond the condition number of the scaled Gram matrix, p the
number of terms.  The tests use 4·(d + p)·u·cond·max|c|, and never more than 1e-8·max|c|."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import zernike_sums as ZS
from conftest import ROOT, load_model
from rayoptics_b200 import _abi, analyses as A, engine as E

U = 2.0**-53


def fringe_list():
    """(n, m) of the Fringe order: groups d = (n + m)/2 = 0 ... 5 with m from d down to 0 (cos,
    then sin), then (12, 0)"""
    out = []
    for d in range(6):
        for m in range(d, -1, -1):
            out += [(2*d - m, m)] * (1 if m == 0 else 2)
    return out + [(12, 0)]


def radial(n, m, rho):
    return sum((-1)**s*math.factorial(n - s)/(math.factorial(s)*math.factorial((n + m)//2 - s)
                                              *math.factorial((n - m)//2 - s))*rho**(n - 2*s)
               for s in range((n - m)//2 + 1))


def disk_points(rng, n):
    r = np.sqrt(rng.uniform(0, 1, n))
    t = rng.uniform(-np.pi, np.pi, n)
    return r*np.cos(t), r*np.sin(t)


# --- the polynomials ---------------------------------------------------------------------------
def test_table_is_the_fringe_list():
    assert [(n, m) for n, m, _, _ in E.FRINGE_TERMS] == fringe_list()
    kinds = [k for _, _, k, _ in E.FRINGE_TERMS]
    for j, (n, m, k, a) in enumerate(E.FRINGE_TERMS):
        assert (k is None) == (m == 0)
        if m and kinds[j - 1] != 'cos':
            assert k == 'cos'                # a cos term first, its sin twin next
        assert len(a) == (n - m)//2 + 1


def test_terms_equal_the_factorial_formula():
    rng = np.random.default_rng(1)
    x, y = disk_points(rng, 2000)
    z = E.zernike_terms(x, y, 37)
    rho, th = np.hypot(x, y), np.arctan2(y, x)
    for j, (n, m, k, _) in enumerate(E.FRINGE_TERMS):
        ang = 1.0 if m == 0 else (np.cos(m*th) if k == 'cos' else np.sin(m*th))
        want = radial(n, m, rho)*ang
        assert np.abs(z[:, j] - want).max() <= 1e-11, (j + 1, n, m)
    assert np.array_equal(z[:, 1], x) and np.array_equal(z[:, 2], y)      # theta from +x


def test_terms_are_orthogonal_on_the_disk():
    """Gauss-Legendre in rho (weight rho) x the trapezoid in theta, exact for these degrees"""
    g, wg = np.polynomial.legendre.leggauss(20)
    rho, wr = (g + 1)/2, wg/2*(g + 1)/2
    nt = 64
    th = np.arange(nt)*2*np.pi/nt
    R, T = np.meshgrid(rho, th, indexing='ij')
    wgt = (wr[:, None]*np.full(nt, 2*np.pi/nt)[None, :]).ravel()
    z = E.zernike_terms((R*np.cos(T)).ravel(), (R*np.sin(T)).ravel(), 37)
    gram = (z*wgt[:, None]).T @ z
    norm = np.array([np.pi/(n + 1)*(1.0 if m == 0 else 0.5) for n, m, _, _ in E.FRINGE_TERMS])
    assert np.abs(np.diag(gram) - norm).max() < 1e-12
    off = gram - np.diag(np.diag(gram))
    assert np.abs(off).max() < 1e-12


def edge_points():
    """points with r2 exactly 1 and their neighbouring doubles, the axes, signed zeros"""
    one = np.array([1.0, np.nextafter(1.0, 0), np.nextafter(1.0, 2)])
    xs = np.concatenate([one, -one, [0.0, -0.0, 0.6, -0.6, 0.8, np.sqrt(0.5)]])
    ys = np.concatenate([[0.0]*6, [1.0, -1.0, 0.8, -0.8, 0.6, np.sqrt(0.5)]])
    x, y = np.meshgrid(xs, ys, indexing='ij')
    return x.ravel(), y.ravel()


def test_device_source_equals_the_restatement_bit_for_bit():
    from hostsim import zernike_build as ZB
    assert ZB.fringe_table() == list(E.FRINGE_TERMS)
    rng = np.random.default_rng(2)
    x, y = disk_points(rng, 5000)
    x = np.concatenate([x, edge_points()[0], rng.uniform(-1.5, 1.5, 500)])
    y = np.concatenate([y, edge_points()[1], rng.uniform(-1.5, 1.5, 500)])
    r2 = x*x + y*y
    assert (r2 == 1.0).any() and ((r2 > 1.0) & (r2 < 1 + 1e-15)).any() and ((r2 < 1.0) & (r2 > 1 - 1e-15)).any()
    for n_terms in (1, 4, 16, 37):
        got = ZB.zernike_terms(x, y, n_terms)
        want = E.zernike_terms(x, y, n_terms)
        assert got.view(np.uint64).tolist() == want.view(np.uint64).tolist(), n_terms


# --- the restatement of the moments --------------------------------------------------------------
def adversarial(rng, n, edge=True):
    """OPDs with magnitudes 1e-9 to 1e3, cancellation, signed zeros; pupil points inside and
    outside the disk, some exactly on it; statuses of every class"""
    w = rng.standard_normal(n)*10.0**rng.integers(-9, 4, n)
    w[rng.random(n) < 0.1] *= -1e3
    w[rng.random(n) < 0.05] = -0.0
    w[rng.random(n) < 0.05] = 0.0
    x, y = rng.uniform(-1.2, 1.2, (2, n))
    if edge:
        ex, ey = edge_points()
        k = rng.integers(0, len(ex), n//10)
        at = rng.choice(n, n//10, replace=False)
        x[at], y[at] = ex[k], ey[k]
    status = np.where(rng.random(n) < 0.8, 0, rng.integers(-2, 7, n))
    return status, w, x, y


@pytest.mark.parametrize('n_terms', [1, 4, 16, 37])
@pytest.mark.parametrize('rays_per_tile, n_tiles, rng_range', [
    (1, 3, None), (33*33, 2, None), (64*64, 3, (5, 27)), (64*64, 2, (9, 9)), (700, 3, (1, 8))])
def test_ordered_sums_within_bound_of_exact(rays_per_tile, n_tiles, rng_range, n_terms):
    rng = np.random.default_rng(rays_per_tile + n_tiles + n_terms)
    shape = ZS.Shape(rays_per_tile, n_tiles, *(rng_range or (0, None)))
    status, w, x, y = adversarial(rng, shape.n_rays)
    got = ZS.ordered_summary(shape, status, w, x, y, n_terms)
    want, absum = ZS.exact_summary(shape, status, w, x, y, n_terms)
    assert (got[:, :8] == want[:, :8]).all()
    cols = ZS.sum_cols(n_terms)
    err = np.abs(got[:, cols] - want[:, cols])
    assert (err <= ZS.sum_bound(absum, ZS.chain_depth(shape))).all()
    assert (got[:, cols[-1] + 1:] == 0).all()
    if shape.chunk_end == shape.chunk_begin:
        assert np.array_equal(got, ZS.identity(n_tiles))


def test_chains_are_sequential_not_pairwise():
    """np.cumsum from +0.0 is the kernel's chain: equal to a plain loop, and different from np.sum
    on data where the order shows"""
    rng = np.random.default_rng(4)
    v = rng.standard_normal((300, 5))*10.0**rng.integers(-8, 8, (300, 5))
    loop = np.zeros(5)
    for r in range(len(v)):
        loop = loop + v[r]
    assert ZS.chained(v, 0).view(np.uint64).tolist() == loop.view(np.uint64).tolist()
    pairwise = np.sum(np.ascontiguousarray(v.T), axis=1)                  # along the contiguous axis
    assert ZS.chained(v, 0).view(np.uint64).tolist() != pairwise.view(np.uint64).tolist()
    assert not np.signbit(ZS.chained(np.full((3, 1), -0.0), 0)).any()       # starts from +0.0


def test_plausible_mistakes_change_the_bits():
    rng = np.random.default_rng(11)
    shape = ZS.Shape(40*40, 2)
    status, w, x, y = adversarial(rng, shape.n_rays)
    J = 16
    good = ZS.ordered_summary(shape, status, w, x, y, J)
    bits = lambda s: s.view(np.uint64).tolist()         # noqa: E731
    for kw in ({'reverse_rays': True}, {'drop_chunk': 3}, {'transposed': True}, {'strict': True}):
        assert bits(ZS.ordered_summary(shape, status, w, x, y, J, **kw)) != bits(good), kw
    assert bits(ZS.ordered_summary(shape, status, w, y, x, J)) != bits(good)       # x and y swapped
    parts = [ZS.ordered_summary(shape.sub(a, b), *_slice(shape, a, b, status, w, x, y), J)
             for a, b in ((0, 2), (2, 4), (4, shape.n_chunks))]          # three parts of tile 0
    assert bits(ZS.combine(parts[::-1])) != bits(ZS.combine(parts))                # parts out of order


def _slice(shape, a, b, *arrays):
    i, j = shape.first_ray(a), shape.first_ray(b)
    return tuple(np.asarray(v)[i:j] for v in arrays)


# --- zernike_statistics ----------------------------------------------------------------------------
def record(w, x, y, n_terms, status=None):
    status = np.zeros(len(w), int) if status is None else status
    s, _ = ZS.exact_summary(ZS.Shape(len(w), 1), status, w, x, y, n_terms)
    return s


def disk_grid(num):
    g = np.linspace(-1, 1, num)
    x, y = (v.ravel() for v in np.meshgrid(g, g, indexing='ij'))
    keep = x*x + y*y <= 1.0
    return x[keep], y[keep]


@pytest.mark.parametrize('n_terms', [4, 16, 37])
def test_statistics_recover_known_coefficients(n_terms):
    rng = np.random.default_rng(n_terms)
    x, y = disk_grid(81)
    lam = 5.5e-4
    c = rng.uniform(-2, 2, n_terms)                     # waves
    w = (E.zernike_terms(x, y, n_terms) @ c)*lam
    st = E.zernike_statistics(record(w, x, y, n_terms), lam, n_terms)
    assert np.abs(st['coef'][0] - c).max() <= 1e-10
    assert st['rms_residual'][0] <= 1e-6*st['rms'][0]
    np.testing.assert_allclose(st['rms'][0], np.std(w/lam), rtol=1e-9)
    np.testing.assert_allclose(st['pv'][0], (w.max() - w.min())/lam, rtol=1e-12)
    assert st['n_used'][0] == len(x) == st['n_ok'][0]


def test_statistics_nan_when_short_of_rays():
    x, y = disk_points(np.random.default_rng(8), 13)
    w = 1e-3*(x + y*y)
    s13 = record(w, x, y, 16)
    s_none = record(w[:3], x[:3], y[:3], 16, status=np.array([1, 2, 3]))
    s_nan = record(np.where(np.arange(len(w)) == 4, np.nan, w), x, y, 4)
    st = E.zernike_statistics(s13, 1e-3, 16)
    assert np.isnan(st['coef']).all() and np.isnan(st['rms_residual']).all() and np.isfinite(st['rms']).all()
    st = E.zernike_statistics(s13, 1e-3, 13)            # 13 rays, 13 terms: determined
    assert np.isfinite(st['coef']).all()
    st = E.zernike_statistics(s_none, 1e-3, 16)
    assert st['n_used'][0] == 0 and np.isnan(st['rms'][0]) and np.isnan(st['coef']).all()
    assert (st['n_missed'][0], st['n_tir'][0], st['n_blocked'][0]) == (1, 1, 1)
    st = E.zernike_statistics(s_nan, 1e-3, 4)
    assert np.isnan(st['coef']).all() and np.isnan(st['rms'][0]) and np.isfinite(st['pv'][0])


def test_statistics_accept_torch_tensors():
    import torch
    x, y = disk_grid(11)
    s = record(0.01*x*y + 0.02*(x*x + y*y), x, y, 9)
    a = E.zernike_statistics(s, 1e-3, 9)
    b = E.zernike_statistics(torch.as_tensor(s), 1e-3, 9)
    for k in a:
        assert torch.is_tensor(b[k])
        np.testing.assert_array_equal(b[k].numpy(), a[k])


# --- zernike_fit through the backend seam --------------------------------------------------------
def lstsq_fit(grid, n_terms):
    """least squares of a RayGrid map restricted to the unit disk: (coefficients, cond of the
    scaled Gram matrix, n)"""
    gx, gy, opd = grid
    m = np.isfinite(opd) & (gx*gx + gy*gy <= 1.0)
    Z = E.zernike_terms(gx[m], gy[m], n_terms)
    c, *_ = np.linalg.lstsq(Z, opd[m], rcond=None)
    G = Z.T @ Z
    d = np.sqrt(np.diag(G))
    return c, np.linalg.cond(G/np.outer(d, d)), int(m.sum())


def check_against_lstsq(fit, opm, fields, wvls, maps, depth):
    """every tile's coefficients against lstsq on its RayGrid map; returns the worst tolerance
    used, relative to the tile's largest |coefficient|"""
    worst = 0.0
    for fi in range(len(fields)):
        for wi, wl in enumerate(wvls):
            c, cond, n = lstsq_fit(maps[fi][wi], fit.num_terms)
            assert fit.n_used[fi, wi] == n
            if n < fit.num_terms:
                assert np.isnan(fit.coef[fi, wi]).all()
                continue
            scale = np.abs(c).max()                      # RayGrid maps are in waves
            tol = min(4*(depth + fit.num_terms)*U*cond, 1e-8)
            worst = max(worst, tol)
            assert np.abs(fit.coef[fi, wi] - c).max() <= tol*scale, (fi, wi, cond)
    return worst


@pytest.mark.parametrize('n_terms', [4, 37])
@pytest.mark.parametrize('name', ['dblgauss', 'rc', 'cellphone', 'fisheye'])
def test_zernike_fit_equals_lstsq_on_raygrids(name, n_terms):
    from test_analyses_vs_reference import OracleBackend
    opm = load_model(name)
    be = OracleBackend(opm)
    num = 24
    fields, wvls = opm.optical_spec.field_of_view.fields, opm.seq_model.wvlns
    fit = A.zernike_fit(opm, num, n_terms, backend=be)
    assert fit.coef.shape == (len(fields), len(wvls), n_terms) and fit.num_terms == n_terms
    maps = [[A.RayGrid(opm, f=fi, wl=wl, num_rays=num, backend=be).grid for wl in wvls]
            for fi in range(len(fields))]
    worst = check_against_lstsq(fit, opm, fields, wvls, maps, depth=num*num)
    print(f'{name}, {n_terms} terms: worst relative tolerance {worst:.3g}')


def test_four_terms_span_the_focus_fit():
    """{Z1, Z2, Z3, Z4} span {1, x, y, r^2}: where every status-0 ray is inside the disk the
    residual equals wavefront_error's rms_focus"""
    from test_analyses_vs_reference import OracleBackend
    opm = load_model('dblgauss')
    be = OracleBackend(opm)
    fit = A.zernike_fit(opm, 32, 4, backend=be)
    wfe = A.wavefront_error(opm, 32, backend=be)
    inside = fit.n_used == wfe.n_ok
    assert inside.sum() >= 3
    np.testing.assert_allclose(fit.rms_residual[inside], wfe.rms_focus[inside], rtol=1e-7)
    np.testing.assert_allclose(fit.rms[inside], wfe.rms[inside], rtol=1e-9)
    np.testing.assert_allclose(fit.coef[..., 3][inside], (wfe.focus[inside])/2, rtol=1e-7)


def test_symmetry_of_the_double_gauss():
    """for fields on the y axis the terms odd in x vanish (cos with odd m, sin with even m).  On
    axis the m != 0 terms vanish, except cos(4 theta) ones: the square grid of pupil samples is
    itself invariant under quarter turns and mirrors, so the radial part the 37 terms cannot
    represent aliases into cos(4 theta), at 1e-7 of the largest term here"""
    from test_analyses_vs_reference import OracleBackend
    opm = load_model('dblgauss')
    be = OracleBackend(opm)
    fit = A.zernike_fit(opm, 33, 37, backend=be)
    fields = opm.optical_spec.field_of_view.fields
    odd_x = [j for j, (n, m, k, _) in enumerate(E.FRINGE_TERMS)
             if (k == 'cos' and m % 2 == 1) or (k == 'sin' and m % 2 == 0)]
    not_round = [j for j, (n, m, k, _) in enumerate(E.FRINGE_TERMS) if m != 0 and not (m == 4 and k == 'cos')]
    square = [j for j, (n, m, k, _) in enumerate(E.FRINGE_TERMS) if m == 4 and k == 'cos']
    for fi, f in enumerate(fields):
        assert f.x == 0.0
        for wi in range(fit.n_wvls):
            c = fit.coef[fi, wi]
            big = np.abs(c).max()
            assert np.abs(c[odd_x]).max() <= 1e-9*big, (fi, wi)
            if f.y == 0.0:
                assert np.abs(c[not_round]).max() <= 1e-9*big, (fi, wi)
                assert np.abs(c[square]).max() <= 1e-6*big, (fi, wi)


# --- ABI -----------------------------------------------------------------------------------------
def test_abi_exports_are_declared():
    hdr = open(os.path.join(ROOT, 'include', 'b200rt.h')).read()
    declared = set(re.findall(r'\b(rt_[a-z0-9_]+)\s*\(', hdr))
    for name in ('rt_grid_zernike_scratch_bytes', 'rt_grid_zernike', 'rt_combine_zernike'):
        assert name in declared and name in _abi.EXPORTS
    assert re.search(r'#define RT_ZERN_DOUBLES (\d+)', hdr).group(1) == str(_abi.RT_ZERN_DOUBLES)
    assert re.search(r'#define RT_ZERN_MAX_TERMS (\d+)', hdr).group(1) == str(_abi.RT_ZERN_MAX_TERMS)
    assert _abi.RT_ABI_VERSION == 6


def test_abi_bad_arguments_without_a_device():
    lib = _abi.load_library()
    buf = (C.c_double*64)()
    st = (C.c_int32*64)()
    fake = C.c_void_p(1)
    assert lib.rt_grid_zernike(None, 0, 1, 4, st, buf, buf, buf, None) == -1
    assert lib.rt_grid_zernike(fake, 0, 1, 4, st, buf, None, buf, None) == -1
    assert 'summary' in lib.rt_last_error().decode()
    for n_terms in (0, -1, 38):
        assert lib.rt_grid_zernike(fake, 0, 1, n_terms, st, buf, buf, buf, None) == -1
        assert 'n_terms' in lib.rt_last_error().decode()
    assert lib.rt_grid_zernike_scratch_bytes(None, 0, 10, 4) == 0
    assert lib.rt_combine_zernike(None, 1, 1, buf, None) == -1
    assert lib.rt_combine_zernike(buf, 0, 1, buf, None) == -1
    with pytest.raises(ValueError):
        E.zernike_terms(0.0, 0.0, 38)
    with pytest.raises(ValueError):
        A.zernike_fit(load_model('singlet'), 8, 0)


def test_combine_summaries_chooses_the_layout_by_width():
    import torch
    rng = np.random.default_rng(5)
    parts = []
    for k in range(3):
        status, w, x, y = adversarial(rng, 300)
        parts.append(ZS.ordered_summary(ZS.Shape(100, 3), status, w, x, y, 6))
    got = E.combine_summaries(torch.as_tensor(np.stack(parts))).numpy()
    want = ZS.combine(parts)
    assert np.array_equal(got[:, :8], want[:, :8])
    np.testing.assert_allclose(got[:, 8:], want[:, 8:], rtol=1e-12, atol=0)
