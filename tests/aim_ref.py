"""Restatement of the chief-ray aiming of csrc/rt_aim.cuh (rt_grid_aim_chief) in numpy.

The iteration is vigcalc.aim_all_fields_batched's, field by field in lock step, with the 2x2 solve
of rt_aim.cuh (``solve2``) in place of np.linalg.solve and the termination of every field recorded.
It is driven by a ``stop_xy(idx, aims)`` function: the stop intercepts ``[k, 2]`` of the (0, 0)
pupil rays of fields ``idx`` aimed at ``aims`` (NaN rows where a ray does not reach the stop).
``oracle_stop_xy`` traces them with oracle/rt_oracle.c through the whole system, as
``cuda_bundle_fn`` does, and reads segment ``stop``.
"""
from __future__ import annotations

import numpy as np

# enum rt_aim_term (include/b200rt.h)
CONVERGED, FIRST_FAILED, DIFF_FAILED, SINGULAR, NO_STEP, MAX_ITER = range(6)
TERM_NAMES = ('converged', 'first ray failed', 'difference ray failed', 'singular', 'no step accepted',
              'max_iter')


def _finite(v):
    return bool(np.isfinite(v))


def solve2(a, b, c, d, r0, r1):
    """aim_solve2 of rt_aim.cuh: [[a, b], [c, d]] s = [r0, r1] by elimination with partial pivoting
    (rows swap only when |c| > |a|), every operation a float64 operation; None when singular"""
    a, b, c, d, r0, r1 = (np.float64(v) for v in (a, b, c, d, r0, r1))
    if abs(c) > abs(a):
        a, b, c, d, r0, r1 = c, d, a, b, r1, r0
    if a == 0.0:
        return None
    l = c/a
    u = d - l*b
    if u == 0.0:
        return None
    y1 = r1 - l*r0
    s1 = y1/u
    s0 = (r0 - b*s1)/a
    if not (_finite(s0) and _finite(s1)):
        return None
    return s0, s1


def _norm(f):
    return max(abs(f[0]), abs(f[1]))


def aim_fields(stop_xy, n, h, tol=1e-13, max_iter=30):
    """aim points ``[n, 2]`` (no x == 0 rule), termination codes ``[n]`` and accepted Newton steps
    ``[n]`` of ``n`` fields"""
    h = np.float64(h)
    x = np.zeros((n, 2))
    term = np.full(n, MAX_ITER, dtype=np.int32)
    iters = np.zeros(n, dtype=np.int32)
    f = np.asarray(stop_xy(list(range(n)), x.copy()), dtype=np.float64)
    active = []
    for i in range(n):
        if np.isfinite(f[i]).all():
            active.append(i)
        else:
            term[i] = FIRST_FAILED
    for _ in range(max_iter):
        still = []
        for i in active:
            if _norm(f[i]) < tol:
                term[i] = CONVERGED
            else:
                still.append(i)
        active = still
        if not active:
            break
        fa = stop_xy(active, np.array([[x[i, 0] + h, x[i, 1] + 0.0] for i in active]))
        fb = stop_xy(active, np.array([[x[i, 0] + 0.0, x[i, 1] + h] for i in active]))
        steps = {}
        for k, i in enumerate(active):
            if not (np.isfinite(fa[k]).all() and np.isfinite(fb[k]).all()):
                term[i] = DIFF_FAILED
                continue
            j00, j10 = (fa[k, 0] - f[i, 0])/h, (fa[k, 1] - f[i, 1])/h
            j01, j11 = (fb[k, 0] - f[i, 0])/h, (fb[k, 1] - f[i, 1])/h
            s = solve2(j00, j01, j10, j11, -f[i, 0], -f[i, 1])
            if s is None:
                term[i] = SINGULAR
                continue
            steps[i] = s
        lam = {i: np.float64(1.0) for i in steps}
        pending, accepted = list(steps), []
        for _bt in range(20):
            if not pending:
                break
            trial = np.array([[x[i, 0] + lam[i]*steps[i][0], x[i, 1] + lam[i]*steps[i][1]] for i in pending])
            got = stop_xy(pending, trial)
            nxt = []
            for k, i in enumerate(pending):
                if np.isfinite(got[k]).all() and _norm(got[k]) < _norm(f[i]):
                    x[i], f[i] = trial[k], got[k]
                    accepted.append(i)
                    iters[i] += 1
                else:
                    lam[i] *= 0.5
                    nxt.append(i)
            pending = nxt
        for i in pending:
            term[i] = NO_STEP
        active = accepted
    return x, term, iters


def oracle_stop_xy(opm, fields, wvl=None):
    """``stop_xy`` of ``fields`` traced by the oracle: the start rays of grid_start_ray_at (the
    oracle's restatement) with the trial aims in the field records, traced through the whole
    system (first_surf 1, apertures not checked), intercept at segment ``stop``"""
    from oracle import rt_oracle
    from rayoptics_b200 import _abi, engine as E, table as T
    from rayoptics_b200.opticalspec import grid_fields_of
    osp, sm = opm.optical_spec, opm.seq_model
    wvl = osp.spectral_region.central_wvl if wvl is None else wvl
    stop = sm.stop_surface
    descs, n_by_wvl, wvls = T.describe_model(sm)
    recs, eprad, z_pupil = grid_fields_of(opm, fields)
    wi = sm.index_for_wavelength(wvl)
    opts = _abi.make_opts(first_surf=1, last_surf=len(descs) - 2)

    def fn(idx, aims):
        rs = [dict(recs[i], aim=[float(a[0]), float(a[1])]) for i, a in zip(idx, aims)]
        out = np.full((len(rs), 2), np.nan)
        if not rs:
            return out
        spec = E.PupilGridSpec(rs, [wi], [0.0], [0.0], eprad, z_pupil, apply_vignetting=False,
                               flip_z_dir=sm.z_dir[0])
        p, d, wv, _ = rt_oracle.grid_start_rays(spec.c_spec(), 0, spec.n_rays)
        r = rt_oracle.trace_bundle(descs, n_by_wvl, p, d, wv, opts, want_full=True, wvls=wvls)
        ok = r['n_seg'] > stop
        out[ok] = r['full'][stop, 0:2, :].T[ok]
        return out
    return fn


def aim_step(opm):
    """h of aim_chief_ray: 1e-4*max(1, enp_radius)"""
    return 1e-4*max(1.0, opm.optical_spec.fod.enp_radius)


def restate(opm, fields, wvl=None, tol=1e-13, max_iter=30):
    """``aim_fields`` of ``fields`` on the oracle: ``(aim [n, 2], term [n], iters [n])``"""
    return aim_fields(oracle_stop_xy(opm, fields, wvl), len(fields), aim_step(opm), tol, max_iter)
