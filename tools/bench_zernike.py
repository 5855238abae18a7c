"""Time the Fringe Zernike fit of the double Gauss (3 fields x 3 wavelengths) at num_rays x
num_rays rays per tile, with 37 and with 16 terms:

1. ``analyses.zernike_fit`` end to end (synchronised wall clock, median of --reps);
2. what it replaces: one ``RayGrid`` per tile plus ``numpy.linalg.lstsq`` on its OPD map restricted
   to the unit disk;
3. the kernels alone, with CUDA events over --launches back-to-back calls after a warm-up, repeated
   --rounds times (median, min and max of the rounds): the moments kernel and its reduction
   (``rt_grid_zernike`` on the per-ray opd / status of one trace) against the opd grid trace
   (``rt_trace_grid`` writing per-ray opd and status) over the same grid.

Prints the card name and power limit of this run and writes one JSON line.

    python tools/bench_zernike.py [--num-rays 512] [--reps 5] [--launches 20] [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def timed(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def per_launch_ms(fn, warmup, launches, rounds):
    """CUDA events around ``launches`` back-to-back calls after ``warmup`` calls, ``rounds``
    times: (median, min, max) ms per call"""
    import torch
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1)/launches)
    return float(np.median(out)), float(min(out)), float(max(out))


def raygrid_lstsq(opm, num, fields, wvls, n_terms):
    """the loop zernike_fit replaces: one RayGrid per tile, lstsq of the map on the disk"""
    from rayoptics_b200 import analyses as A, engine as E
    out = []
    for fi in range(len(fields)):
        for wl in wvls:
            gx, gy, w = A.RayGrid(opm, f=fi, wl=wl, num_rays=num).grid
            m = np.isfinite(w) & (gx*gx + gy*gy <= 1.0)
            out.append(np.linalg.lstsq(E.zernike_terms(gx[m], gy[m], n_terms), w[m], rcond=None)[0])
    return np.array(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-rays', type=int, default=512)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    from rayoptics_b200 import model as M, analyses as A, engine as E
    if not torch.cuda.is_available():
        sys.exit('bench_zernike needs a CUDA device')
    opm = M.OpticalModel.load(os.path.join(ROOT, 'tests', 'golden', 'models', 'dblgauss.json'))
    fields, wvls = list(opm.optical_spec.field_of_view.fields), list(opm.seq_model.wvlns)
    n = a.num_rays
    rec = {'bench': 'zernike_fit', 'model': 'dblgauss', 'num_rays': n, 'rays': len(fields)*len(wvls)*n*n,
           'card': card()}
    print(f'card (name, power limit, max SM clock): {rec["card"]}')

    tab = A._table_for(opm)
    args, kw = A.wavefront_grid_args(opm, tab, n, fields, wvls, opm.optical_spec.defocus.focus_shift)
    grid = E.PupilGrid(*args, device=tab.device, **kw)
    res = E.BundleResult(grid.n_rays, tab.n_ifc, torch.device('cuda', tab.device), ('opd', 'status'))
    k_opd = per_launch_ms(lambda: E.trace_grid(tab, grid, res=res, summary=False), a.warmup, a.launches,
                          a.rounds)
    rec['kernel_opd_trace_ms'] = k_opd
    print(f'kernel: opd trace writing per-ray opd + status   {k_opd[0]:7.3f} ms  (min {k_opd[1]:.3f}, '
          f'max {k_opd[2]:.3f})')
    agree_all = True
    for n_terms in (37, 16):
        A.zernike_fit(opm, n, n_terms)                                   # warm-up of this shape
        t_fit, fit = timed(lambda: A.zernike_fit(opm, n, n_terms), a.reps)
        raygrid_lstsq(opm, n, fields, wvls, n_terms)
        t_rg, coef = timed(lambda: raygrid_lstsq(opm, n, fields, wvls, n_terms), a.reps)
        got = fit.coef.reshape(-1, n_terms)
        scale = np.abs(coef).max(axis=1, keepdims=True)
        agree = bool((np.abs(got - coef) <= 1e-8*scale).all())
        agree_all &= agree
        k_z = per_launch_ms(lambda: E.grid_zernike(grid, 0, grid.n_chunks, n_terms, res.status, res.opd),
                            a.warmup, a.launches, a.rounds)
        rec[f'terms_{n_terms}'] = {'zernike_fit_s': t_fit, 'raygrid_lstsq_s': t_rg, 'ratio': t_rg/t_fit,
                                   'kernel_moments_reduce_ms': k_z, 'kernel_ratio_to_opd_trace': k_z[0]/k_opd[0],
                                   'coefficients_agree': agree}
        print(f'{n_terms} terms: zernike_fit {t_fit*1e3:9.3f} ms   {len(fields)*len(wvls)} RayGrid + lstsq '
              f'{t_rg*1e3:9.3f} ms   ratio {t_rg/t_fit:6.2f}   coefficients agree: {agree}')
        print(f'{n_terms} terms: kernel moments + reduce {k_z[0]:7.3f} ms  (min {k_z[1]:.3f}, max {k_z[2]:.3f}; '
              f'/ opd trace {k_z[0]/k_opd[0]:5.3f}; {a.rounds} rounds of {a.launches} launches after {a.warmup})')
    grid.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    if not agree_all:
        sys.exit('zernike_fit does not agree with lstsq on the RayGrid maps')


if __name__ == '__main__':
    main()
