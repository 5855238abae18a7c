"""Time the wavefront-error table of the double Gauss (3 fields x 3 wavelengths) at num_rays x
num_rays rays per tile:

1. ``analyses.wavefront_error`` end to end (synchronised wall clock, median of --reps);
2. what it replaces: one ``RayGrid`` per tile plus numpy statistics of its OPD map;
3. the kernels alone, with CUDA events over --launches back-to-back launches after a warm-up: the
   wavefront-error trace (``rt_trace_grid_wfe``: trace, sums, reduction) against the existing
   opd grid trace (``rt_trace_grid`` writing per-ray OPD, no sums) over the same grid.

Prints the card name and power limit of this run and writes one JSON line.

    python tools/bench_wavefront_error.py [--num-rays 512] [--reps 5] [--launches 20] [--out FILE]
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
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
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


def per_launch_ms(fn, warmup, launches):
    """CUDA events around ``launches`` back-to-back calls after ``warmup`` calls: ms per call"""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)/launches


def raygrid_statistics(opm, num, fields, wvls):
    """the loop wavefront_error replaces: one RayGrid per tile, statistics of the map in numpy"""
    from rayoptics_b200 import analyses as A
    out = []
    for fi in range(len(fields)):
        for wl in wvls:
            gx, gy, w = A.RayGrid(opm, f=fi, wl=wl, num_rays=num).grid
            m = np.isfinite(w)
            w, x, y = w[m], gx[m], gy[m]
            rms = w.std()
            a3 = np.stack([np.ones_like(x), x, y], axis=1)
            a4 = np.concatenate([a3, (x*x + y*y)[:, None]], axis=1)
            r3 = w - a3 @ np.linalg.lstsq(a3, w, rcond=None)[0]
            r4 = w - a4 @ np.linalg.lstsq(a4, w, rcond=None)[0]
            out.append((rms, w.max() - w.min(), np.sqrt(np.mean(r3*r3)), np.sqrt(np.mean(r4*r4))))
    return np.array(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-rays', type=int, default=512)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    from rayoptics_b200 import model as M, analyses as A, engine as E
    if not torch.cuda.is_available():
        sys.exit('bench_wavefront_error needs a CUDA device')
    opm = M.OpticalModel.load(os.path.join(ROOT, 'tests', 'golden', 'models', 'dblgauss.json'))
    fields, wvls = list(opm.optical_spec.field_of_view.fields), list(opm.seq_model.wvlns)
    n = a.num_rays

    A.wavefront_error(opm, n)                                         # warm-up of this shape
    t_wfe, wfe = timed(lambda: A.wavefront_error(opm, n), a.reps)
    raygrid_statistics(opm, n, fields, wvls)
    t_rg, stats = timed(lambda: raygrid_statistics(opm, n, fields, wvls), a.reps)
    got = np.stack([wfe.rms.ravel(), wfe.pv.ravel(), wfe.rms_tilt.ravel(), wfe.rms_focus.ravel()], axis=1)
    agree = bool(np.allclose(got, stats, rtol=1e-9, atol=0))

    # the kernels on one grid: the WFE trace against the opd trace that writes per-ray OPD
    tab = A._table_for(opm)
    args, kw = A.wavefront_grid_args(opm, tab, n, fields, wvls, opm.optical_spec.defocus.focus_shift)
    grid = E.PupilGrid(*args, device=tab.device, **kw)
    res = E.BundleResult(grid.n_rays, tab.n_ifc, torch.device('cuda', tab.device), ('opd',))
    k_wfe = per_launch_ms(lambda: E.trace_grid_wfe(tab, grid), a.warmup, a.launches)
    k_opd = per_launch_ms(lambda: E.trace_grid(tab, grid, res=res, outputs=('opd',), summary=False),
                          a.warmup, a.launches)
    grid.close()

    rays = len(fields)*len(wvls)*n*n
    rec = {'bench': 'wavefront_error', 'model': 'dblgauss', 'num_rays': n, 'rays': rays, 'card': card(),
           'wavefront_error_s': t_wfe, 'raygrid_loop_s': t_rg, 'ratio': t_rg/t_wfe,
           'kernel_wfe_ms': k_wfe, 'kernel_opd_ms': k_opd, 'kernel_ratio': k_wfe/k_opd,
           'statistics_agree': agree}
    print(f'card: {rec["card"]}')
    print(f'wavefront_error {t_wfe*1e3:9.3f} ms   {len(fields)*len(wvls)} RayGrid + numpy {t_rg*1e3:9.3f} ms   '
          f'ratio {t_rg/t_wfe:6.2f}')
    print(f'kernel: wfe trace + sums {k_wfe:7.3f} ms   opd trace writing per-ray OPD {k_opd:7.3f} ms   '
          f'(wfe / opd {k_wfe/k_opd:5.3f}; {a.launches} launches after {a.warmup})')
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    if not agree:
        sys.exit('wavefront_error does not agree with the RayGrid statistics')


if __name__ == '__main__':
    main()
