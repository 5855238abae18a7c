"""Time the diffraction MTF of the double Gauss (3 fields x 3 wavelengths) at num_rays x num_rays rays
per tile (default 64 and 256):

1. ``analyses.mtf`` end to end (synchronised wall clock, median of --reps);
2. what it replaces: one ``RayGrid`` per tile, ``calc_psf`` of its wavefront map (maxdim = 2 x
   num_rays) and a numpy FFT of that PSF, whose axis slices are the MTF;
3. the kernels alone, with CUDA events over --launches back-to-back calls after a warm-up, repeated
   --rounds times (median, min and max of the rounds): the pupil function and the autocorrelation
   (``rt_grid_pupil_function`` + ``rt_grid_mtf`` on the per-ray opd / status of one trace) against the
   opd grid trace over the same grid.

The two routes are compared on the axial tile: the PSF route's MTF at the device's native shifts
(its frequency grid is the same when maxdim = 2 x num_rays, up to the reference's zeroing of pupil
values equal to 1).  Prints the card name and power limit of this run and writes one JSON line.

    python tools/bench_mtf.py [--num-rays 64 256] [--reps 5] [--launches 20] [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_zernike import card, timed, per_launch_ms       # noqa: E402


def psf_route(opm, num, fields, wvls):
    """the route ``mtf`` replaces: RayGrid + calc_psf + numpy FFT of the PSF, per tile; returns the
    MTF slices along pupil x and y at shifts 0 ... num-1, [n_tiles, 2, num]"""
    from rayoptics_b200 import analyses as A
    out = []
    for fi in range(len(fields)):
        for wl in wvls:
            w = A.RayGrid(opm, f=fi, wl=wl, num_rays=num).grid[2]
            psf = A.calc_psf(w, num, 2*num)
            otf = np.fft.fft2(np.fft.ifftshift(psf))
            m = np.abs(otf)/np.abs(otf[0, 0])
            out.append([m[:num, 0], m[0, :num]])
    return np.array(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-rays', type=int, nargs='+', default=[64, 256])
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    from rayoptics_b200 import model as M, analyses as A, engine as E
    if not torch.cuda.is_available():
        sys.exit('bench_mtf needs a CUDA device')
    opm = M.OpticalModel.load(os.path.join(ROOT, 'tests', 'golden', 'models', 'dblgauss.json'))
    fields, wvls = list(opm.optical_spec.field_of_view.fields), list(opm.seq_model.wvlns)
    rec = {'bench': 'mtf', 'model': 'dblgauss', 'tiles': len(fields)*len(wvls), 'card': card()}
    print(f'card (name, power limit, max SM clock): {rec["card"]}')
    tab = A._table_for(opm)
    lam = np.array([[opm.nm_to_sys_units(w) for w in wvls]]*len(fields)).ravel()
    for n in a.num_rays:
        args, kw = A.wavefront_grid_args(opm, tab, n, fields, wvls, opm.optical_spec.defocus.focus_shift)
        grid = E.PupilGrid(*args, device=tab.device, **kw)
        res = E.BundleResult(grid.n_rays, tab.n_ifc, torch.device('cuda', tab.device), ('opd', 'status'))
        E.trace_grid(tab, grid, res=res, summary=False)
        k_opd = per_launch_ms(lambda: E.trace_grid(tab, grid, res=res, summary=False), a.warmup, a.launches,
                              a.rounds)

        def kernels():
            P, PT = E.grid_pupil_function(grid, res.status, res.opd, lam)
            return E.grid_mtf(grid, res.status, P, PT)
        k_mtf = per_launch_ms(kernels, a.warmup, a.launches, a.rounds)
        A.mtf(opm, n)                                                    # warm-up of this shape
        t_mtf, r = timed(lambda: A.mtf(opm, n), a.reps)
        psf_route(opm, n, fields, wvls)
        t_psf, m_psf = timed(lambda: psf_route(opm, n, fields, wvls), a.reps)
        diff = float(max(np.abs(m_psf[0, 0] - r.mtf_x[0, 0]).max(), np.abs(m_psf[0, 1] - r.mtf_y[0, 0]).max()))
        rec[f'n{n}'] = {'rays': grid.n_rays, 'mtf_s': t_mtf, 'raygrid_psf_fft_s': t_psf, 'ratio': t_psf/t_mtf,
                        'kernel_pupil_mtf_ms': k_mtf, 'kernel_opd_trace_ms': k_opd,
                        'axial_max_mtf_difference_to_psf_route': diff}
        print(f'{n}^2: mtf {t_mtf*1e3:9.3f} ms   {rec["tiles"]} RayGrid + calc_psf + FFT {t_psf*1e3:9.3f} ms   '
              f'ratio {t_psf/t_mtf:7.2f}   axial max |MTF difference| {diff:.2e}')
        print(f'{n}^2: kernels pupil function + mtf {k_mtf[0]:8.3f} ms  (min {k_mtf[1]:.3f}, max {k_mtf[2]:.3f}); '
              f'opd trace {k_opd[0]:.3f} ms; {a.rounds} rounds of {a.launches} launches after {a.warmup}')
        grid.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
