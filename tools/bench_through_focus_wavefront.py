"""Time the through-focus wavefront analysis of the double Gauss (3 fields x 3 wavelengths, 21 focus
planes over +-0.1 mm, freqs 25 / 50 / 100 cycles/mm) at num_rays x num_rays rays per tile (default 64
and 256):

1. ``analyses.through_focus_wavefront`` end to end (synchronised wall clock, median of --reps);
2. the device route without it: K x (``zernike_fit`` + ``mtf``), each of which traces the grid again;
3. at --host-rays only (default 32): the reference's rapid-refocus route on the host, one
   ``trace_wavefront`` per tile and K x ``focus_wavefront`` per tile (the numpy statistics are not
   included: the route is already orders of magnitude slower);
4. the kernels alone, with CUDA events over --launches back-to-back calls after a warm-up, repeated
   --rounds times (median, min and max of the rounds): the opd-focus trace against the single-focus
   opd trace, the per-plane consumers (Zernike moments, pupil function, autocorrelation at the listed
   shifts), and ``rt_grid_mtf_shifts`` against ``rt_grid_mtf``.

Prints the card name and power limit of this run and writes one JSON line.

    python tools/bench_through_focus_wavefront.py [--num-rays 64 256] [--planes 21] [--reps 5] [--out FILE]
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

FREQS = [25.0, 50.0, 100.0]


def host_route(opm, num, fields, wvls, focs):
    from rayoptics_b200 import analyses as A
    for fld in fields:
        for wl in wvls:
            pkg = A.trace_wavefront(opm, fld, wl, focs[0], num_rays=num)
            for f in focs:
                A.focus_wavefront(opm, pkg, fld, wl, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-rays', type=int, nargs='+', default=[64, 256])
    ap.add_argument('--planes', type=int, default=21)
    ap.add_argument('--host-rays', type=int, default=32)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    from rayoptics_b200 import model as M, analyses as A, engine as E, waveabr as W
    if not torch.cuda.is_available():
        sys.exit('bench_through_focus_wavefront needs a CUDA device')
    opm = M.OpticalModel.load(os.path.join(ROOT, 'tests', 'golden', 'models', 'dblgauss.json'))
    fields, wvls = list(opm.optical_spec.field_of_view.fields), list(opm.seq_model.wvlns)
    focs = list(np.linspace(-0.1, 0.1, a.planes))
    K = len(focs)
    rec = {'bench': 'through_focus_wavefront', 'model': 'dblgauss', 'tiles': len(fields)*len(wvls), 'planes': K,
           'freqs': FREQS, 'card': card()}
    print(f'card (name, power limit, max SM clock): {rec["card"]}')
    tab = A._table_for(opm)
    dev = torch.device('cuda', tab.device)
    lam = np.array([[opm.nm_to_sys_units(w) for w in wvls]]*len(fields)).ravel()
    for n in a.num_rays:
        r = {}
        tfw = lambda: A.through_focus_wavefront(opm, n, foc=focs, freqs=FREQS)        # noqa: E731
        tfw()
        r['through_focus_wavefront_s'], out = timed(tfw, a.reps)

        def per_plane():
            for f in focs:
                A.zernike_fit(opm, n, 9, foc=f)
                A.mtf(opm, n, foc=f, freqs=FREQS)
        per_plane()
        r['k_zernike_fit_mtf_s'], _ = timed(per_plane, max(1, a.reps//2))
        r['ratio_per_plane'] = r['k_zernike_fit_mtf_s']/r['through_focus_wavefront_s']
        # kernels
        wave, ref_img, spheres, _ = W.setup_tiles_focus(opm, tab, fields, wvls, focs)
        args, kw = A._wavefront_grid_args(opm, tab, n, fields, wvls, focs[0], wave[0], ref_img[0])
        grid = E.PupilGrid(*args, device=tab.device, **kw)
        sph = torch.as_tensor(spheres.reshape(K, grid.n_tiles, -1), device=dev)
        res = E.BundleResult(grid.n_rays, tab.n_ifc, dev, ('opd', 'status'))
        st = E.BundleResult(grid.n_rays, tab.n_ifc, dev, ('status',))
        r['kernel_opd_focus_trace_ms'] = per_launch_ms(lambda: E.trace_grid_opd_focus(tab, grid, sph, res=st),
                                                       a.warmup, a.launches, a.rounds)
        r['kernel_opd_trace_ms'] = per_launch_ms(lambda: E.trace_grid(tab, grid, res=res, summary=False),
                                                 a.warmup, a.launches, a.rounds)
        planes, _ = E.trace_grid_opd_focus(tab, grid, sph, res=st)
        shifts = torch.as_tensor(out.shifts.astype(np.int32), device=dev)
        pup = E.grid_pupil_function(grid, st.status, planes[0], lam)

        def consumers():
            E.grid_zernike(grid, 0, grid.n_chunks, 9, st.status, planes[0])
            E.grid_pupil_function(grid, st.status, planes[0], lam, out=pup)
            E.grid_mtf_shifts(grid, st.status, pup[0], pup[1], shifts)
        r['kernel_per_plane_consumers_ms'] = per_launch_ms(consumers, a.warmup, a.launches, a.rounds)
        r['kernel_mtf_shifts_ms'] = per_launch_ms(lambda: E.grid_mtf_shifts(grid, st.status, pup[0], pup[1], shifts),
                                                  a.warmup, a.launches, a.rounds)
        r['kernel_mtf_all_shifts_ms'] = per_launch_ms(lambda: E.grid_mtf(grid, st.status, pup[0], pup[1]),
                                                      a.warmup, a.launches, a.rounds)
        r['n_shifts'] = int(len(shifts))
        r['opd_planes_bytes'] = K*grid.n_rays*8
        grid.close()
        if n == a.host_rays:
            host_route(opm, n, fields[:1], wvls[:1], focs[:2])                   # warm-up
            r['host_refocus_s'], _ = timed(lambda: host_route(opm, n, fields, wvls, focs), 1)
        rec[f'n{n}'] = r
        print(f'{n}^2: through_focus_wavefront {r["through_focus_wavefront_s"]*1e3:9.3f} ms   '
              f'{K} x (zernike_fit + mtf) {r["k_zernike_fit_mtf_s"]*1e3:9.3f} ms   ratio {r["ratio_per_plane"]:6.2f}')
        print(f'{n}^2: kernels: opd-focus trace {r["kernel_opd_focus_trace_ms"][0]:.3f} ms, single opd trace '
              f'{r["kernel_opd_trace_ms"][0]:.3f} ms, per-plane consumers {r["kernel_per_plane_consumers_ms"][0]:.3f} ms, '
              f'mtf at {len(shifts)} shifts {r["kernel_mtf_shifts_ms"][0]:.3f} ms vs all {n} '
              f'{r["kernel_mtf_all_shifts_ms"][0]:.3f} ms')
        if 'host_refocus_s' in r:
            print(f'{n}^2: host trace_wavefront + {K} x focus_wavefront per tile {r["host_refocus_s"]:.2f} s')
    if a.host_rays not in a.num_rays:
        host_route(opm, a.host_rays, fields[:1], wvls[:1], focs[:2])
        t, _ = timed(lambda: host_route(opm, a.host_rays, fields, wvls, focs), 1)
        rec[f'host_refocus_n{a.host_rays}_s'] = t
        tfw = lambda: A.through_focus_wavefront(opm, a.host_rays, foc=focs, freqs=FREQS)   # noqa: E731
        tfw()
        rec[f'through_focus_wavefront_n{a.host_rays}_s'], _ = timed(tfw, a.reps)
        print(f'{a.host_rays}^2: host trace_wavefront + {K} x focus_wavefront per tile {t:.2f} s; '
              f'through_focus_wavefront {rec[f"through_focus_wavefront_n{a.host_rays}_s"]*1e3:.3f} ms')
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
