"""Time relative illumination on the double Gauss and the cellphone lens (3 fields x 3 wavelengths) at
num_rays x num_rays rays per tile (default 64, 256 and 1024):

1. ``analyses.relative_illumination`` end to end (synchronised wall clock, median of --reps);
2. the route a user has without it: one ``engine.trace_grid`` per tile with the ``d`` and ``status``
   outputs copied to the host, then ``engine.illumination_sums_host`` of each tile;
3. the kernels alone, with CUDA events over --launches back-to-back calls after a warm-up, repeated
   --rounds times (median, min and max of the rounds): the grid trace with the ``d`` and ``status``
   outputs, and ``rt_grid_illumination`` on its outputs.

The two routes' records are compared bit for bit.  Prints the card name and power limit of this run
and writes one JSON line.

    python tools/bench_relative_illumination.py [--num-rays 64 256 1024] [--reps 3] [--out FILE]
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


def per_tile_route(opm, tab, n, fields, wvls):
    """one trace per tile, its per-ray outputs copied to the host, the sums in numpy: [n_tiles, 10]"""
    from rayoptics_b200 import engine as E
    out = []
    for f in fields:
        for w in wvls:
            g = E.grid_for_model(opm, tab, n, fields=[f], wvls=[w], pupil_range=(-1.0, 1.0),
                                 apply_vignetting=False, ref_img=None)
            r = E.trace_grid(tab, g, outputs=('d', 'status'), summary=False)
            st, d = r.status.cpu().numpy(), r.d.cpu().numpy()
            out.append(E.illumination_sums_host(st.reshape(n, n), d[0].reshape(n, n), d[1].reshape(n, n),
                                                g.pupil_x[0], g.pupil_y[0]))
            g.close()
    return np.array(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--models', nargs='+', default=['dblgauss', 'cellphone'])
    ap.add_argument('--num-rays', type=int, nargs='+', default=[64, 256, 1024])
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    from rayoptics_b200 import model as M, analyses as A, engine as E
    if not torch.cuda.is_available():
        sys.exit('bench_relative_illumination needs a CUDA device')
    rec = {'bench': 'relative_illumination', 'card': card()}
    print(f'card (name, power limit, max SM clock): {rec["card"]}')
    for name in a.models:
        opm = M.OpticalModel.load(os.path.join(ROOT, 'tests', 'golden', 'models', name + '.json'))
        fields, wvls = list(opm.optical_spec.field_of_view.fields)[:3], list(opm.seq_model.wvlns)[:3]
        tab = A._table_for(opm)
        for n in a.num_rays:
            grid = E.grid_for_model(opm, tab, n, fields=fields, wvls=wvls, pupil_range=(-1.0, 1.0),
                                    apply_vignetting=False, ref_img=None)
            res = E.BundleResult(grid.n_rays, tab.n_ifc, torch.device('cuda', tab.device), ('d', 'status'))
            k_trace = per_launch_ms(lambda: E.trace_grid(tab, grid, res=res, summary=False), a.warmup,
                                    a.launches, a.rounds)
            k_illum = per_launch_ms(lambda: E.grid_illumination(grid, res.status, res.d[0], res.d[1]), a.warmup,
                                    a.launches, a.rounds)
            A.relative_illumination(opm, n, fields=fields, wvls=wvls)            # warm-up of this shape
            t_ri, r = timed(lambda: A.relative_illumination(opm, n, fields=fields, wvls=wvls), a.reps)
            per_tile_route(opm, tab, n, fields[:1], wvls[:1])
            t_host, rec_host = timed(lambda: per_tile_route(opm, tab, n, fields, wvls), a.reps)
            same = bool(np.array_equal(r.record.view(np.uint64), rec_host.view(np.uint64)))
            rec[f'{name}_n{n}'] = {'tiles': grid.n_tiles, 'rays': grid.n_rays, 'relative_illumination_s': t_ri,
                                   'per_tile_trace_host_sums_s': t_host, 'ratio': t_host/t_ri,
                                   'kernel_trace_ms': k_trace, 'kernel_illumination_ms': k_illum,
                                   'records_identical': same}
            print(f'{name} {n}^2 ({grid.n_tiles} tiles): relative_illumination {t_ri*1e3:9.3f} ms   per-tile '
                  f'trace + host sums {t_host*1e3:9.3f} ms   ratio {t_host/t_ri:7.2f}   records identical {same}')
            print(f'{name} {n}^2: kernels trace {k_trace[0]:8.3f} ms (min {k_trace[1]:.3f}, max {k_trace[2]:.3f}); '
                  f'rt_grid_illumination {k_illum[0]:8.3f} ms (min {k_illum[1]:.3f}, max {k_illum[2]:.3f}); '
                  f'{a.rounds} rounds of {a.launches} launches after {a.warmup}')
            grid.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
